"""State-space initialisers on the H100: the superset epilogue and the broadcast index against ATen's
own CUDA kernels (bit for bit, on the same draws), against the CPU restatement, and the replica models
end to end through materialize_module and InitPlan."""
import math

import pytest
import torch

import ssm_replicas as R
from oracle import tdx_oracle as O
from torchdistx_b200 import _C
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, last_materialize_stats, materialize_module, materialize_tensor
from torchdistx_b200.plan import InitPlan

pytestmark = pytest.mark.gpu

TDX = {torch.float32: C.TDX_F32, torch.bfloat16: C.TDX_BF16, torch.float16: C.TDX_F16}
N = 1 << 20
C1 = math.log(R.T_MAX) - math.log(R.T_MIN)
C2 = math.log(R.T_MIN)


def fused(dtype, lo, hi, epi, n=N):
    out = torch.empty(n, dtype=dtype, device="cuda")
    d = C.make_desc(out.data_ptr(), dtype=TDX[dtype], src=C.TDX_SRC_UNIFORM, elem_count=n, seed=77, p0=lo, p1=hi,
                    epi=epi)
    ws = torch.empty(C.prepare([d]), dtype=torch.uint8, device="cuda")
    C.submit(ws.data_ptr(), ws.numel())
    torch.cuda.synchronize()
    return out, d


def dt_eager(x):
    dt = torch.exp(x * C1 + C2).clamp(min=R.FLOOR)
    return dt + torch.log(-torch.expm1(-dt))


CASES = {
    "exp": ((-4.0, 4.0), [(C.TDX_EPI_EXP,)], torch.exp),
    "log": ((0.0, 8.0), [(C.TDX_EPI_LOG,)], torch.log),
    "expm1": ((-4.0, 4.0), [(C.TDX_EPI_EXPM1,)], torch.expm1),
    "inv_softplus": ((1e-4, 2.0), [(C.TDX_EPI_INV_SOFTPLUS,)], lambda x: x + torch.log(-torch.expm1(-x))),
    "muladd": ((0.0, 1.0), [(C.TDX_EPI_MULADD, C1, C2)], lambda x: x * C1 + C2),
    "dt_chain": ((0.0, 1.0), [(C.TDX_EPI_MULADD, C1, C2), (C.TDX_EPI_EXP,), (C.TDX_EPI_CLAMP, R.FLOOR, math.inf),
                              (C.TDX_EPI_INV_SOFTPLUS,)], dt_eager),
}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", sorted(CASES))
def test_fused_step_equals_aten_on_the_same_draws(case, dtype):
    (lo, hi), epi, eager = CASES[case]
    raw, _ = fused(dtype, lo, hi, [])
    got, d = fused(dtype, lo, hi, epi)
    want = eager(raw)
    assert want.dtype == dtype
    assert torch.equal(got.view(torch.uint8), want.view(torch.uint8)), \
        (case, dtype, int((got.view(torch.uint8) != want.view(torch.uint8)).sum()))
    # the CPU restatement (C libm): within a few ulp of the libdevice functions -- of the operands where
    # x + log(-expm1(-x)) cancels (|terms| < 10 here)
    head = C.make_desc(0, dtype=d.dtype, src=d.src, elem_count=1 << 14, seed=77, p0=lo, p1=hi, epi=epi)
    exp_bits = R.as_tensor(O.generate(head), dtype).cuda()
    g = got[: 1 << 14]
    cancels = dtype == torch.float32 and case in ("inv_softplus", "dt_chain")
    ok = torch.isclose(g.float(), exp_bits.float(), rtol=4e-6 if dtype == torch.float32 else 1e-2,
                       atol=1e-5 if cancels else 0) | \
        (torch.isnan(g) & torch.isnan(exp_bits)) | (g == exp_bits)
    assert ok.all(), (case, dtype, g[~ok][:4], exp_bits[~ok][:4])


@pytest.mark.parametrize("begin,count,shift", [(0, 16 * 4096, 0), (3, 16 * 4096 - 7, 1), (4097, 999, 3)])
def test_periodic_iota_is_arange_expand_log(begin, count, shift):
    D, n = 4096, 16
    whole = torch.log(torch.arange(1, n + 1, dtype=torch.float32, device="cuda")[None, :].expand(D, -1).contiguous())
    buf = torch.full((count + shift,), float("nan"), device="cuda")
    d = C.make_desc(buf.data_ptr() + 4 * shift, dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_begin=begin, elem_count=count,
                    p0=1, p1=1, epi=[(C.TDX_EPI_LOG,)], iota_period=n)
    ws = torch.empty(C.prepare([d]), dtype=torch.uint8, device="cuda")
    assert C.submit(ws.data_ptr(), ws.numel()) == 1
    torch.cuda.synchronize()
    assert torch.equal(buf[shift:], whole.view(-1)[begin: begin + count])
    cols = torch.arange(1, n + 1, dtype=torch.float32, device="cuda")[:, None].expand(-1, 7).contiguous().log()
    out = torch.empty(n * 7, device="cuda")
    d = C.make_desc(out.data_ptr(), dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_count=n * 7, p0=1, p1=1,
                    epi=[(C.TDX_EPI_LOG,)], iota_period=n, iota_repeat=7)
    ws = torch.empty(C.prepare([d]), dtype=torch.uint8, device="cuda")
    C.submit(ws.data_ptr(), ws.numel())
    torch.cuda.synchronize()
    assert torch.equal(out, cols.view(-1))
    assert torch.equal(out.cpu(), R.as_tensor(O.generate(d), torch.float32)) or \
        (out.cpu().view(torch.int32) - R.as_tensor(O.generate(d), torch.float32).view(torch.int32)).abs().max() <= 1


class Model(torch.nn.Module):
    def __init__(self, dtype=torch.float32):
        super().__init__()
        self.mamba2 = R.Mamba2Mixer(4096, dtype, "cuda")
        self.mamba = R.MambaMixer(512, 16, 16, "cuda")
        self.qwen = R.GatedDeltaNet(4096, dtype, "cuda")
        self.bufs = R.Buffers(12, 5, "cuda")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_materialize_replicas(dtype):
    torch.manual_seed(3)
    m = deferred_init(Model, dtype)
    plan = InitPlan.from_module(m)
    gen = torch.cuda.default_generators[0]
    off0 = gen.get_offset()
    materialize_module(m)
    torch.cuda.synchronize()
    st = last_materialize_stats()
    assert st["generic_ops"] == 0 and st["fused_tensors"] == st["tensors"], st
    off1 = gen.get_offset()
    # A_log: bit-exact with the eager construction on CUDA
    assert torch.equal(m.mamba2.A_log, torch.log(torch.arange(1, 4097, dtype=torch.float32, device="cuda")))
    assert torch.equal(m.mamba.A_log, torch.log(torch.arange(1, 17, dtype=torch.float32, device="cuda"))[None, :]
                       .expand(512, -1).contiguous())
    assert torch.equal(m.bufs.cols, torch.log(torch.arange(1, 13, dtype=torch.float32, device="cuda")[:, None]
                                              .expand(-1, 5).contiguous()))
    assert torch.equal(m.bufs.rep, torch.log(torch.arange(1, 13, dtype=torch.float32, device="cuda").repeat(5, 1)))
    # RNG tensors: hard ranges (the dtype's rounding of the bounds), no NaN
    lo, hi = R.inv_softplus(R.T_MIN), R.inv_softplus(R.T_MAX)
    tol = 1e-5 if dtype == torch.float32 else 0.02 * abs(lo)
    for dt in (m.mamba2.dt_bias.float(), m.mamba.dt_proj.bias.float()):
        assert not torch.isnan(dt).any() and dt.min() >= lo - tol and dt.max() <= hi + tol
        assert dt.std() > 0.1
    qa = m.qwen.A_log.float()
    assert not torch.isnan(qa).any() and qa.max() <= math.log(16) + 0.01 and qa.std() > 0.5
    # InitPlan.materialize from the same generator state: the same bits
    gen.set_offset(off0)
    t = plan.materialize()
    assert gen.get_offset() == off1
    for name, p in list(m.named_parameters()) + list(m.named_buffers()):
        assert torch.equal(t[name], p), name
    # shards concatenate to the whole
    for world in (2, 3):
        parts = []
        for r in range(world):
            gen.set_offset(off0)
            parts.append(plan.materialize(shard=(r, world)))
        for name, p in m.named_parameters():
            whole = torch.cat([q[name].reshape(-1) for q in parts])
            assert torch.equal(whole, p.reshape(-1)), (world, name)


def test_index_program_divided_by_an_inexact_scalar():
    """`exp(arange(n)) / 0.001`: ATen's CUDA kernel multiplies by float(1.0 / 0.001) = 1000.0, not by
    1.0f / float(0.001) = 999.99994 (the step the planner used to fold: 59 of 171 elements an ulp off)."""
    build = lambda: torch.arange(171, device="cuda").exp() / 0.001  # noqa: E731
    t = deferred_init(build)
    assert dict(_C.plan_info(t))["source"] == "iota"
    got = materialize_tensor(t)
    assert last_materialize_stats()["generic_ops"] == 0
    assert torch.equal(got, build())
