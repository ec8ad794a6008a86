"""Tensor-parallel blocks on the H100: the window kernels against the CPU restatement
(oracle/tdx_oracle.c) and against the plain kernels' unsharded tensor, and the engine's Shard(d) blocks
(ranks emulated in one process) against the unsharded materialize_module of the same recording."""
import math

import numpy as np
import pytest
import torch
from torch.distributed.tensor.parallel import ColwiseParallel, RowwiseParallel

from oracle import cases
from oracle import tdx_oracle as O
from torchdistx_b200 import _C
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import _tp_slots, deferred_init, last_descriptors, last_materialize_stats, \
    materialize_module
from torchdistx_b200.parallel import tp_placements
from torchdistx_b200.plan import InitPlan

from test_tp_shard_cpu import COPIES_ARGS, COPIES_PLAN, MODELS, Copies, block

pytestmark = pytest.mark.gpu
TORCH = {C.TDX_F32: torch.float32, C.TDX_BF16: torch.bfloat16, C.TDX_F16: torch.float16}


def run(descs):
    ws = torch.empty(C.load().tdx_init_workspace_bytes(len(descs)), dtype=torch.uint8, device="cuda")
    C.launch(descs, ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def desc(t, dtype, src, begin, count, offset=0, **kw):
    return C.make_desc(t.data_ptr() + offset * t.element_size(), dtype=dtype, src=src, elem_begin=begin,
                       elem_count=count, seed=0x5EED, offset=64, p0=kw.pop("p0", 0.0), p1=kw.pop("p1", 1.0), **kw)


def window(t, dtype, src, begin, count, w, p, offset=0, **kw):
    d = desc(t, dtype, src, begin, count, offset, **kw)
    d.reserved |= C.TDX_FLAG_WINDOW
    d.fill_bits[0], d.fill_bits[1] = w, p
    return d


CASES = [(dt, src, algo) for dt in (C.TDX_F32, C.TDX_BF16, C.TDX_F16) for src in (C.TDX_SRC_UNIFORM, C.TDX_SRC_NORMAL)
         for algo in ((0, C.TDX_ALGO_WIDE32) if dt != C.TDX_F32 else (0,))]
EPIS = {"none": [], "mul_add": [(C.TDX_EPI_MUL, 0.5), (C.TDX_EPI_ADD, 0.25)], "exp": [(C.TDX_EPI_EXP, 0.0)],
        # trunc_normal_(std=0.02, a=-0.04, b=0.04): uniform_(2l - 1, 2u - 1), erfinv_, mul_, add_, clamp_ (uniform
        # draws only)
        "trunc_normal": [(C.TDX_EPI_ERFINV, 0.0), (C.TDX_EPI_MUL, 0.02 * math.sqrt(2.0)), (C.TDX_EPI_ADD, 0.0),
                         (C.TDX_EPI_CLAMP, -0.04, 0.04)]}
# (rows, cols, first column, columns, destination offset in elements, elements cut off the end): whole
# tiles of aligned vectors, a last partial tile, a last partial run and vector, unaligned W and start,
# and an unaligned destination
GEOMETRY = {"aligned": (96, 4096, 1024, 1536, 0, 0), "aligned_tail": (37, 4096, 1024, 1536, 0, 0),
            "ragged_end": (20, 512, 128, 256, 0, 3), "unaligned": (37, 1000, 7, 333, 0, 0),
            "odd_dst": (20, 256, 8, 64, 1, 0)}


@pytest.mark.parametrize("dt,src,algo,epi", [(*c, k) for c in CASES for k in EPIS
                                             if k != "trunc_normal" or c[1] == C.TDX_SRC_UNIFORM])
@pytest.mark.parametrize("geo", list(GEOMETRY))
def test_window_kernel_against_the_restatement_and_the_plain_kernel(dt, src, algo, epi, geo):
    rows, cols, c0, ncol, off, cut = GEOMETRY[geo]
    n = rows * ncol - cut
    whole = torch.empty(rows * cols, dtype=TORCH[dt], device="cuda")
    out = torch.zeros(n + off, dtype=TORCH[dt], device="cuda")
    kw = dict(algo=algo, epi=EPIS[epi], p0=-0.95 if epi == "trunc_normal" else 0.0, p1=0.95 if epi == "trunc_normal" else 0.5)
    run([desc(whole, dt, src, 0, rows * cols, **kw)])
    run([window(out, dt, src, c0, n, ncol, cols, off, **kw)])
    got = out[off:]
    if not EPIS[epi]:  # the same generator code as the plain kernels: bit for bit
        want = whole.view(rows, cols)[:, c0:c0 + ncol].reshape(-1)[:n]
        assert torch.equal(got.view(torch.uint8), want.contiguous().view(torch.uint8))
    d = window(out, dt, src, c0, n, ncol, cols, **kw)
    e = torch.from_numpy(O.generate(d).view(np.uint8)).view(TORCH[dt]).double()
    g = got.cpu().double()
    if src == C.TDX_SRC_UNIFORM and not EPIS[epi]:
        assert torch.equal(g, e)
    elif dt == C.TDX_F32:  # the generators' approximate MUFU functions (and CUDA's erfinvf, expf) against libm
        assert bool(((g - e).abs() <= 2e-5 * (1 + e.abs())).all()), float(((g - e).abs() / (1 + e.abs())).max())
    else:
        # T1' (DESIGN.md section 5): identical bits but for <= 0.2 % of the elements, 1 ulp apart; every step
        # of an epilogue rounds again, so a chain may flip up to 0.2 % per rounding, by an ulp of its
        # largest intermediate (the drawn value: |x| < 2 here)
        steps = 1 + len(EPIS[epi])
        assert (g != e).double().mean().item() <= 0.002 * steps
        mag = torch.maximum(g.abs(), e.abs()).clamp_min(1.0 if EPIS[epi] else 2.0 ** -14)
        ulp = torch.exp2(torch.floor(torch.log2(mag)) - (7 if dt == C.TDX_BF16 else 10))
        if algo == C.TDX_ALGO_WIDE32 and src == C.TDX_SRC_NORMAL:
            # the fp32 Box-Muller value, then rounded: T1''s fp32 bar, std min(1e-3, 4e-7/|z| + 2e-6 (1 + |z|)),
            # and 1 ulp of the 16-bit type
            z = (e / 0.5).abs().clamp_min(1e-30)
            ulp = ulp + 0.5 * torch.clamp(4e-7 / z + 2e-6 * (1 + z), max=1e-3)
        assert bool(((g - e).abs() <= ulp * (1 + 1e-6)).all()), float(((g - e).abs() / ulp).max())


def test_windowed_and_plain_descriptors_in_one_submission():
    a = torch.empty(64, 512, dtype=torch.bfloat16, device="cuda")
    b = torch.empty(64 * 128, dtype=torch.bfloat16, device="cuda")
    da = desc(a, C.TDX_BF16, C.TDX_SRC_NORMAL, 0, a.numel(), p1=0.02)
    db = window(b, C.TDX_BF16, C.TDX_SRC_NORMAL, 256, b.numel(), 128, 512, p1=0.02)
    run([da, db])
    a1, b1 = a.clone(), b.clone()
    a.zero_(), b.zero_()
    run([da])
    run([db])
    assert torch.equal(a, a1) and torch.equal(b, b1) and torch.equal(b1.view(64, 128), a1[:, 256:384])


def tp_local(build, plan, rank, world, seed=1):
    """{parameter name: this rank's tensor}, built by the engine call materialize_module(parallelize_plan=...)
    makes (its traversal, mask and tied-parameter rule; ranks emulated in one process), and the layouts."""
    torch.manual_seed(seed)
    m = deferred_init(build)
    dims = tp_placements(m, plan)
    slots, unique, make = _tp_slots(m, dims)
    done = make(torch.device("cuda"), rank, world)
    return {slots[i][2]: done[i] for i in unique if slots[i][2]}, dims


def tp_blocks(case, dtype, rank, world):
    return tp_local(lambda: cases.build(case, dtype, "cuda"), MODELS[case](), rank, world)


@pytest.mark.parametrize("case", list(MODELS))
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_blocks_concatenate_to_the_unsharded_model(case, dtype):
    torch.manual_seed(1)
    full = deferred_init(lambda: cases.build(case, dtype, "cuda"))
    materialize_module(full)
    whole = {k: v.detach() for k, v in full.named_parameters()}
    for world in (2, 3, 8):
        parts = [tp_blocks(case, dtype, r, world) for r in range(world)]
        dims = parts[0][1]
        for r, (got, _) in enumerate(parts):
            for k, t in whole.items():
                want = block(t, world, r, dims.get(k))
                assert got[k].shape == want.shape and torch.equal(got[k].view(torch.uint8).reshape(-1),
                                                                  want.contiguous().view(torch.uint8).reshape(-1)), (k, r)
        assert any(dims[k] == 1 for k in whole if k in dims)
    assert last_materialize_stats()["generic_ops"] == 0


def test_init_plan_materialize_matches_the_engine():
    for r in range(3):
        got, dims = tp_blocks("tiny_llama", "bf16", r, 3)
        torch.manual_seed(1)
        plan = InitPlan.from_module(deferred_init(lambda: cases.build("tiny_llama", "bf16", "cuda")))
        mine = plan.materialize(shard=(r, 3), placements=dims)
        for k, t in got.items():
            assert torch.equal(mine[k].view(torch.uint8), t.view(torch.uint8)), (k, r)


def test_llama3_8b_down_proj_at_tp8_statistics():
    w = torch.empty(4096, 1792, dtype=torch.bfloat16, device="cuda")
    run([window(w, C.TDX_BF16, C.TDX_SRC_NORMAL, 1792 * 3, w.numel(), 1792, 14336, p1=0.02)])
    x = w.double()
    n = x.numel()
    assert abs(x.mean().item()) <= 5 * 0.02 / math.sqrt(n)
    assert abs(x.std().item() / 0.02 - 1) <= 5 / math.sqrt(2 * n) + 2.0 ** -8
    from scipy import stats
    assert stats.kstest((x.flatten()[:: 97] / 0.02).cpu().numpy(), "norm").pvalue > 1e-3


def whole_of(build, seed=1):
    torch.manual_seed(seed)
    full = deferred_init(build)
    materialize_module(full)
    return {k: v.detach() for k, v in full.named_parameters()}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_copy_programs_under_shard_1_are_built_whole_and_narrowed(dtype):
    args = COPIES_ARGS()
    build = lambda: Copies(*args, dtype).cuda()
    whole = whole_of(build)
    for world in (2, 3, 8):
        for r in range(world):
            got, dims = tp_local(build, COPIES_PLAN(), r, world)
            assert last_materialize_stats()["narrowed_tensors"] == 2 and last_materialize_stats()["generic_ops"] == 0
            for k, t in whole.items():
                want = block(t, world, r, dims.get(k))
                assert got[k].shape == want.shape and torch.equal(got[k], want), (k, world, r)


LLAMA3_8B = dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                 num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=8192)
LLAMA3_8B_PLAN = lambda: {
    "model.embed_tokens": RowwiseParallel(), "lm_head": ColwiseParallel(),
    **{f"model.layers.*.{m}": ColwiseParallel() for m in ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj",
                                                            "mlp.gate_proj", "mlp.up_proj")},
    "model.layers.*.self_attn.o_proj": RowwiseParallel(), "model.layers.*.mlp.down_proj": RowwiseParallel()}


def llama3_8b():
    import transformers as T

    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            return T.LlamaForCausalLM(T.LlamaConfig(**LLAMA3_8B))
    finally:
        torch.set_default_dtype(prev)


def test_llama3_8b_tp8_rank_blocks_are_slices_of_the_whole_model():
    """Full size, bf16: the Colwise blocks go through the shared-memory-table kernel (a launch of GBs),
    the Rowwise ones through the window kernels, in one submission."""
    whole = whole_of(llama3_8b)
    for r in (0, 5):
        got, dims = tp_local(llama3_8b, LLAMA3_8B_PLAN(), r, 8)
        descs = last_descriptors()
        assert sum(bool(d.reserved & C.TDX_FLAG_WINDOW) for d in descs) == 64  # o_proj and down_proj, 32 layers
        for k, t in whole.items():
            want = block(t, 8, r, dims.get(k))
            assert got[k].shape == want.shape and torch.equal(got[k].view(torch.int16), want.contiguous().view(torch.int16)), (k, r)
        del got
        torch.cuda.empty_cache()


def test_materialize_module_on_a_one_rank_mesh_hands_dtensors_to_parallelize_module(tmp_path):
    import torch.distributed as dist
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import DTensor, Replicate, Shard
    from torch.distributed.tensor.parallel import parallelize_module

    dist.init_process_group("nccl", init_method=f"file://{tmp_path}/pg", rank=0, world_size=1)
    try:
        mesh = init_device_mesh("cuda", (1,))
        for case in MODELS:
            whole = whole_of(lambda: cases.build(case, "bf16", "cuda"))
            torch.manual_seed(1)
            m = deferred_init(lambda: cases.build(case, "bf16", "cuda"))
            dims = tp_placements(m, MODELS[case]())
            materialize_module(m, device_mesh=mesh, parallelize_plan=MODELS[case]())
            before = {k: p for k, p in m.named_parameters()}
            for k, p in before.items():
                if k in dims:
                    want = [Replicate()] if dims[k] is None else [Shard(dims[k])]
                    assert isinstance(p.data, DTensor) and list(p.placements) == want and p.shape == whole[k].shape, k
                    assert p.to_local().is_cuda and torch.equal(p.to_local(), whole[k]), k
                else:
                    assert not isinstance(p.data, DTensor) and torch.equal(p, whole[k]), k
            parallelize_module(m, mesh, MODELS[case]())
            for k, p in m.named_parameters():
                if k in before and k in dims:
                    assert torch.equal(p.to_local(), before[k].to_local()) and list(p.placements) == list(before[k].placements), k
    finally:
        dist.destroy_process_group()
