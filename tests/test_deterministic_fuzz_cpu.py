"""The deterministic sources on the host, without a GPU: random index programs, sinusoid tables, band masks
and host copies (tests/det_programs.py), each with the planner's verdict restated from its rules.

For every seed: the fuse / replay verdict of plan_report against the program's label, then
InitPlan.from_module -> descriptors -> the CPU restatement of the kernels (oracle/tdx_oracle.c) against the same program run eagerly on
the CPU.  Bit-exact wherever the kernels do no fp32 arithmetic ATen's CPU kernels do differently: index
programs without steps, band masks, constants, copies and casts -- and every replayed program, which the
plan stores by value.  Programs with fp32 steps (ATen's CPU `/` divides where the CUDA kernel multiplies by
the reciprocal, its vectorised exp / log / pow are not libm's) are held to a few ulp, stated below;
tests/test_deterministic_fuzz_gpu.py holds the kernels to eager CUDA bit for bit."""
import random

import pytest
import torch

import band_replicas as R
import det_programs as D
from oracle import tdx_oracle as O
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, plan_report
from torchdistx_b200.plan import InitPlan

SEEDS = 6000  # seeds of the whole file (about a minute on one core)
CHUNKS = 10
# fp32 steps: 64 ulp, times (1 + |ln|y|| / 8) -- an exp of an argument that is an ulp apart is |arg| ulp apart,
# and a chain of up to five steps carries that on (exp(x / 7) through expm1 reaches 1e36: ln 83)
FP32_STEP_RTOL = 2.0 ** -17
ULP16 = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}


def verdict_errors(progs, report):
    """Programs whose planner verdict is not their label (a near miss fused, or a fusible program replayed),
    or fused as another source."""
    bad = []
    for p in progs:
        info = report[p.name]
        sources = {info["source"]} | {g["source"] for g in info["segments"]}  # (a padding row: a const segment first)
        if p.fuse and not (info["fusible"] and p.family in sources):
            bad.append(f"{p.name}: label fuse/{p.family}, planner {info['source']} "
                       f"(first unfusable op {info['first_unfusable_op']!r}): {p.text}")
        if not p.fuse and info["fusible"]:
            bad.append(f"{p.name}: label replay, planner fused it as {info['source']}: {p.text}")
    return bad


def same_bits(got, want):
    """Equal bytes, or both NaN."""
    if got.dtype in (torch.float32, torch.bfloat16, torch.float16):
        return (got == want) | (torch.isnan(got) & torch.isnan(want)) | (
            got.view(torch.uint8).view(-1, got.element_size()) == want.view(torch.uint8).view(-1, got.element_size())
        ).all(1).view(got.shape)
    return got == want


def close(got, want, p):
    """Within the stated bound of eager CPU: see the module docstring."""
    exact = same_bits(got, want)
    if p.exact_on_cpu():
        return exact
    g, w = got.double(), want.double()
    finite = torch.isfinite(g) & torch.isfinite(w)
    if got.dtype == torch.float32:
        # (+ 2^-22: log of an argument near 1 cancels, the difference stays absolute)
        tol = FP32_STEP_RTOL * (1 + w.abs().clamp(min=1e-30).log().abs() / 8) * w.abs() + 2.0 ** -22
    else:  # one fp32 difference can move a 16-bit rounding by one step
        tol = ULP16[got.dtype] * w.abs() + 2.0 ** -24
    return exact | (finite & ((g - w).abs() <= tol))


def sincos_close(got, want, p, entry):
    """Sinusoid tables, as tests/test_sincos_tables_cpu.py: 4 * 2^-24 in fp32 (libm's and ATen's CPU
    sinf / cosf), one step in 16 bits, plus what a column value that differs carries through r * f."""
    seg = next(g for g in entry.segments if g["source"] == "sincos")
    half = seg["sincos_half"]
    col = C.make_desc(0, dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_count=half, p0=seg["p0"], p1=seg["p1"],
                      epi=seg["epilogue"])
    f_o = R.as_tensor(O.generate(col), torch.float32).double()
    f_e = p.col().double()
    differ = ~((f_o == f_e) | (torch.isnan(f_o) & torch.isnan(f_e)))
    rows = got.shape[0]
    slack = torch.where(differ, (rows - 1) * (2 * (f_o - f_e).abs() + f_e.abs() * 2.0 ** -23), torch.zeros(half))
    slack = torch.nan_to_num(torch.cat([slack, slack]), nan=0.0, posinf=0.0)[None, :]
    g, w = got.double(), want.double()
    ok = same_bits(got, want) | ((g - w).abs() <= 4 * 2.0 ** -24 + slack + (0 if got.dtype == torch.float32 else
                                                                            ULP16[got.dtype] * w.abs() + 2.0 ** -24))
    # (a column of inf or NaN: sin and cos of it are NaN on both sides, or the row is 0)
    return ok | ~torch.isfinite(f_e).repeat(2)[None, :]


def check_seed(seed, stats):
    r = random.Random(seed)
    progs = D.gen_module(r)
    m = deferred_init(D.DetModule, progs)
    errors = verdict_errors(progs, plan_report(m))
    plan = InitPlan.from_module(m)
    got = O.evaluate_plan(plan, 7, 0)[0]
    eager = dict(list(D.DetModule(progs).named_parameters()) + list(D.DetModule(progs).named_buffers()))
    entries = {e.name: e for e in plan.entries}
    for p in progs:
        x, want = got[p.name], eager[p.name].detach()
        assert x.dtype == want.dtype and x.shape == want.shape, (seed, p.name, x.dtype, want.dtype, p.text)
        e = entries[p.name]
        ok = sincos_close(x, want, p, e) if e.source == "sincos" else close(x, want, p) if e.source != "value" \
            else same_bits(x, want)
        if not bool(ok.all()):
            i = (~ok).flatten().nonzero()[:4].flatten()
            errors.append(f"{p.name}: {int((~ok).sum())} of {ok.numel()} differ, e.g. got {x.flatten()[i].tolist()} "
                          f"want {want.flatten()[i].tolist()}: {p.text}")
        key = p.family if p.fuse else "replay"
        stats[key] = stats.get(key, 0) + 1
    return [f"seed {seed}: {m}" for m in errors]


@pytest.mark.parametrize("chunk", range(CHUNKS))
def test_restated_plans_match_eager_cpu(chunk):
    stats, errors = {}, []
    per = SEEDS // CHUNKS
    for seed in range(chunk * per, (chunk + 1) * per):
        errors += check_seed(seed, stats)
    assert not errors, "\n".join(errors[:20]) + f"\n({len(errors)} in all)"
    # the generator keeps every family on the fused path and keeps near misses in the mix
    for fam in ("iota", "sincos", "band", "gather", "replay"):
        assert stats.get(fam, 0) >= per // 20, stats


def test_shards_of_restated_plans_concatenate_to_the_whole():
    """Parameters are chunked along dim 0: each element range starts mid-row, mid-period, mid-vector."""
    for seed in range(40):
        r = random.Random(10_000 + seed)
        progs = D.gen_module(r)
        plan = InitPlan.from_module(deferred_init(D.DetModule, progs))
        whole = O.evaluate_plan(plan, 7, 0)[0]
        kinds = {e.name: e.kind for e in plan.entries}
        for world in (2, 3, 8):
            parts = [O.evaluate_plan(plan, 7, 0, shard=(rank, world))[0] for rank in range(world)]
            for name, t in whole.items():
                if kinds[name] == "param" and t.dim() >= 1:
                    cat = torch.cat([q[name] for q in parts])
                else:
                    assert all(torch.equal(q[name].view(torch.uint8), t.view(torch.uint8)) for q in parts), name
                    continue
                assert torch.equal(cat.reshape(-1).view(torch.uint8), t.reshape(-1).view(torch.uint8)), (seed, name, world)
