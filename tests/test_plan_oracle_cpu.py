"""The whole host side against eager PyTorch, without a GPU.

    constructor under deferred_init -> tape -> planner -> InitPlan (JSON round trip) -> C-ABI
    descriptor table (InitPlan.descriptors) -> the stream's CPU restatement (oracle/tdx_oracle.c)

compared with the SAME constructor run eagerly on the CPU (which is what the reference's replay
gives, bit for bit: tests/test_parity_cpu_reference.py).  The kernels are checked against the
restatement element by element on the GPU (tests/test_kernels_gpu.py), so this closes the chain for
the part a GPU is not needed for: what the planner folds (constants, dead passes, epilogues,
segments, casts, index programs), the RNG bookkeeping and the shard arithmetic.

Tiers (SURVEY.md 8c): deterministic tensors T0 (bit-exact; index programs with float arithmetic to
4 ulp: ATen's CUDA arithmetic -- multiply by the fp32 reciprocal, powf -- is restated, the eager run
used the CPU's), RNG tensors T1 against the eager sample with the verbatim tolerances, hard range
checks from the folded parameters.  16-bit tensors are compared with the eager fp32 sample rounded
to the dtype (tests/test_t1_fullsize_gpu.py explains why not with ATen's own bf16 CPU kernel).
"""
import math

import pytest
import torch

from oracle import cases
from oracle import tdx_oracle as O
from torchdistx_b200.deferred_init import deferred_init
from torchdistx_b200.plan import InitPlan, offset_increment

SEED, OFFSET = 1234, 40


def named(m):
    # (tied weights under each of their names, like the plan lists them)
    return dict(list(m.named_parameters(remove_duplicate=False)) + list(m.named_buffers(remove_duplicate=False)))


def plan_of(case, dtype, tmp_path=None, post=None):
    def build():
        m = cases.build(case, dtype)
        return post(m) if post else m

    plan = InitPlan.from_module(deferred_init(build))
    if tmp_path is not None:  # what another process / another host language would start from
        path = str(tmp_path / "plan.json")
        plan.save(path)
        plan = InitPlan.load(path)
    return plan


def check_t1(name, x, ref, sixteen_bit, moments=True, scale=1.0, alpha=1e-3):
    from scipy import stats

    xd, rd = x.double().flatten(), ref.double().flatten()
    n = xd.numel()
    assert bool(torch.isfinite(xd).all()), name
    r_mean, r_std = rd.mean().item(), rd.std().item()
    if n < 64:  # (a few elements: the reference sample's own moments are too noisy to be a yardstick)
        return
    if r_std == 0.0:  # (a program that clamps -- almost -- everything to one value)
        # (equal up to the last bits: a `div_` after the clamp is a multiplication by the fp32 reciprocal
        # here, as in ATen's CUDA kernel, and a true division in the eager CPU run)
        tol = 2.0 ** -7 if sixteen_bit else 2.0 ** -21
        # (90 %: the eager sample happened to clamp everything; a wrong constant would match nowhere)
        assert ((xd - rd[0]).abs() <= tol * abs(rd[0].item())).double().mean().item() >= 0.9, name
        return
    if sixteen_bit and min(xd.unique().numel(), rd.unique().numel()) < 32:
        # (a 16-bit tensor whose spread is a few grid steps -- `x * 0.02 + 3.0` in bf16: the moments are
        # those of the rounding, not of the distribution; a wrong scale or offset still lands elsewhere)
        assert abs(xd.mean().item() - r_mean) <= 2.0 ** -7 * max(abs(r_mean), 1e-30) + 4 * r_std, name
        return
    if moments:  # (the bounds assume a sample whose variance estimate is not ruled by a few tail events)
        assert abs(xd.mean().item() - r_mean) <= scale * 5 * r_std / math.sqrt(n), (name, xd.mean().item(), r_mean, r_std, n)
        slack = 2.0 ** -8 if sixteen_bit else 0.0
        assert abs(xd.std().item() / r_std - 1) <= scale * 5 / math.sqrt(2 * n) + slack, (name, xd.std().item(), r_std, n)
    if n >= 1024:
        ks = stats.ks_2samp(xd.numpy(), rd.numpy())
        assert ks.pvalue > alpha, (name, ks)


def eager(case, dtype, post=None):
    """The constructor run for real: in the plan's dtype (deterministic tensors) and in fp32 (the
    RNG sample 16-bit tensors are compared with, after rounding)."""
    torch.manual_seed(SEED)
    a = cases.build(case, dtype)
    torch.manual_seed(SEED)
    b = cases.build(case, "fp32") if dtype != "fp32" else a
    if post:
        a, b = post(a), (post(b) if b is not a else a)
    return named(a), named(b)


def compare_with_eager(plan, got, own, wide, skip=(), clamps_by_ks_only=False, scale=1.0, alpha=1e-3):
    n_rng = n_const = n_iota = 0
    for e in plan.entries:
        if e.source == "alias":  # tied parameters stay one tensor
            assert got[e.name] is got[e.alias_of] and own[e.name] is own[e.alias_of], e.name
            continue
        if e.name in skip or e.source == "uninit":
            continue
        x, r = got[e.name], own[e.name].detach()
        assert x.dtype == r.dtype and tuple(x.shape) == tuple(r.shape), e.name
        if e.source == "value":
            assert torch.equal(x, r), e.name
            continue
        sixteen = x.dtype in (torch.bfloat16, torch.float16)
        flat, rflat, wflat = x.reshape(-1), r.reshape(-1), wide[e.name].detach().reshape(-1)
        for g in e.segment_list():
            lo, hi = g["begin"], g["end"]
            xs, rs = flat[lo:hi], rflat[lo:hi]
            if g["source"] == "uninit":
                continue
            if g["source"] == "const":
                assert torch.equal(xs.view(torch.uint8), rs.view(torch.uint8)), (e.name, lo, hi)
                n_const += 1
            elif g["source"] == "iota":
                if g["epilogue"]:
                    tol = 2.0 ** -7 if x.dtype == torch.bfloat16 else 2.0 ** -10 if x.dtype == torch.float16 else 4 * 2.0 ** -23
                    torch.testing.assert_close(xs.float(), rs.float(), rtol=tol, atol=0.0)
                else:
                    assert torch.equal(xs, rs), e.name
                n_iota += 1
            else:
                # 16-bit normals: the eager fp32 sample rounded (ATen's bf16 CPU normal_ draws from 8-bit
                # uniforms).  16-bit uniform programs: the eager 16-bit run itself -- every step of
                # `uniform_ -> erfinv_ -> mul_ -> add_ -> clamp_` rounds to the dtype, near 1.0 in steps
                # of 2^-8, and the epilogue restates exactly that (TDX_EPI_NOROUND is the opt-out)
                ref = wflat[lo:hi].to(x.dtype) if sixteen and g["source"] == "normal" else rs
                # (a clamp that keeps a far tail -- randn().clamp_(2, 3) -- leaves a mixture whose moments
                # are decided by a handful of elements: the distribution test alone judges those)
                clamped = clamps_by_ks_only and any((step[0] & 0xFF) == 4 for step in g["epilogue"])  # TDX_EPI_CLAMP (| flags)
                check_t1(f"{e.name}[{lo}:{hi}]", xs, ref, sixteen, moments=not clamped, scale=scale, alpha=alpha)
                if g["source"] == "uniform" and not g["epilogue"]:  # hard range: uniform in [from, to)
                    lim = lambda v: torch.tensor(v, dtype=x.dtype).item()  # (uniform_ rounds its bounds to the dtype)
                    assert xs.min().item() >= lim(g["p0"]) and xs.max().item() <= lim(g["p1"]), (e.name, g["p0"], g["p1"])
                    if not sixteen:
                        assert xs.max().item() < g["p1"], e.name
                n_rng += 1
    return n_rng, n_const, n_iota


@pytest.mark.parametrize("case,dtype", [("init_zoo", "fp32"), ("init_zoo", "bf16"), ("tiny_llama", "fp32"),
                                        ("tiny_llama", "bf16"), ("tiny_gpt2", "fp32"), ("padded_embeddings", "fp32"),
                                        ("padded_embeddings", "bf16"), ("mlp_stack", "fp32"),
                                        ("torch_transformer", "fp32")])
def test_descriptor_table_reproduces_the_eager_constructor(case, dtype, tmp_path):
    plan = plan_of(case, dtype, tmp_path)
    got, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    own, wide = eager(case, dtype)
    assert {e.name for e in plan.entries} == set(own)
    n_rng, n_const, n_iota = compare_with_eager(plan, got, own, wide)
    assert n_rng >= 2 and n_rng + n_const + n_iota >= 4, (n_rng, n_const, n_iota)
    # the generator ends where the passes (dead ones included, clones not) put it
    passes = {}
    for e in plan.entries:
        for pid, n in zip(e.rng_ids, e.rng_numels):
            passes[pid] = n
    assert end == OFFSET + sum(offset_increment(n) for n in passes.values())


def test_trunc_normal_stays_inside_its_bounds_and_casts_fold():
    plan = plan_of("init_zoo", "fp32")
    got = O.evaluate_plan(plan, SEED, OFFSET)[0]
    # nn.init.trunc_normal_(mean=0.1, std=0.02, a=-0.04, b=0.06): uniform -> erfinv -> mul -> add -> clamp;
    # the window ends two sigma BELOW the mean, so the mass piles up under b
    t = got["trunc"]
    assert -0.04 <= t.min().item() and t.max().item() <= torch.tensor(0.06).item() and t.median().item() > 0.05
    # Module.to(bf16) after an fp32 construction: the native 16-bit stream where nothing can tell,
    # the fp32 stream rounded (TDX_ALGO_WIDE32) where a second tensor must agree with the first
    plan = plan_of("cast_variant", "fp32")
    got = O.evaluate_plan(plan, SEED, OFFSET)[0]
    e = {x.name: x for x in plan.entries}
    assert e["b"].wide and not e["a"].wide and got["b"].dtype == torch.bfloat16
    assert torch.equal(got["b"], got["a"].to(torch.bfloat16))  # `b = a.to(bf16)`: bit for bit
    own, wide = eager("cast_variant", "fp32")
    compare_with_eager(plan, got, own, own)  # (the eager model IS an fp32 sample rounded by .to)


def test_rotary_buffers_of_a_converted_model():
    post = lambda m: m.to(torch.bfloat16)
    plan = plan_of("tiny_llama", "fp32", post=post)
    got = O.evaluate_plan(plan, SEED, OFFSET)[0]
    own, _ = eager("tiny_llama", "fp32", post=post)
    for name in ("model.rotary_emb.inv_freq", "model.rotary_emb.original_inv_freq"):
        assert got[name].dtype == torch.bfloat16
        # one rounding of the fp32 program: at most one bf16 ulp from the eager CPU result
        torch.testing.assert_close(got[name].float(), own[name].float(), rtol=2.0 ** -7, atol=0.0)
        assert (got[name] == own[name]).float().mean().item() > 0.9


def test_clones_share_their_sources_stream():
    plan = plan_of("clones", "fp32")
    got, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    own, _ = eager("clones", "fp32")
    by_pass = {}
    for e in plan.entries:
        if e.source in ("uniform", "normal") and not e.segments:
            by_pass.setdefault((tuple(e.rng_ids), e.source, e.p0, e.p1, tuple(e.epilogue)), []).append(e.name)
    twins = [v for v in by_pass.values() if len(v) > 1]
    assert twins, "the case has deep-copied layers"
    for names in twins:
        for other in names[1:]:
            assert torch.equal(got[names[0]], got[other]) and torch.equal(own[names[0]], own[other]), names
    passes = {pid: n for e in plan.entries for pid, n in zip(e.rng_ids, e.rng_numels)}
    assert end == OFFSET + sum(offset_increment(n) for n in passes.values())  # a copy consumes nothing


@pytest.mark.parametrize("case,dtype", [("tiny_llama", "bf16"), ("padded_embeddings", "fp32"), ("init_zoo", "fp32")])
def test_shards_concatenate_to_the_whole_and_agree_on_the_generator(case, dtype):
    plan = plan_of(case, dtype)
    full, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    kinds = {e.name: e.kind for e in plan.entries}
    for world in (2, 3, 8):
        parts = [O.evaluate_plan(plan, SEED, OFFSET, shard=(r, world))[:2] for r in range(world)]
        assert all(p[1] == end for p in parts)  # every rank advances its generator identically
        for name, t in full.items():
            if kinds[name] == "param" and t.dim() >= 1:
                rows = -(-t.shape[0] // world)
                for r, (p, _) in enumerate(parts):  # the layout of torch.chunk(t, world, 0)
                    exp = t[r * rows: (r + 1) * rows]
                    assert p[name].shape == exp.shape and torch.equal(p[name].reshape(-1).view(torch.uint8),
                                                                      exp.reshape(-1).view(torch.uint8)), (name, world, r)
            else:
                assert all(torch.equal(p[name].reshape(-1).view(torch.uint8), t.reshape(-1).view(torch.uint8))
                           for p, _ in parts), name


def test_seed_and_offset_select_the_stream():
    plan = plan_of("mlp_stack", "fp32")
    a = O.evaluate_plan(plan, SEED, OFFSET)[0]
    b = O.evaluate_plan(plan, SEED, OFFSET)[0]
    c = O.evaluate_plan(plan, SEED + 1, OFFSET)[0]
    d = O.evaluate_plan(plan, SEED, OFFSET + 4)[0]
    w = next(e.name for e in plan.entries if e.source in ("uniform", "normal"))
    assert torch.equal(a[w], b[w]) and not torch.equal(a[w], c[w]) and not torch.equal(a[w], d[w])


def test_a_parameter_stored_by_value_is_chunked_like_the_others():
    """A deterministic program the planner cannot fold (`tril`) is embedded in the plan; as a
    PARAMETER it is still this rank's rows only (what materialize_module(shard=...) does with a
    replayed parameter), as a buffer it is replicated."""
    from torch import nn

    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.p = nn.Parameter(torch.tril(torch.ones(7, 4)) * 0.5)
            self.register_buffer("b", torch.tril(torch.ones(5, 5)))
            self.w = nn.Parameter(torch.empty(7, 3).normal_())

    plan = InitPlan.from_module(deferred_init(M))
    kinds = {e.name: e.source for e in plan.entries}
    assert kinds["p"] == "value" and kinds["b"] == "value" and kinds["w"] == "normal", kinds
    full, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    assert torch.equal(full["p"], torch.tril(torch.ones(7, 4)) * 0.5)
    for world in (2, 3, 8):
        parts = [O.evaluate_plan(plan, SEED, OFFSET, shard=(r, world))[:2] for r in range(world)]
        assert all(e == end for _, e in parts)
        for name in ("p", "w"):
            assert torch.equal(torch.cat([p[name] for p, _ in parts]), full[name]), (name, world)
            assert [p[name].shape[0] for p, _ in parts] == [c.shape[0] for c in torch.chunk(full[name], world, 0)] + \
                [0] * (world - len(torch.chunk(full[name], world, 0))), (name, world)
        assert all(torch.equal(p["b"], full["b"]) for p, _ in parts)


@pytest.mark.parametrize("family", cases.FAMILIES + cases.FAMILIES_ENGINE_ONLY)
def test_model_families_initialise_to_what_their_constructors_compute(family):
    """Real constructors (HF `_init_weights`, torch.nn defaults) at toy sizes: every parameter and
    buffer the plan describes -- normal / uniform / truncated-normal weights, constant norms and
    biases, padded embedding rows, rotary and position index programs, tied weights -- against the
    eagerly built model, T0 / T1 (the fuzz tests' x1.5 bounds: ~40 statistical checks per family)."""
    fn = cases.families()[family]
    plan = InitPlan.from_module(deferred_init(fn))
    got = O.evaluate_plan(plan, SEED, OFFSET)[0]
    torch.manual_seed(0)
    own = named(fn())
    assert {e.name for e in plan.entries} == set(own)
    n_rng, n_const, n_iota = compare_with_eager(plan, got, own, own, clamps_by_ks_only=True, scale=1.5, alpha=1e-6)
    assert n_rng >= 2
    by_value = [e.name for e in plan.entries if e.source == "value"]
    assert len(by_value) <= 1, by_value  # (BatchNorm's num_batches_tracked / one HF scalar buffer: never a weight)
