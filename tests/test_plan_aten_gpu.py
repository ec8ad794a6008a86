"""Plans for ATen's own CUDA stream on the H100. A plan built with `rng="aten"`, saved, loaded and
materialised after `torch.manual_seed(s)` holds the tensors ATen gives, bit for bit, and leaves the
generator at the same offset. This holds whole, as `shard=` chunks, as tensor-parallel `placements=` blocks,
as FSDP2 x TP `blocks=`, and handed to FSDP2 in place by `init_sharded_module`. Its descriptor table is the
one `materialize_module(rng="aten")` submits for the same layout.

The yardstick is eager CUDA for a module whose constructor draws in materialize_module's traversal order
(children first, then own parameters and buffers). For other modules it is the op-by-op ATen replay of
the same recording, `fused=False`: the reference's semantics. A Hugging Face model draws every linear's
default initialisation before `_init_weights` redraws them, and GPT-2 draws for an `lm_head` weight that
tying then drops. Eager order cannot be recovered from such a recording."""
import os
import sys

import pytest
import torch
import torch.multiprocessing as mp
from torch import nn

from oracle import cases
from torchdistx_b200 import _C
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, last_descriptors, materialize_module
from torchdistx_b200.parallel import local_block, tp_placements
from torchdistx_b200.plan import InitPlan, init_sharded_module

import ssm_replicas as R
from test_fsdp_tp_cpu import MESHES, MODELS, apply_steps, built, coordinates, fake_blocks, fake_rank, shard_2d
from test_tp_shard_cpu import MODELS as TP_PLANS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 21


def fp32_then_bf16(make):
    def build():
        prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.float32)
        try:
            with torch.device("cuda"):
                return make().to(torch.bfloat16)
        finally:
            torch.set_default_dtype(prev)
    return build


class StateSpace(nn.Module):
    """Mamba-2, Mamba and Qwen3-Next initialisers: `exp`, `clamp`, `log`, `expm1` and the inverse softplus
    on draws, and `log` of broadcast index programs."""

    def __init__(self):
        super().__init__()
        self.mamba2 = R.Mamba2Mixer(96, device="cuda")
        self.mamba = R.MambaMixer(96, 16, device="cuda")
        self.qwen = R.GatedDeltaNet(64, device="cuda")


def layers():
    """Draws in traversal order: default inits, a padding row, a 16-bit normal and a truncated normal."""
    m = nn.Sequential(nn.Linear(300, 77), nn.Embedding(1003, 96, padding_idx=1), nn.LayerNorm(96),
                      nn.Linear(96, 40, bias=False))
    nn.init.trunc_normal_(m[3].weight, std=0.02)  # (the last tensor drawn: its two passes stay in traversal order)
    return m


def bf16_layers():
    with torch.device("cuda"):
        return layers().to(torch.bfloat16).requires_grad_(False).requires_grad_(True)


# name -> (constructor, the default dtype it records under, drawn in traversal order)
BUILDS = {
    "layers_fp32": (lambda: cases.build("mlp_stack", "fp32", "cuda"), torch.float32, True),
    "layers_fp32_then_bf16": (fp32_then_bf16(layers), torch.float32, True),
    "state_space": (StateSpace, torch.float32, True),
    "tiny_llama_bf16": (lambda: cases.build("tiny_llama", "bf16", "cuda"), torch.bfloat16, False),
    "init_zoo_fp32": (lambda: cases.build("init_zoo", "fp32", "cuda"), torch.float32, False),
    "tiny_gpt2_fp32": (lambda: cases.build("tiny_gpt2", "fp32", "cuda"), torch.float32, False),
    "llama_fp32_then_bf16": (fp32_then_bf16(cases.tiny_llama), torch.float32, False),
}


def tensors(m):
    return {k: v.detach() for k, v in list(m.named_parameters(remove_duplicate=False)) +
            list(m.named_buffers(remove_duplicate=False))}


def reference(build, default_dtype=torch.float32, in_order=False, seed=SEED):
    """The yardstick's tensors and the generator's offset after them: eager CUDA, or the replay."""
    torch.manual_seed(seed)
    if in_order:
        m = build()
    else:
        m = deferred_init(build)
        torch.manual_seed(seed)
        prev = torch.get_default_dtype()
        torch.set_default_dtype(default_dtype)  # (a factory recorded without a dtype takes the current one)
        try:
            _C.materialize_module(m, False, None, None, None, False)
        finally:
            torch.set_default_dtype(prev)
    return tensors(m), torch.cuda.default_generators[0].get_offset()


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(
        a.detach().contiguous().reshape(-1).view(torch.uint8), b.detach().contiguous().reshape(-1).view(torch.uint8))


def saved_plan(build, tmp_path):
    InitPlan.from_module(deferred_init(build), rng="aten").save(str(tmp_path / "p.json"))
    plan = InitPlan.load(str(tmp_path / "p.json"))
    assert plan.rng == "aten"
    return plan


@pytest.mark.parametrize("case", list(BUILDS))
def test_saved_plan_is_aten(case, tmp_path):
    build = BUILDS[case][0]
    want, want_offset = reference(*BUILDS[case])
    plan = saved_plan(build, tmp_path)
    torch.manual_seed(SEED)
    got = plan.materialize(device="cuda")
    assert torch.cuda.default_generators[0].get_offset() == want_offset
    m = deferred_init(build)
    torch.manual_seed(SEED)
    materialize_module(m, rng="aten")
    engine = tensors(m)
    assert torch.cuda.default_generators[0].get_offset() == want_offset
    for k, t in want.items():
        assert same_bits(got[k], t), k
        assert same_bits(engine[k], t), k
    if case == "tiny_gpt2_fp32":
        assert got["lm_head.weight"] is got["transformer.wte.weight"]


def check_layout(plan, whole, steps_of, **kw):
    torch.manual_seed(SEED)
    got = plan.materialize(device="cuda", **kw)
    for k, t in whole.items():
        if k in got:
            assert same_bits(got[k], apply_steps(t, steps_of(k))), (k, steps_of(k), kw)


@pytest.mark.parametrize("case", ["layers_fp32_then_bf16", "tiny_llama_bf16", "llama_fp32_then_bf16", "init_zoo_fp32"])
def test_shards_are_chunks_of_the_whole(case, tmp_path):
    whole, _ = reference(*BUILDS[case])
    plan = saved_plan(BUILDS[case][0], tmp_path)
    params = {e.name for e in plan.entries if e.kind == "param"}
    for world in (2, 3, 8):
        for r in range(world):
            check_layout(plan, whole, lambda k: [(0, r, world)] if k in params and whole[k].dim() else [],
                         shard=(r, world))


@pytest.mark.parametrize("case", list(TP_PLANS))
def test_tp_placements_are_chunks_of_the_whole(case, tmp_path):
    build = lambda: cases.build(case, "fp32", "cuda")
    whole, _ = reference(build)
    plan = saved_plan(build, tmp_path)
    placements = tp_placements(deferred_init(build), TP_PLANS[case]())
    alias = {e.name: e.alias_of for e in plan.entries if e.source == "alias"}
    for world in (2, 3):
        for r in range(world):
            dim = lambda k: placements.get(alias.get(k, k))
            check_layout(plan, whole, lambda k: [] if dim(k) is None else [(dim(k), r, world)], shard=(r, world),
                         placements=placements)


def test_fsdp_tp_blocks_are_chunks_of_the_whole(tmp_path):
    build = lambda: built(MODELS["tiny_llama"][0], torch.float32, "cuda")
    whole, _ = reference(build)
    plan = saved_plan(build, tmp_path)
    alias = {e.name for e in plan.entries if e.source == "alias"}
    for blocks in fake_blocks("tiny_llama", MESHES["dp2_tp4"]):
        blocks = {k: v for k, v in blocks.items() if k not in alias}
        check_layout(plan, whole, lambda k: blocks.get(k, []), blocks=blocks)


def fields(d):
    """A descriptor's fields, its output address aside (and the parameters a source does not read: a
    constant's or a band's p0 / p1, a staged copy source's address)."""
    out = {name: getattr(d, name) for name, _ in C.TdxInitDesc._fields_ if name not in ("dst", "fill_bits", "epi")}
    out["fill_bits"] = tuple(d.fill_bits)
    out["epi"] = [(s.op, s.a, s.b) for s in d.epi[:d.n_epi]]
    if d.src in (C.TDX_SRC_CONST, C.TDX_SRC_BAND):
        del out["p0"], out["p1"]
    if d.src == C.TDX_SRC_GATHER:
        out["fill_bits"] = (0, d.fill_bits[1])
    return out


@pytest.mark.parametrize("case", ["layers_fp32_then_bf16", "tiny_llama_bf16", "llama_fp32_then_bf16", "state_space"])
def test_plan_descriptors_are_the_engines(case, tmp_path):
    """(Models whose every tensor the plan folds: a plan stores a replayed tensor by value, where the engine
    also writes the fusible storages it reads, such as init_zoo's `tril(ones).bool()` mask.)"""
    build = BUILDS[case][0]
    plan = saved_plan(build, tmp_path)
    p = torch.cuda.get_device_properties(0)
    props = (p.multi_processor_count, p.max_threads_per_multi_processor)
    drawn = 0
    for shard in (None, (0, 3), (2, 3), (5, 8)):
        m = deferred_init(build)
        torch.manual_seed(SEED)
        materialize_module(m, shard=shard, rng="aten")
        engine = [fields(d) for d in last_descriptors()]
        table, end = plan.descriptors(SEED, 0, shard, device_props=props)
        mine = [fields(d) for _, _, descs in table for d in descs]
        assert len(mine) == len(engine), (shard, len(mine), len(engine))
        for i, (a, b) in enumerate(zip(mine, engine)):
            assert a == b, (shard, i, {k: (a[k], b.get(k)) for k in a if a[k] != b.get(k)})
        assert end == torch.cuda.default_generators[0].get_offset()
        drawn += sum(d.algo in (C.TDX_ALGO_ATEN, C.TDX_ALGO_ATEN_WIDE) for d in last_descriptors())
    assert drawn > 0


# ------------------------------------------------------------------------------------ the hand-off
SENTINEL = 0x7F


def _handoff_worker(rank, shape, plan_path, outdir):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    torch.cuda.set_device(0)

    def one(mesh):
        fn, tp_plan = MODELS["llama_v11_h12"]
        with torch.device("meta"):
            m = fn()
        shard_2d(m, tp_plan(), mesh)
        m.to_empty(device="cuda")
        blocks = {k: local_block(p, k) for k, p in m.named_parameters()}
        local = lambda p: p.to_local() if hasattr(p, "to_local") else p
        # every byte of the storages FSDP2 and the buffers own, set to a sentinel
        storages = {}
        for p in list(m.parameters()) + list(m.buffers()):
            t = local(p).detach()
            s = t.untyped_storage()
            storages.setdefault(s.data_ptr(), [s, []])[1].append(
                (t.storage_offset() * t.element_size(), (t.storage_offset() + t.numel()) * t.element_size()))
        for s, _ in storages.values():
            torch.empty(0, dtype=torch.uint8, device="cuda").set_(s).fill_(SENTINEL)
        torch.manual_seed(SEED)
        init_sharded_module(m, InitPlan.load(plan_path))
        torch.cuda.synchronize()
        whole, _ = reference(lambda: built(fn, torch.float32, "cuda"))
        bad = [k for k, p in list(m.named_parameters()) + list(m.named_buffers())
               if not same_bits(local(p), apply_steps(whole[k], blocks.get(k, [])))]
        # bytes outside every local tensor: FSDP2's padding
        padding = touched = 0
        for s, ranges in storages.values():
            raw = torch.empty(0, dtype=torch.uint8, device="cuda").set_(s)
            outside = torch.ones(raw.numel(), dtype=torch.bool, device="cuda")
            for lo, hi in ranges:
                outside[lo:hi] = False
            padding += int(outside.sum())
            touched += int((raw[outside] != SENTINEL).sum())
        return dict(bad=bad, padding=padding, touched=touched,
                    two_d=sum(len({d for d, _, n in s if n > 1}) == 2 for s in blocks.values()))

    result = fake_rank(shape, rank, one, device_type="cuda")
    torch.save(result, os.path.join(outdir, f"rank{rank}.pt"))


def test_init_sharded_module_hands_off_atens_bits(tmp_path):
    """One process per coordinate of a dp2 x tp4 mesh, each one rank of the fake backend on CUDA: meta
    model -> parallelize_module -> fully_shard -> to_empty("cuda") -> init_sharded_module(model, aten plan)."""
    build = lambda: built(MODELS["llama_v11_h12"][0], torch.float32, "cuda")
    saved_plan(build, tmp_path)
    shape = MESHES["dp2_tp4"]
    mp.spawn(_handoff_worker, args=(shape, str(tmp_path / "p.json"), str(tmp_path)), nprocs=len(coordinates(shape)),
             join=True)
    padding = 0
    for r in coordinates(shape):
        res = torch.load(str(tmp_path / f"rank{r}.pt"))
        assert not res["bad"] and res["touched"] == 0 and res["two_d"] > 0, (r, res)
        padding += res["padding"]
    assert padding > 0  # (vocabulary 11 and hidden 12 over dp2 x tp4: FSDP2 pads uneven rows)
