"""Tensor-parallel blocks without a GPU: tiny Llama and OPT recordings through InitPlan -> JSON ->
descriptors(placements) -> the CPU restatement of windowed descriptors (oracle/tdx_oracle.c).  Every
rank's Shard(d) block is the rank's torch.chunk of the unsharded restatement, bit for bit, and the
unsharded restatement is the eager constructor's tensor (constants bit-exact, draws T1); the generator
advances the same on every rank.  Also: tp_placements against what parallelize_module does on two gloo
ranks (and materialize_module(parallelize_plan=...) there, by ATen replay), the ValueError cases and the
library's validation of windowed descriptors."""
import os
import socket
import sys
import types

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from torch import nn
from torch.distributed.tensor.parallel import (ColwiseParallel, PrepareModuleInput, RowwiseParallel,
                                               SequenceParallel)

from oracle import cases
from oracle import tdx_oracle as O
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, materialize_module
from torchdistx_b200.parallel import tp_placements
from torchdistx_b200.plan import InitPlan, narrowed

from test_plan_oracle_cpu import OFFSET, SEED, compare_with_eager, eager, plan_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LLAMA_PLAN = lambda: {
    "model.embed_tokens": ColwiseParallel(),
    "model.layers.*.self_attn.q_proj": ColwiseParallel(),
    "model.layers.*.self_attn.k_proj": ColwiseParallel(),
    "model.layers.*.self_attn.v_proj": ColwiseParallel(),
    "model.layers.*.self_attn.o_proj": RowwiseParallel(),
    "model.layers.*.mlp.gate_proj": ColwiseParallel(),
    "model.layers.*.mlp.up_proj": ColwiseParallel(),
    "model.layers.*.mlp.down_proj": RowwiseParallel(),
    "lm_head": ColwiseParallel(),
}
OPT_PLAN = lambda: {  # (OPT's embedding has a padding row: a constant run inside every rank's block)
    "model.decoder.embed_tokens": ColwiseParallel(),
    "model.decoder.layers.*.self_attn.[qkv]_proj": ColwiseParallel(),
    "model.decoder.layers.*.self_attn.out_proj": RowwiseParallel(),
    "model.decoder.layers.*.fc1": ColwiseParallel(),
    "model.decoder.layers.*.fc2": RowwiseParallel(),
}
MODELS = {"tiny_llama": LLAMA_PLAN, "family_opt": OPT_PLAN}

def block(whole, world, rank, dim):
    """Rank `rank`'s torch.chunk(whole, world, dim) (empty for trailing ranks without rows)."""
    if dim is None:
        return whole
    per = -(-whole.shape[dim] // world)
    start = min(whole.shape[dim], rank * per)
    return whole.narrow(dim, start, min(per, whole.shape[dim] - start))


def check_blocks(plan, placements, whole, end, worlds=(2, 3, 8)):
    n_windows = 0
    tied = {e.name: e.alias_of for e in plan.entries if e.source == "alias"}  # (one tensor, its first name's layout)
    for world in worlds:
        parts = [O.evaluate_plan(plan, SEED, OFFSET, shard=(r, world), placements=placements) for r in range(world)]
        for r, (got, e_end, windows) in enumerate(parts):
            assert e_end == end  # every rank advances its generator identically
            n_windows += windows
            for name, t in whole.items():
                want = block(t, world, r, placements.get(tied.get(name, name)))
                assert got[name].shape == want.shape and torch.equal(
                    got[name].reshape(-1).view(torch.uint8), want.contiguous().reshape(-1).view(torch.uint8)), \
                    (name, world, r)
        for name, dim in placements.items():  # the blocks concatenate along d to the whole
            if dim is not None:
                cat = torch.cat([p[0][name] for p in parts], dim)
                assert torch.equal(cat.view(torch.uint8), whole[name].view(torch.uint8)), (name, world)
    return n_windows


@pytest.mark.parametrize("case", list(MODELS))
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_tp_blocks_are_chunks_of_the_eager_model(case, dtype, tmp_path):
    plan = plan_of(case, dtype, tmp_path)  # (through the JSON file)
    placements = tp_placements(deferred_init(lambda: cases.build(case, dtype)), MODELS[case]())
    assert {d for d in placements.values()} == {0, 1, None} if case == "family_opt" else {0, 1}
    whole, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    own, wide = eager(case, dtype)
    compare_with_eager(plan, whole, own, wide)  # the unsharded restatement is the eager model
    assert check_blocks(plan, placements, whole, end) > 0  # (Rowwise weights: windowed descriptors)


class Geometry(nn.Module):
    """A 3-D parameter with a constant row in the middle (Shard(1) and Shard(2): unaligned W, ragged and
    empty trailing ranks), a uniform and a truncated normal (an epilogue)."""

    def __init__(self):
        super().__init__()
        self.w3 = nn.Parameter(torch.empty(3, 10, 13))
        self.u = nn.Parameter(torch.empty(6, 21))
        self.tn = nn.Parameter(torch.empty(5, 40))
        nn.init.normal_(self.w3, 0.0, 0.5)
        nn.init.uniform_(self.u, -1.0, 1.0)
        nn.init.trunc_normal_(self.tn, std=0.02)
        with torch.no_grad():
            self.w3[1, 4].zero_()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("placements", [{"w3": 1, "u": 1, "tn": 1}, {"w3": 2, "u": 0, "tn": None}])
def test_three_dims_unaligned_ragged_and_empty_ranks(dtype, placements, tmp_path):
    torch.manual_seed(0)
    plan = InitPlan.from_module(deferred_init(lambda: Geometry().to(dtype)))
    plan.save(str(tmp_path / "p.json"))
    plan = InitPlan.load(str(tmp_path / "p.json"))
    whole, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    check_blocks(plan, placements, whole, end, worlds=(2, 3, 4, 8))


class Copies(nn.Module):
    """Weights built from host tensors (copy programs: no windowed descriptor), one of them a
    sinusoid table in an nn.Embedding (Marian's idiom), planned with Shard(1)."""

    def __init__(self, table, grid, dtype=torch.float32):
        super().__init__()
        self.pos = nn.Embedding(*table.shape, dtype=dtype)
        self.lin = nn.Linear(grid.shape[1], grid.shape[0], dtype=dtype)
        with torch.no_grad():
            self.pos.weight.copy_(table)
            self.lin.weight.copy_(grid)


COPIES_PLAN = lambda: {"pos": ColwiseParallel(), "lin": RowwiseParallel()}
COPIES_ARGS = lambda: (torch.from_numpy(np.random.default_rng(0).normal(size=(50, 24))),
                       torch.arange(6 * 10, dtype=torch.float64).reshape(6, 10) / 7)


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_copy_programs_under_shard_1_are_built_whole_and_narrowed(dtype):
    args = COPIES_ARGS()  # (real tensors: built outside the recording)
    build = lambda: Copies(*args, cases.DTYPES[dtype])
    torch.manual_seed(0)
    plan = InitPlan.from_module(deferred_init(build))
    placements = tp_placements(deferred_init(build), COPIES_PLAN())
    assert placements == {"pos.weight": 1, "lin.weight": 1, "lin.bias": None}
    entries = {e.name: e for e in plan.entries}
    assert all(narrowed(entries[k], (0, 3), 1) for k in ("pos.weight", "lin.weight"))
    whole, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    torch.manual_seed(0)
    eager_model = build()
    for k in ("pos.weight", "lin.weight"):  # (copies: bit for bit)
        assert torch.equal(whole[k], dict(eager_model.named_parameters())[k].detach()), k
    check_blocks(plan, placements, whole, end, worlds=(2, 3, 8))
    # one rank, or no shard at all: the layout changes nothing (and nothing is narrowed)
    for shard in (None, (0, 1)):
        got, e_end, _ = O.evaluate_plan(plan, SEED, OFFSET, shard=shard, placements=placements)
        assert e_end == end and all(torch.equal(got[k], whole[k]) for k in whole), shard


def test_descriptors_of_a_padded_embedding_under_shard_1():
    plan = plan_of("family_opt", "fp32")
    (entry,) = [e for e in plan.entries if e.name == "model.decoder.embed_tokens.weight"]
    assert [g["source"] for g in entry.segment_list()] == ["normal", "const", "normal"]  # padding_idx = 1
    table, _ = plan.descriptors(SEED, OFFSET, (1, 3), placements={entry.name: 1})
    (descs,) = [d for e, _, d in table if e is entry]
    # rows [0, 1) and [2, 512) of columns [22, 44): two windowed draws around one fill of the padding row
    kinds = [(d.src, bool(d.reserved & C.TDX_FLAG_WINDOW), int(d.elem_count)) for d in descs]
    assert kinds == [(C.TDX_SRC_NORMAL, False, 22), (C.TDX_SRC_CONST, False, 22), (C.TDX_SRC_NORMAL, True, 510 * 22)]
    assert list(descs[2].fill_bits) == [22, 64] and descs[2].elem_begin == 2 * 64 + 22


def test_library_validates_the_windowed_descriptor():
    good = dict(dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=64, elem_begin=8, p1=0.02)

    def win(w, p, **kw):
        d = C.make_desc(1 << 21, **dict(good, **kw))
        d.reserved |= C.TDX_FLAG_WINDOW
        d.fill_bits[0], d.fill_bits[1] = w, p
        return d

    for ok in (win(16, 48), win(16, 16), win(5, 7), win(16, 48, algo=C.TDX_ALGO_WIDE32),
               win(16, 48, src=C.TDX_SRC_UNIFORM, epi=[(C.TDX_EPI_EXP, 0.0)])):
        assert C.prepare([ok]) > 0
    bad = [win(0, 48), win(16, 15),  # W == 0, P < W
           win(16, 48, src=C.TDX_SRC_CONST, dtype=C.TDX_RAW16, fill_itemsize=2), win(16, 48, src=C.TDX_SRC_IOTA, dtype=C.TDX_F32),
           win(16, 1 << 62, elem_count=16 * 5)]  # the last run starts beyond 2^64
    for d in bad:
        with pytest.raises(RuntimeError, match="TDX_FLAG_WINDOW"):
            C.prepare([d])


def test_value_errors():
    mesh = types.SimpleNamespace(ndim=1, device_type="cpu")
    m = deferred_init(lambda: cases.build("tiny_llama", "fp32"))
    with pytest.raises(ValueError, match="1-D `device_mesh`"):
        materialize_module(m, device_mesh=types.SimpleNamespace(ndim=2), parallelize_plan=LLAMA_PLAN())
    with pytest.raises(ValueError, match="either `shard` or `parallelize_plan`"):
        materialize_module(m, shard=(0, 2), device_mesh=mesh, parallelize_plan=LLAMA_PLAN())
    with pytest.raises(ValueError, match="'model.norm' is a LlamaRMSNorm"):
        materialize_module(m, device_mesh=mesh, parallelize_plan={"model.norm": ColwiseParallel()})
    with pytest.raises(ValueError, match="'lm_head' has style PrepareModuleInput"):
        materialize_module(m, device_mesh=mesh, parallelize_plan={"lm_head": PrepareModuleInput()})

    def strided():
        lin = nn.Linear(4, 8)
        lin.weight = nn.Parameter(torch.empty(4, 8).t())
        return nn.Sequential(lin)

    with pytest.raises(ValueError, match="'0.weight' is not contiguous"):
        materialize_module(deferred_init(strided), device_mesh=mesh, parallelize_plan={"0": RowwiseParallel()})
    # a tied parameter whose names the plan lays out differently
    tied = lambda: cases.build("tiny_llama", "fp32").__class__(
        __import__("transformers").LlamaConfig(vocab_size=512, hidden_size=64, intermediate_size=128,
                                              num_hidden_layers=1, num_attention_heads=4, tie_word_embeddings=True))
    with pytest.raises(ValueError, match="'model.embed_tokens.weight' and 'lm_head.weight' are one tied parameter"):
        materialize_module(deferred_init(tied), device_mesh=mesh,
                           parallelize_plan={"model.embed_tokens": ColwiseParallel(), "lm_head": ColwiseParallel()})
    # SequenceParallel replicates every parameter of any module
    assert tp_placements(m, {"model.norm": SequenceParallel()}) == {"model.norm.weight": None}


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _placements_of(model):
    from torch.distributed.tensor import DTensor, Shard

    out = {}
    for name, p in model.named_parameters():
        if isinstance(p.data, DTensor):
            (pl,) = p.placements
            out[name] = pl.dim if isinstance(pl, Shard) else None
    return out


def _worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor.parallel import parallelize_module

    dist.init_process_group("gloo", rank=rank, world_size=world)
    mesh = init_device_mesh("cpu", (world,))
    result = {}
    for case, plan in MODELS.items():
        ref = cases.build(case, "fp32")  # eager: the layouts parallelize_module gives
        parallelize_module(ref, mesh, plan())
        torch.manual_seed(SEED)  # the unsharded materialisation (on the CPU: ATen replay, chunked after)
        full = deferred_init(lambda: cases.build(case, "fp32"))
        materialize_module(full)
        whole = {k: v.detach().clone() for k, v in full.named_parameters()}
        torch.manual_seed(SEED)
        m = deferred_init(lambda: cases.build(case, "fp32"))
        materialize_module(m, device_mesh=mesh, parallelize_plan=plan())
        locals_before = {k: (p.to_local() if hasattr(p, "to_local") else p).detach().clone() for k, p in m.named_parameters()}
        mine = _placements_of(m)
        shapes = {k: tuple(p.shape) for k, p in m.named_parameters()} == {k: tuple(v.shape) for k, v in whole.items()}
        parallelize_module(m, mesh, plan())  # passes the built model through unchanged
        after = {k: (p.to_local() if hasattr(p, "to_local") else p).detach() for k, p in m.named_parameters()}
        result[case] = dict(torch=_placements_of(ref), mine=mine, after=_placements_of(m),
                            unchanged=all(torch.equal(locals_before[k], after[k]) for k in locals_before),
                            blocks=all(torch.equal(locals_before[k], block(whole[k], world, rank, mine.get(k)))
                                       for k in locals_before),
                            shapes=shapes)
    torch.save(result, os.path.join(outdir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_placements_and_blocks_match_parallelize_module_on_two_gloo_ranks(tmp_path):
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    for rank in range(2):
        res = torch.load(str(tmp_path / f"rank{rank}.pt"))
        for case, plan in MODELS.items():
            r = res[case]
            want = tp_placements(deferred_init(lambda: cases.build(case, "fp32")), plan())
            # (OPT ties lm_head to the embedding; parallelize_module replaces the embedding's Parameter
            # and leaves the tied name to the old object, a plain tensor in the eager model)
            after = {k: v for k, v in r["after"].items() if k in r["torch"]}
            assert r["torch"] == want == r["mine"] == after, (case, r["torch"], want)
            assert r["unchanged"] and r["blocks"] and r["shapes"], (case, rank, r)
