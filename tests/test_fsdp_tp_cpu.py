"""FSDP2 over tensor parallelism without a GPU.

- Layouts against torch itself: eight gloo ranks build tiny Llama and OPT models eagerly (uneven sizes:
  vocab 11, hidden 12), run ``parallelize_module`` over the ``tp`` mesh dimension and ``fully_shard`` over
  ``dp`` (or HSDP's ``rep`` x ``dp``); on every rank and parameter, ``local_block`` applied to the eager
  tensor is ``to_local()``.
- Values through the host chain, per coordinate: the layouts come from a meta model handed to
  ``parallelize_module`` and ``fully_shard`` on one rank of the fake backend; the deferred recording
  goes through InitPlan -> JSON -> ``descriptors(blocks=...)`` -> the CPU restatement
  (oracle/tdx_oracle.c).  Every block is its chunk steps applied to the unsharded restatement, bit
  for bit, and the unsharded restatement is the eager constructor's tensor (constants bit-exact, draws
  T1); every rank advances the generator alike.
- The ValueErrors of ``local_block``, ``init_sharded_module`` and ``blocks=``, and the descriptors of the
  ``shard=`` / ``placements=`` calls, unchanged from the release before ``blocks=``."""
import ctypes
import hashlib
import os
import socket
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch import nn

from oracle import cases
from oracle import tdx_oracle as O
from torchdistx_b200.deferred_init import deferred_init
from torchdistx_b200.parallel import local_block, tp_placements
from torchdistx_b200.plan import InitPlan, chunk_steps, init_sharded_module, narrowed

from test_plan_oracle_cpu import OFFSET, SEED, check_t1, compare_with_eager, named, plan_of
from test_tp_shard_cpu import COPIES_ARGS, COPIES_PLAN, LLAMA_PLAN, OPT_PLAN, Copies, Geometry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MESHES = {"dp2_tp4": (2, 4), "dp4_tp2": (4, 2), "hsdp_2x2_tp2": (2, 2, 2)}


def small_llama():
    import transformers as T

    return T.LlamaForCausalLM(T.LlamaConfig(vocab_size=11, hidden_size=12, intermediate_size=20, num_hidden_layers=2,
                                            num_attention_heads=3, num_key_value_heads=1))


def small_opt():
    import transformers as T

    return T.OPTForCausalLM(T.OPTConfig(vocab_size=11, hidden_size=12, ffn_dim=20, num_hidden_layers=1,
                                        num_attention_heads=3, word_embed_proj_dim=12, max_position_embeddings=16,
                                        pad_token_id=1))


# name -> (constructor of the module at the default dtype and device, tensor-parallel plan)
MODELS = {"llama_v11_h12": (small_llama, LLAMA_PLAN), "opt_v11_h12": (small_opt, OPT_PLAN),
          "tiny_llama": (lambda: cases.CASES["tiny_llama"](), LLAMA_PLAN),
          "family_opt": (lambda: cases.families()["opt"](), OPT_PLAN)}


def built(fn, dtype=torch.float32, device="cpu"):
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        with torch.device(device):
            return fn()
    finally:
        torch.set_default_dtype(prev)


def coordinates(shape):
    n = 1
    for s in shape:
        n *= s
    return range(n)


def apply_steps(t, steps):
    """Chunk steps applied with torch.chunk itself (an index past the last chunk: no rows)."""
    for d, i, n in steps:
        chunks = torch.chunk(t, n, d)
        t = chunks[i] if i < len(chunks) else t.narrow(d, t.shape[d], 0)
    return t


def shard_2d(model, plan, mesh):
    """parallelize_module over the mesh's last dimension, then fully_shard over the others."""
    from torch.distributed.fsdp import fully_shard
    from torch.distributed.tensor.parallel import parallelize_module

    names = mesh.mesh_dim_names
    parallelize_module(model, mesh[names[-1]], plan)
    fully_shard(model, mesh=mesh[names[:-1]] if len(names) > 2 else mesh[names[0]])
    return model


def mesh_of(shape, device_type="cpu"):
    from torch.distributed.device_mesh import init_device_mesh

    return init_device_mesh(device_type, shape, mesh_dim_names=("rep", "dp", "tp")[-len(shape):])


def fake_rank(shape, rank, fn, device_type="cpu"):
    """`fn(mesh)` on rank `rank` of the fake backend (no communication), on a (dp, tp) or (rep, dp, tp) mesh."""
    from torch.testing._internal.distributed.fake_pg import FakeStore

    world = len(coordinates(shape))
    dist.init_process_group("fake", store=FakeStore(), rank=rank, world_size=world)
    try:
        return fn(mesh_of(shape, device_type))
    finally:
        dist.destroy_process_group()


def llama3_8b_meta():
    import transformers as T
    from test_tp_shard_gpu import LLAMA3_8B

    return T.LlamaForCausalLM(T.LlamaConfig(**LLAMA3_8B))


def _llama3_8b_plan():
    from test_tp_shard_gpu import LLAMA3_8B_PLAN

    return LLAMA3_8B_PLAN()


# every model whose layouts are read: (constructor, tensor-parallel plan)
LAYOUTS = {**MODELS, "copies": (lambda: Copies(*COPIES_ARGS()), COPIES_PLAN), "llama3_8b": (llama3_8b_meta, _llama3_8b_plan)}


def _layout_worker(i, shape, ranks, names, outdir):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

    def layouts(mesh):
        out = {}
        for name in names:
            fn, plan = LAYOUTS[name]
            with torch.device("meta"):
                m = fn()
            shard_2d(m, plan(), mesh)
            out[name] = {n: local_block(p, n) for n, p in m.named_parameters()}
        return out

    torch.save(fake_rank(shape, ranks[i], layouts), os.path.join(outdir, f"rank{ranks[i]}.pt"))


_layouts = {}


def fake_blocks(name, shape, ranks=None):
    """[{parameter name: local_block}] per rank of `ranks` (default: all): the model through
    parallelize_module and fully_shard on the meta device, in a fresh process per rank (one rank of the fake
    backend each: a process keeps meshes of an earlier process group)."""
    ranks = tuple(coordinates(shape) if ranks is None else ranks)
    key = (shape, ranks)
    if name not in _layouts.get(key, {}):
        names = [name] if name == "llama3_8b" else [n for n in LAYOUTS if n != "llama3_8b"]
        with tempfile.TemporaryDirectory() as d:
            mp.spawn(_layout_worker, args=(shape, ranks, names, d), nprocs=len(ranks), join=True)
            got = [torch.load(os.path.join(d, f"rank{r}.pt")) for r in ranks]
        _layouts.setdefault(key, {}).update({n: [g[n] for g in got] for n in names})
    return _layouts[key][name]


# --------------------------------------------------------------------------- layouts against torch
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    result = {}
    for mesh_name, shape in MESHES.items():
        mesh = mesh_of(shape)
        for case in ("llama_v11_h12", "opt_v11_h12"):
            fn, plan = MODELS[case]
            torch.manual_seed(SEED)  # (every rank: the same eager tensors)
            m = fn()
            whole = {k: v.detach().clone() for k, v in m.named_parameters(remove_duplicate=False)}
            shard_2d(m, plan(), mesh)
            rows = []
            for k, p in m.named_parameters():
                steps = local_block(p, k)
                local = p.to_local()
                want = apply_steps(whole[k], steps)
                rows.append((k, [type(pl).__name__ for pl in p.placements], steps, tuple(local.shape),
                             want.shape == local.shape and torch.equal(want, local)))
            result[(mesh_name, case)] = rows
    torch.save(result, os.path.join(outdir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_local_blocks_are_what_parallelize_module_and_fully_shard_hold_on_eight_gloo_ranks(tmp_path):
    mp.spawn(_worker, args=(8, _free_port(), str(tmp_path)), nprocs=8, join=True)
    empty = one_row = strided = 0
    for rank in range(8):
        for key, rows in torch.load(str(tmp_path / f"rank{rank}.pt")).items():
            for name, placements, steps, shape, ok in rows:
                assert ok, (rank, key, name, placements, steps, shape)
                empty += shape[0] == 0
                one_row += shape[0] == 1
                strided += "_StridedShard" in placements
    assert empty and one_row and strided, (empty, one_row, strided)


# ------------------------------------------------------------------------------- the host chain
def layouts_per_rank(case, shape, plan):
    """[{entry name: chunk steps}] per rank, tied names the plan lists as an alias left out (the tensor is
    built under its first name)."""
    alias = {e.name for e in plan.entries if e.source == "alias"}
    return [{k: v for k, v in b.items() if k not in alias} for b in fake_blocks(case, shape)]


def check_coordinates(plan, per_rank, whole, end, own=None):
    """Every rank's blocks are its chunk steps of the unsharded restatement, bit for bit; T1 against the
    eager block for single-source draws.  Returns the number of windowed descriptors."""
    windows = 0
    entries = {e.name: e for e in plan.entries}
    for blocks in per_rank:
        got, e_end, w = O.evaluate_plan(plan, SEED, OFFSET, blocks=blocks)
        assert e_end == end  # (global sizes only: every rank advances the generator alike)
        windows += w
        for name, steps in blocks.items():
            want = apply_steps(whole[name], steps)
            assert got[name].shape == want.shape and torch.equal(
                got[name].reshape(-1).view(torch.uint8), want.contiguous().reshape(-1).view(torch.uint8)), (name, steps)
            e = entries[name]
            if own is not None and e.source in ("uniform", "normal") and not e.segments and not e.epilogue:
                sixteen = got[name].dtype in (torch.bfloat16, torch.float16)
                check_t1(f"{name}{steps}", got[name], apply_steps(own[name].detach(), steps), sixteen)
    return windows


@pytest.mark.parametrize("case", ["llama_v11_h12", "opt_v11_h12", "tiny_llama", "family_opt"])
@pytest.mark.parametrize("mesh", list(MESHES))
def test_blocks_through_the_host_chain_per_coordinate(case, mesh, tmp_path):
    fn = MODELS[case][0]
    plan = InitPlan.from_module(deferred_init(lambda: built(fn)))
    plan.save(str(tmp_path / "p.json"))
    plan = InitPlan.load(str(tmp_path / "p.json"))
    whole, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    torch.manual_seed(SEED)
    own = named(built(fn))
    compare_with_eager(plan, whole, own, own)  # the unsharded restatement is the eager model
    per_rank = layouts_per_rank(case, MESHES[mesh], plan)
    dp, tp = MESHES[mesh][-2:]
    assert len({repr(b) for b in per_rank}) == dp * tp  # (every (dp, tp) coordinate its own layout; HSDP's replicas alike)
    assert check_coordinates(plan, per_rank, whole, end, own) > 0  # (dim-0 rows x a Shard(1) range: windows)
    if case.startswith("opt"):  # the padding row: a constant run inside every rank's window
        (e,) = [e for e in plan.entries if e.name == "model.decoder.embed_tokens.weight"]
        assert [g["source"] for g in e.segment_list()] == ["normal", "const", "normal"]
        assert any(len(b[e.name]) == 2 and b[e.name][0][0] == 0 and b[e.name][1][0] == 1 for b in per_rank)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_three_dims_and_dim_0_rows_of_every_window(dtype, tmp_path):
    torch.manual_seed(0)
    plan = InitPlan.from_module(deferred_init(lambda: Geometry().to(dtype)))
    plan.save(str(tmp_path / "p.json"))
    plan = InitPlan.load(str(tmp_path / "p.json"))
    whole, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    for dp, tp in ((2, 4), (3, 2), (4, 3)):
        per_rank = [{"w3": [(0, d, dp), (2, t, tp)], "u": [(0, d, dp), (1, t, tp)], "tn": [(0, t, tp), (0, d, dp)]}
                    for d in range(dp) for t in range(tp)]
        assert check_coordinates(plan, per_rank, whole, end) > 0


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_copy_programs_are_built_whole_and_narrowed_on_both_dims(dtype):
    args = COPIES_ARGS()  # (real tensors: built outside the recording)
    fn = lambda: Copies(*args, cases.DTYPES[dtype])
    torch.manual_seed(0)
    plan = InitPlan.from_module(deferred_init(fn))
    whole, end, _ = O.evaluate_plan(plan, SEED, OFFSET)
    torch.manual_seed(0)
    eager_model = fn()
    for k in ("pos.weight", "lin.weight"):  # (copies: bit for bit)
        assert torch.equal(whole[k], dict(eager_model.named_parameters())[k].detach()), k
    entries = {e.name: e for e in plan.entries}
    for shape in MESHES.values():
        per_rank = fake_blocks("copies", shape)
        assert any(narrowed(entries["pos.weight"], steps=b["pos.weight"]) and b["pos.weight"][0][0] == 0
                   for b in per_rank)
        check_coordinates(plan, per_rank, whole, end)


# ----------------------------------------------------------------------------------- errors
def test_local_block_value_errors():
    from torch.distributed.tensor import DTensor, Partial, Replicate, Shard
    from torch.distributed.tensor.placement_types import _StridedShard

    def check(mesh):
        z = lambda *s: torch.zeros(*s)
        dt = lambda local, pl, **kw: nn.Parameter(DTensor.from_local(local, mesh, pl, run_check=False, **kw))
        assert local_block(z(3, 5), "plain") == []
        assert local_block(dt(z(2, 3), [Replicate(), Shard(0)]), "w") == [(0, 1, 4)]  # (rank 5: coordinate (1, 1))
        assert local_block(dt(z(2, 3), [_StridedShard(0, split_factor=4), Shard(0)]), "w") == [(0, 1, 4), (0, 1, 2)]
        with pytest.raises(ValueError, match=r"'p' with placements \(Partial\(sum\), Shard\(dim=0\)\).*Partial"):
            local_block(dt(z(2, 3), [Partial(), Shard(0)]), "p")
        with pytest.raises(ValueError, match="'s'.*_StridedShard is supported only"):
            local_block(dt(z(2, 3), [_StridedShard(0, split_factor=3), Shard(0)]), "s")
        with pytest.raises(ValueError, match="'s'.*_StridedShard is supported only"):
            local_block(dt(z(2, 3), [_StridedShard(1, split_factor=4), Shard(0)]), "s")
        with pytest.raises(ValueError, match="'b'.*restricts more than dim 0 and one other dimension"):
            local_block(dt(z(2, 3, 4), [Shard(1), Shard(2)]), "b")
        with pytest.raises(ValueError, match="'t'.*not contiguous"):
            local_block(dt(z(3, 2).t(), [Shard(0), Replicate()]), "t")

    fake_rank((2, 4), 5, check)


def _handed_off(fn, plan):
    """`go(mesh)`: a meta model through parallelize_module and fully_shard, to_empty on the CPU."""
    def go(mesh):
        with torch.device("meta"):
            m = fn()
        shard_2d(m, plan, mesh)
        return m.to_empty(device="cpu")

    return go


def test_init_sharded_module_value_errors():
    from torch.distributed.tensor import DTensor, Replicate, Shard

    plan = InitPlan.from_module(deferred_init(small_llama))

    def check(mesh):
        m = _handed_off(small_llama, LLAMA_PLAN())(mesh)
        with pytest.raises(ValueError, match="give both `rank` and `world`"):
            init_sharded_module(m, plan, rank=0)
        short = InitPlan([e for e in plan.entries if e.name != "model.norm.weight"])
        with pytest.raises(ValueError, match="'model.norm.weight' is not in the plan"):
            init_sharded_module(m, short)
        other = InitPlan.from_module(deferred_init(lambda: built(small_llama, torch.bfloat16)))
        with pytest.raises(ValueError, match=r"is torch.float32 \[.*\] in the module and torch.bfloat16"):
            init_sharded_module(m, other)
        import transformers as T

        wider = InitPlan.from_module(deferred_init(lambda: T.LlamaForCausalLM(T.LlamaConfig(
            vocab_size=13, hidden_size=12, intermediate_size=20, num_hidden_layers=2, num_attention_heads=3,
            num_key_value_heads=1))))
        with pytest.raises(ValueError, match=r"'model.embed_tokens.weight' is torch.float32 \[11, 12\] in the module "
                                             r"and torch.float32 \[13, 12\] in the plan"):
            init_sharded_module(m, wider)
        # a local tensor smaller than its block: global (8, 4) as Shard(0) over dp and Replicate over tp
        # is 4 rows on rank 5, the local tensor 3
        lin = nn.Linear(4, 8, bias=False)
        lin.weight = nn.Parameter(DTensor.from_local(torch.zeros(3, 4), mesh, [Shard(0), Replicate()], run_check=False,
                                                     shape=torch.Size([8, 4]), stride=(4, 1)))
        with pytest.raises(ValueError, match=r"'weight': the local tensor holds 12 elements, its block \[\(4, 8\), "
                                             r"\(0, 4\)\] has 16"):
            init_sharded_module(lin, InitPlan.from_module(deferred_init(lambda: nn.Linear(4, 8, bias=False))))
        # OPT ties lm_head to the embedding; parallelize_module gives the embedding a new Parameter
        opt = _handed_off(small_opt, OPT_PLAN())(mesh)
        with pytest.raises(ValueError, match="'model.decoder.embed_tokens.weight' and 'lm_head.weight' are one tied "
                                             "parameter in the plan, but the module lays them out differently"):
            init_sharded_module(opt, InitPlan.from_module(deferred_init(small_opt)))

    fake_rank((2, 4), 5, check)


def test_blocks_value_errors():
    torch.manual_seed(0)
    plan = InitPlan.from_module(deferred_init(Geometry))
    with pytest.raises(ValueError, match=r"'w3': the block \[\(0, 3\), \(0, 5\), \(0, 7\)\] restricts more than "
                                         "dim 0 and one other dimension"):
        plan.descriptors(SEED, OFFSET, blocks={"w3": [(1, 0, 2), (2, 0, 2)]})
    with pytest.raises(ValueError, match="give either `blocks` or `shard` / `placements`"):
        plan.descriptors(SEED, OFFSET, shard=(0, 2), blocks={"w3": [(0, 0, 2)]})


# ----------------------------------------------------------------------------- compatibility
# sha256 over every rank's descriptor table (entry names, sizes, the 128-byte descriptors, the generator
# offset after) of tiny Llama in fp32 from (SEED, OFFSET), as the release before `blocks=` computed them:
# placements= the Colwise / Rowwise plan, and shard= (rank, world)
PARENT = {
    ("tp", 2): "0cae5a4fd0b3ea3b6f11354763c94d6a445970e8c84f123e24e980b8158ec61d",
    ("tp", 3): "90fe9c417aa713ad1aaed35f84c77141323df8b144b3147e58e3eceeb4592020",
    ("tp", 8): "a91dc36f2ecef05d2447591545f39605b2da530ce7dd10e33b91eb25e13ac332",
    ("shard", 2): "28136989169ef6a45321dae6cbf02fd1fa354d4d27346f55d14a5acc21cc6093",
    ("shard", 3): "623570add19c6375f9cd3dce82106912fa7962fba0016816339d60e96bacc66b",
    ("shard", 8): "6239781aee9e9d6bae2daf9d25fcfcf92c2e7730ee2b44dd60a710546d68b0b1",
}


def _table_bytes(table, end):
    out = [repr(end).encode()]
    for e, sizes, descs in table:
        out.append(repr((e.name, list(sizes))).encode())
        out += [ctypes.string_at(ctypes.addressof(d), ctypes.sizeof(d)) for d in descs]
    return b"".join(out)


@pytest.mark.parametrize("mode,world", [(m, w) for m in ("tp", "shard") for w in (2, 3, 8)])
def test_shard_and_placements_descriptors_are_unchanged(mode, world):
    plan = plan_of("tiny_llama", "fp32")
    placements = tp_placements(deferred_init(lambda: cases.build("tiny_llama", "fp32")), LLAMA_PLAN())
    kw = dict(placements=placements) if mode == "tp" else {}
    h = hashlib.sha256()
    for r in range(world):
        table = _table_bytes(*plan.descriptors(SEED, OFFSET, (r, world), **kw))
        h.update(table)
        # the same layout given as chunk steps is the same table
        blocks = {e.name: chunk_steps(e, (r, world), placements.get(e.name) if mode == "tp" else 0)
                  for e in plan.entries}
        assert _table_bytes(*plan.descriptors(SEED, OFFSET, blocks=blocks)) == table, r
    assert h.hexdigest() == PARENT[(mode, world)]
