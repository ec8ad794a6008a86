"""Plans for ATen's own CUDA stream (`InitPlan.from_module(..., rng="aten")`) without a GPU.

- The file: version 7 with `"rng": "aten"`, a JSON round trip, and default plans unchanged.
- The draw dtype: a model built in fp32 and cast to bf16 draws every cast parameter on fp32
  (`aten_wide`), which the default stream's `wide` does not record.
- The descriptor table, `descriptors(..., device_props=(132, 2048))`, evaluated with the C restatement of
  ATen's stream (oracle/tdx_oracle.c). It must equal the restatement of each whole draw, cut to
  every rank's block, under `shard=`, tensor-parallel `placements=` and FSDP2 x TP `blocks=`. The generator
  must end at the sum of ATen's increments.
- Refusals: random programs ATen's stream cannot take, and a table asked for without device properties."""
import json

import numpy as np
import pytest
import torch
from torch import nn

from oracle import cases
from oracle import tdx_oracle as O
from torchdistx_b200 import _C
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init
from torchdistx_b200.parallel import tp_placements
from torchdistx_b200.plan import FORMAT_ATEN, InitPlan, chunk_steps, narrowed

from test_aten_stream_cpu import policy
from test_fsdp_tp_cpu import MESHES, apply_steps, fake_blocks
from test_tp_shard_cpu import MODELS as TP_PLANS

H100 = (132, 2048)  # (multiprocessor count, max threads per multiprocessor)
SEED, OFFSET = 1234, 40
ROUND_TRIP = [("tiny_llama", "bf16"), ("tiny_llama", "fp32"), ("init_zoo", "fp32"), ("tiny_gpt2", "fp32"),
              ("padded_embeddings", "bf16"), ("clones", "fp32"), ("cast_variant", "fp32"), ("torch_transformer", "fp32"),
              ("family_opt", "fp32")]


def record(case, dtype):
    return deferred_init(lambda: cases.build(case, dtype))


def drawn(g):
    return g["source"] in ("uniform", "normal")


# ------------------------------------------------------------------------------------------- the file
@pytest.mark.parametrize("case,dtype", ROUND_TRIP)
def test_aten_plans_are_version_7_and_default_plans_are_unchanged(case, dtype, tmp_path):
    aten = InitPlan.from_module(record(case, dtype), rng="aten")
    fused = InitPlan.from_module(record(case, dtype))
    assert (aten.rng, fused.rng) == ("aten", "fused")
    aten.save(str(tmp_path / "a.json"))
    fused.save(str(tmp_path / "f.json"))
    doc, fdoc = json.load(open(tmp_path / "a.json")), json.load(open(tmp_path / "f.json"))
    assert (doc["format"], doc["rng"]) == (FORMAT_ATEN, "aten")
    assert set(fdoc) == {"format", "entries"} and fdoc["format"] != FORMAT_ATEN
    assert "aten_wide" not in (tmp_path / "f.json").read_text()
    again = InitPlan.load(str(tmp_path / "a.json"))
    assert again.rng == "aten" and [e.__dict__ for e in again.entries] == [e.__dict__ for e in aten.entries]
    assert InitPlan.load(str(tmp_path / "f.json")).rng == "fused"
    # the aten plan is the default plan plus the draw dtype, every entry with a draw listed as segments
    assert len(aten.entries) == len(fused.entries)
    for a, f in zip(fields(aten), fields(fused)):
        segs = [{k: v for k, v in g.items() if k != "aten_wide"} for g in a.pop("segments")]
        assert segs == f.pop("segments") and a == f, a["name"]
    for a in aten.entries:
        for g in a.segment_list():
            assert ("aten_wide" in g) == drawn(g), (a.name, g["source"])
        if any(drawn(g) for g in a.segment_list()):
            assert a.segments, a.name


def fields(plan):
    """The entries as dicts: segments listed, and RNG pass ids numbered in order of appearance (they name
    the recording, which differs between two recordings of one constructor)."""
    ids, out = {}, []
    for e in plan.entries:
        d = dict(e.__dict__, segments=e.segment_list())
        d["rng_ids"] = [ids.setdefault(i, len(ids)) for i in e.rng_ids]
        out.append(d)
    return out


def test_load_checks_the_stream_against_the_version(tmp_path):
    plan = InitPlan.from_module(record("init_zoo", "fp32"), rng="aten")
    plan.save(str(tmp_path / "a.json"))
    doc = json.load(open(tmp_path / "a.json"))
    for bad in ({**doc, "rng": "fused"}, {k: v for k, v in doc.items() if k != "rng"},
                {**doc, "format": "torchdistx_b200.InitPlan/6"}, {**doc, "format": "torchdistx_b200.InitPlan/8"}):
        (tmp_path / "b.json").write_text(json.dumps(bad))
        with pytest.raises(ValueError):
            InitPlan.load(str(tmp_path / "b.json"))
    with pytest.raises(ValueError, match="rng"):
        InitPlan.from_module(record("linear128", "fp32"), rng="ATen")


def test_plan_info_default_is_unchanged_and_aten_adds_its_verdict():
    m = record("cast_variant", "fp32")
    for name, t in list(m.named_parameters()) + list(m.named_buffers()):
        default, fused, aten = _C.plan_info(t), _C.plan_info(t, "fused"), _C.plan_info(t, rng="aten")
        assert "aten_refusal" not in default and all("aten_wide" not in g for g in default["segments"])
        strip = lambda d: {k: v for k, v in d.items() if k != "segments"}
        assert strip(default) == strip(fused) and default["segments"] == fused["segments"], name
        assert aten["aten_refusal"] == "" and {**strip(aten), "aten_refusal": None} == {**strip(default), "aten_refusal": None}
        for g, h in zip(aten["segments"], default["segments"]):
            assert {k: v for k, v in g.items() if k != "aten_wide"} == h, name
    with pytest.raises(ValueError, match="rng"):
        _C.plan_info(m.a, rng="philox")


def fp32_then_bf16():
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float32)
    try:
        return cases.tiny_llama().to(torch.bfloat16)
    finally:
        torch.set_default_dtype(prev)


def test_a_llama_cast_to_bf16_draws_on_fp32():
    aten = {e.name: e for e in InitPlan.from_module(deferred_init(fp32_then_bf16), rng="aten").entries}
    fused = {e.name: e for e in InitPlan.from_module(deferred_init(fp32_then_bf16)).entries}
    n = 0
    for name, e in aten.items():
        if e.dtype != "BFloat16" or e.source in ("alias", "value"):
            continue
        for g in e.segment_list():
            if drawn(g):
                assert g["aten_wide"], name
                n += 1
        assert not fused[name].wide and not any(g["wide"] for g in fused[name].segment_list()), name
    assert n >= 2 * 7 + 1  # seven linears per layer and the embedding, all drawn on fp32


# ------------------------------------------------------------------------------ the descriptor table
class Programs:
    """Numbers the draw programs (source, parameters, epilogue, algo) a block's elements come from."""

    def __init__(self):
        self.ids = {}

    def __call__(self, src, p0, p1, epi, algo):
        key = (src, float(p0), float(p1), tuple(tuple(float(x) for x in s) for s in epi), algo)
        return self.ids.setdefault(key, len(self.ids))


def table_of(plan, steps_of, programs, **kw):
    """{name: (values, program ids)} of what the descriptor table writes, by the restatement (NaN / -1: an
    element no draw writes, -2: no descriptor), and the generator offset after it."""
    table, end = plan.descriptors(SEED, OFFSET, device_props=H100, **kw)
    out = {}
    for e, sizes, descs in table:
        if e.source in ("alias", "value"):
            continue
        numel = int(np.prod(sizes)) if sizes else 1
        isz = torch.empty((), dtype=getattr(torch, {"Float": "float32", "BFloat16": "bfloat16", "Half": "float16",
                                                  "Long": "int64", "Bool": "bool"}.get(e.dtype, "float32"))).element_size()
        vals, ids = np.full(numel, np.nan, dtype=np.float32), np.full(numel, -2, dtype=np.int64)
        for d in descs:
            at = int(d.dst or 0) // isz
            n = int(d.elem_count)
            if d.src in (C.TDX_SRC_UNIFORM, C.TDX_SRC_NORMAL):
                assert d.algo in (C.TDX_ALGO_ATEN, C.TDX_ALGO_ATEN_WIDE), e.name
                assert d.fill_bits[1] in {_C.aten_stream_policy(n, *H100)[0] for n in e.rng_numels}, e.name
                vals[at:at + n] = O.aten_units(d)
                ids[at:at + n] = programs(d.src, d.p0, d.p1, [(d.epi[k].op, d.epi[k].a, d.epi[k].b) for k in range(d.n_epi)],
                                          d.algo)
            else:
                assert not d.reserved & C.TDX_FLAG_WINDOW or d.src == C.TDX_SRC_CONST
                ids[at:at + n] = -1
        out[e.name] = (vals.reshape(sizes), ids.reshape(sizes))
        if narrowed(e, steps=steps_of(e)):  # (listed whole: narrowed on the device)
            out[e.name] = tuple(apply_steps(torch.from_numpy(x), steps_of(e)).numpy() for x in out[e.name])
    return out, end


def whole_draws(plan, programs):
    """{name: (values, program ids)} of every whole tensor, restated from the plan's entries alone: each
    pass at ATen's offset in plan order, each drawn element by its global index; and the offset after."""
    offset, at_pass, out = OFFSET, {}, {}
    for e in plan.entries:
        if e.source in ("alias", "value"):
            continue
        offsets = []
        for k, n in enumerate(e.rng_numels):
            pid = e.rng_ids[k] if e.rng_ids else None
            if pid is None or pid not in at_pass:
                at_pass[pid] = offset
                offset += policy(n, *H100)[1]
            offsets.append(at_pass[pid])
        numel = int(np.prod(e.sizes)) if e.sizes else 1
        vals, ids = np.full(numel, np.nan, dtype=np.float32), np.full(numel, -2, dtype=np.int64)
        for g in e.segment_list():
            lo, hi = g["begin"], g["end"]
            if g["source"] == "uninit":
                continue
            if not drawn(g):
                ids[lo:hi] = -1
                continue
            src = C.TDX_SRC_NORMAL if g["source"] == "normal" else C.TDX_SRC_UNIFORM
            algo = C.TDX_ALGO_ATEN_WIDE if g["aten_wide"] else C.TDX_ALGO_ATEN
            vals[lo:hi] = O.aten_units(C.make_desc(0, dtype=C.TDX_F32, src=src, elem_begin=lo - g["origin"],
                                                   elem_count=hi - lo, seed=SEED, offset=offsets[g["rng_pass"]],
                                                   algo=algo, aten_stride=policy(e.rng_numels[g["rng_pass"]], *H100)[0]))
            ids[lo:hi] = programs(src, g["p0"], g["p1"], g["epilogue"], algo)
        out[e.name] = (vals.reshape(e.sizes), ids.reshape(e.sizes))
    return out, offset


def check_layout(plan, steps_of, **kw):
    """Every block of the table is its chunk steps of the whole restatement; returns the drawn elements."""
    programs = Programs()
    whole, end = whole_draws(plan, programs)
    got, got_end = table_of(plan, steps_of, programs, **kw)
    assert got_end == end
    n = 0
    for name, (vals, ids) in whole.items():
        want_v, want_i = (apply_steps(torch.from_numpy(x), steps_of_name(plan, steps_of, name)).numpy() for x in (vals, ids))
        gv, gi = got[name]
        assert gv.shape == want_v.shape, (name, gv.shape, want_v.shape)
        assert np.array_equal(gi, want_i) and np.array_equal(gv, want_v, equal_nan=True), name
        n += int((gi >= 0).sum())
    return n


def steps_of_name(plan, steps_of, name):
    return steps_of(next(e for e in plan.entries if e.name == name))


def plan_through_json(case, dtype, tmp_path):
    plan = InitPlan.from_module(record(case, dtype), rng="aten")
    plan.save(str(tmp_path / "p.json"))
    return InitPlan.load(str(tmp_path / "p.json"))


@pytest.mark.parametrize("case,dtype", [("tiny_llama", "bf16"), ("family_opt", "fp32"), ("init_zoo", "fp32"),
                                        ("cast_variant", "fp32"), ("padded_embeddings", "bf16")])
def test_dim0_shards_are_slices_of_the_whole_draw(case, dtype, tmp_path):
    plan = plan_through_json(case, dtype, tmp_path)
    whole = check_layout(plan, lambda e: [])
    assert whole > 0
    for world in (2, 3, 8):
        total = 0
        for r in range(world):
            total += check_layout(plan, lambda e: chunk_steps(e, (r, world)), shard=(r, world))
        assert total == whole - sum(int(np.prod(e.sizes)) for e in plan.entries
                                    if e.kind == "param" and e.source not in ("alias", "value") and not e.sizes)


@pytest.mark.parametrize("case", list(TP_PLANS))
def test_tp_placements_are_slices_of_the_whole_draw(case, tmp_path):
    plan = plan_through_json(case, "fp32", tmp_path)
    placements = tp_placements(record(case, "fp32"), TP_PLANS[case]())
    assert 1 in placements.values() and 0 in placements.values()
    windows = 0
    for world in (2, 3):
        for r in range(world):
            check_layout(plan, lambda e: chunk_steps(e, (r, world), placements.get(e.name)), shard=(r, world),
                         placements=placements)
            table, _ = plan.descriptors(SEED, OFFSET, (r, world), placements=placements, device_props=H100)
            windows += sum(bool(d.reserved & C.TDX_FLAG_WINDOW) for _, _, descs in table for d in descs)
    assert windows > 0  # (Rowwise weights: windowed ATen-stream descriptors)


def test_fsdp_tp_blocks_are_slices_of_the_whole_draw(tmp_path):
    plan = plan_through_json("tiny_llama", "fp32", tmp_path)
    alias = {e.name for e in plan.entries if e.source == "alias"}
    two_d = 0
    for blocks in fake_blocks("tiny_llama", MESHES["dp2_tp4"]):
        blocks = {k: v for k, v in blocks.items() if k not in alias}
        check_layout(plan, lambda e: list(blocks.get(e.name, [])), blocks=blocks)
        two_d += sum(len({d for d, _, n in s if n > 1}) == 2 for s in blocks.values())
    assert two_d > 0


# ---------------------------------------------------------------------------------------------- refusals
class Transposed(nn.Module):
    def __init__(self):
        super().__init__()
        self.ok = nn.Parameter(torch.empty(8, 8).normal_())
        self.w = nn.Parameter(torch.empty(30, 20).t().normal_().t())


class Huge(nn.Module):
    def __init__(self):
        super().__init__()
        self.w = nn.Parameter(torch.empty(2**30 + 1, dtype=torch.bfloat16).normal_())


class Reciprocal(nn.Module):
    def __init__(self):
        super().__init__()
        self.w = nn.Parameter(1.0 / torch.rand(64, 8))


class Pow(nn.Module):
    def __init__(self):
        super().__init__()
        self.w = nn.Parameter(2.0 ** torch.rand(64, 8))


@pytest.mark.parametrize("cls,reason", [(Huge, "64-bit"), (Reciprocal, "reciprocal"), (Pow, "pow")])
def test_programs_atens_stream_cannot_take_are_refused(cls, reason):
    """The default stream folds these; ATen's stream replays them, which a plan cannot hold."""
    m = deferred_init(cls)
    info = _C.plan_info(m.w, rng="aten")
    assert _C.plan_info(m.w)["fusible"] and reason in info["aten_refusal"] and not info["fusible"]
    with pytest.raises(ValueError, match=rf"'w' .*{reason}"):
        InitPlan.from_module(m, rng="aten")


def test_a_draw_through_a_transposed_view_is_refused():
    """The planner does not fold a draw through a strided view on either stream: refused as any random
    program it cannot fold."""
    m = deferred_init(Transposed)
    assert _C.plan_info(m.ok, rng="aten")["fusible"] and not _C.plan_info(m.w, rng="aten")["fusible"]
    with pytest.raises(ValueError, match="'w' has a random initialisation program"):
        InitPlan.from_module(m, rng="aten")


def test_aten_plan_descriptors_need_the_device():
    plan = InitPlan.from_module(record("linear128", "fp32"), rng="aten")
    with pytest.raises(ValueError, match="device_props"):
        plan.descriptors(SEED, OFFSET)
    table, end = plan.descriptors(SEED, OFFSET, device_props=H100)
    assert end == OFFSET + policy(128 * 128, *H100)[1] + policy(128, *H100)[1]  # kaiming_uniform_, then the bias
    # the default stream ignores the device
    fused = InitPlan.from_module(record("linear128", "fp32"))
    assert [bytes(d) for _, _, ds in fused.descriptors(SEED, OFFSET)[0] for d in ds] == \
        [bytes(d) for _, _, ds in fused.descriptors(SEED, OFFSET, device_props=H100)[0] for d in ds]
