"""Copies of host-built tensors (TDX_SRC_GATHER) without a GPU: planner verdicts on the real Pegasus,
Marian and RWKV classes, the negatives that stay opaque, the version check, descriptor validation, and
the host chain InitPlan -> JSON -> descriptors -> CPU restatement (oracle/tdx_oracle.c) against the
eager CPU construction, whole and in shards."""
import json
import warnings

import numpy as np
import pytest
import torch
import transformers as T
from torch import nn

from oracle import tdx_oracle as O
from torchdistx_b200 import _C
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, materialize_tensor, plan_report
from torchdistx_b200.plan import FORMAT_GATHER, InitPlan

warnings.filterwarnings("ignore", module="transformers")

_ENC_DEC = dict(vocab_size=64, d_model=32, encoder_layers=1, decoder_layers=1, encoder_attention_heads=2,
                decoder_attention_heads=2, encoder_ffn_dim=64, decoder_ffn_dim=64, max_position_embeddings=50)
PEGASUS = lambda: T.PegasusModel(T.PegasusConfig(**_ENC_DEC))
MARIAN = lambda: T.MarianModel(T.MarianConfig(**_ENC_DEC, pad_token_id=0, decoder_start_token_id=0))
RWKV = lambda: T.RwkvModel(T.RwkvConfig(vocab_size=64, hidden_size=40, num_hidden_layers=3, attention_hidden_size=40,
                                        intermediate_size=64, context_length=16))
TABLES = ["encoder.embed_positions.weight", "decoder.embed_positions.weight"]


def fraction(r):
    return sum(v["numel"] for v in r.values() if v["fusible"]) / sum(v["numel"] for v in r.values())


@pytest.mark.parametrize("build", [PEGASUS, MARIAN], ids=["pegasus", "marian"])
def test_pegasus_and_marian_tables_fold(build):
    r = plan_report(deferred_init(build))
    assert fraction(r) == 1.0, {k: v["first_unfusable_op"] for k, v in r.items() if not v["fusible"]}
    for t in TABLES:
        info = r[t]
        (seg,) = info["segments"]  # the two column halves make one host image
        assert (info["source"], seg["gather_period"], seg["gather_repeat"]) == ("gather", 0, 0), info
        assert len(seg["gather_bytes"]) == 50 * 32 * 4


def test_rwkv_time_parameters_fold_and_what_stays_opaque():
    r = plan_report(deferred_init(RWKV))
    for layer in range(3):
        a, f = f"blocks.{layer}.attention.", f"blocks.{layer}.feed_forward."
        for name in [a + "time_decay", a + "time_mix_key", a + "time_mix_value", a + "time_mix_receptance",
                     f + "time_mix_key", f + "time_mix_receptance"]:
            assert r[name]["source"] == "gather" and r[name]["fusible"], (name, r[name])
    # What is left: orthogonal_ (a QR decomposition of a normal draw) for the embedding and every
    # linear weight, and time_first -- `ones_like(time_first * log(0.3) + zigzag)` reads the
    # parameter while it is still uninitialised, a reader that is replayed at its point in history
    opaque = {k for k, v in r.items() if not v["fusible"]}
    linear = {f"blocks.{i}.{m}.{w}.weight" for i in range(3)
              for m, ws in (("attention", ("key", "value", "receptance", "output")),
                            ("feed_forward", ("key", "receptance", "value"))) for w in ws}
    time_first = {f"blocks.{i}.attention.time_first" for i in range(3)}
    assert opaque == {"embeddings.weight"} | linear | time_first, sorted(opaque)
    rest = sum(r[k]["numel"] for k in opaque)
    assert fraction(r) == pytest.approx(1.0 - rest / sum(v["numel"] for v in r.values()))


def test_broadcast_and_cast_forms():
    row = torch.arange(6, dtype=torch.float64) / 7  # real tensors, built outside the recording
    col = torch.tensor([[1.5], [2.5], [3.5]])

    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.a = nn.Parameter(torch.empty(4, 6))
            self.b = nn.Parameter(torch.empty(3, 5))
            self.c = nn.Parameter(torch.empty(2, 3, 5))
            self.register_buffer("ids", torch.empty(3, dtype=torch.int64))
            with torch.no_grad():
                self.a.copy_(row)  # broadcast over rows: P = 6
                self.b.copy_(col)  # each value repeated along a row: P = 3, R = 5
                self.c.copy_(col.expand(3, 5))  # an expand of a real tensor
                self.ids.copy_(torch.tensor([3, 1, 2]))

    r = plan_report(deferred_init(lambda: M().to(torch.bfloat16)))
    geo = lambda n: (r[n]["source"], r[n]["dtype"], r[n]["segments"][0]["gather_period"], r[n]["segments"][0]["gather_repeat"])
    assert geo("a") == ("gather", "BFloat16", 6, 0)
    assert geo("b") == ("gather", "BFloat16", 3, 5)
    assert geo("c") == ("gather", "BFloat16", 3, 5)
    assert geo("ids") == ("gather", "Long", 0, 0)


class Negatives(nn.Module):
    def __init__(self, big, strided):
        super().__init__()
        self.big = nn.Parameter(torch.empty(big.shape))
        self.strided = nn.Parameter(torch.empty(strided.shape))
        with torch.no_grad():
            self.big.copy_(big)
            self.strided.copy_(strided)


def test_negatives_stay_opaque():
    # (a real CUDA source: tests/test_gather_init_gpu.py)
    big = torch.randn(300_000)  # 1.2 MB: over the bound
    strided = torch.randn(6, 4).t()  # non-contiguous
    r = plan_report(deferred_init(Negatives, big, strided))
    for name in ("big", "strided"):
        assert r[name]["source"] == "opaque" and not r[name]["fusible"], (name, r[name])
    # a source of exactly 1 MB folds
    assert plan_report(deferred_init(Negatives, torch.randn(1 << 18), torch.ones(4, 6)))[
        "big"]["source"] == "gather"


def test_a_source_mutated_after_recording_raises_the_version_error():
    src = torch.ones(8)

    def build():
        p = nn.Parameter(torch.empty(8))
        with torch.no_grad():
            p.copy_(src)
        return p

    p = deferred_init(build)
    assert dict(_C.plan_info(p))["source"] == "gather"
    src.add_(1)
    assert dict(_C.plan_info(p))["source"] == "opaque"  # read when evaluated: the version check sees it
    with pytest.raises(RuntimeError, match="updated in-place"):
        materialize_tensor(p)
    # unchanged, the value is the one at materialisation time (not a snapshot of recording time)
    src2 = torch.ones(8)
    q = deferred_init(lambda: nn.Parameter(torch.empty(8)).requires_grad_(False).copy_(src2))
    assert torch.equal(materialize_tensor(q), torch.ones(8))


def test_library_validates_the_gather_descriptor():
    good = dict(dtype=C.TDX_F32, src=C.TDX_SRC_GATHER, elem_count=64, gather_src=1 << 20, gather_period=8)
    assert C.prepare([C.make_desc(1 << 21, **good)]) > 0
    assert C.prepare([C.make_desc(1 << 21, **dict(good, dtype=C.TDX_I64))]) > 0
    assert list(C.make_desc(0, **dict(good, gather_repeat=3)).fill_bits) == [1 << 20, 8 | 3 << 32]
    bad = [C.make_desc(1 << 21, **dict(good, gather_src=0)),  # null source
           C.make_desc(1 << 21, **dict(good, dtype=C.TDX_RAW32)),  # unsupported dtype
           C.make_desc(1 << 21, **dict(good, dtype=C.TDX_I64, epi=[(C.TDX_EPI_MUL, 2.0)])),  # int64 with a step
           C.make_desc(1 << 21, **dict(good, algo=1)),  # flag bits
           C.make_desc(1 << 21, **dict(good, flags=C.TDX_FLAG_SRC_NOROUND)),
           C.make_desc(1 << 21, **dict(good, gather_period=0, gather_repeat=2)),
           C.make_desc(1 << 21, **dict(good, gather_src=(1 << 20) + 2))]  # not element-aligned
    for d in bad:
        with pytest.raises(RuntimeError, match="TDX_SRC_GATHER|raw dtypes"):
            C.prepare([d])


class Steps(nn.Module):
    """Gather segments with a padding row, an epilogue and a broadcast source, in `dtype` from the start
    (steps on a 16-bit tensor round after each; the scalars are exact in every dtype, because ATen's
    CPU kernels round a scalar to a 16-bit dtype first and its CUDA kernels do not)."""

    def __init__(self, table, row, dtype):
        super().__init__()
        self.table = nn.Parameter(torch.empty(table.shape, dtype=dtype))
        self.scaled = nn.Parameter(torch.empty(37, row.numel(), dtype=dtype))
        with torch.no_grad():
            self.table.copy_(table)
            self.table[3].zero_()
            self.scaled.copy_(row).mul_(0.375).add_(1.25)


class Both(nn.Module):
    def __init__(self, table, row, dtype):
        super().__init__()
        self.peg = PEGASUS().to(dtype)  # (the tables' cast: the host source converted once)
        self.steps = Steps(table, row, dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_plan_round_trip_and_cpu_restatement(tmp_path, dtype):
    table = torch.from_numpy(np.random.default_rng(0).normal(size=(61, 24)))  # float64, like numpy's
    row = torch.linspace(-2, 2, 24)

    torch.manual_seed(0)
    plan = InitPlan.from_module(deferred_init(Both, table, row, dtype))
    p = tmp_path / "plan.json"
    plan.save(str(p))
    assert json.load(open(p))["format"] == FORMAT_GATHER and plan.uses_gather()
    plan = InitPlan.load(str(p))
    whole, _, _ = O.evaluate_plan(plan, 7, 0)
    got = {e.name: whole[e.name] for e in plan.entries if any(g["source"] == "gather" for g in e.segments)}
    torch.manual_seed(0)
    both = Both(table, row, dtype)
    eager = {f"peg.{t}": dict(both.peg.named_parameters())[t] for t in TABLES}
    eager.update({"steps.table": both.steps.table, "steps.scaled": both.steps.scaled})
    assert set(got) == set(eager)
    for name, want in eager.items():
        want = want.detach()
        assert got[name].dtype == dtype and got[name].shape == want.shape, name
        assert torch.equal(got[name].view(torch.uint8), want.contiguous().view(torch.uint8)), (name, dtype)
    # shards of the parameters are torch.chunk of the whole (61 and 37 rows: ragged)
    for world in (2, 3, 8):
        parts = [O.evaluate_plan(plan, 7, 0, shard=(r, world))[0] for r in range(world)]
        for name, whole in got.items():
            cat = torch.cat([q[name] for q in parts])
            assert torch.equal(cat.view(torch.uint8), whole.view(torch.uint8)), (world, name)
