"""Causal-mask buffers (TDX_SRC_BAND) without a GPU: planner verdicts on the real transformers classes,
the programs that stay opaque, InitPlan for models that could not be planned before, descriptor
validation, and the host chain InitPlan -> JSON -> descriptors -> CPU restatement of the kernel
(oracle/tdx_oracle.c) against the eager CPU construction, whole, in shards and at odd ranges."""
import json
import warnings

import pytest
import torch
import transformers as T
from torch import nn

import band_replicas as R
from oracle import tdx_oracle as O
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, materialize_module, plan_report
from torchdistx_b200.plan import FORMAT, FORMAT_BAND, InitPlan, entry_descriptors

warnings.filterwarnings("ignore", module="transformers")

P = 32  # positions of the toy models (a mask is P x P)
MODELS = {
    "gpt_bigcode": lambda: T.GPTBigCodeModel(T.GPTBigCodeConfig(
        vocab_size=64, n_positions=P, n_embd=32, n_layer=2, n_head=2)),
    "gpt_neo": lambda: T.GPTNeoModel(T.GPTNeoConfig(
        vocab_size=64, max_position_embeddings=P, hidden_size=32, num_layers=2, num_heads=2,
        attention_types=[[["global", "local"], 1]], window_size=8)),
    "imagegpt": lambda: T.ImageGPTModel(T.ImageGPTConfig(vocab_size=64, n_positions=P, n_embd=32, n_layer=1, n_head=2)),
    "openai_gpt": lambda: T.OpenAIGPTModel(T.OpenAIGPTConfig(vocab_size=64, n_positions=P, n_embd=32, n_layer=1, n_head=2)),
    "bark": lambda: T.BarkSemanticModel(T.BarkSemanticConfig(
        block_size=P, input_vocab_size=64, output_vocab_size=64, num_layers=1, num_heads=2, hidden_size=32)),
    "clvp": lambda: T.ClvpDecoder(T.ClvpDecoderConfig(
        vocab_size=64, max_position_embeddings=P, max_text_tokens=P, hidden_size=32, num_hidden_layers=1,
        num_attention_heads=2)),
}
TRUE, ONE_F32 = 1, 0x3F800000
# every mask: (name, lo, hi, IN bits); R = C = P, OUT = 0
MASKS = {
    "gpt_bigcode": [("bias", -P, 0, TRUE)],
    "gpt_neo": [("h.0.attn.attention.bias", -P, 0, TRUE), ("h.1.attn.attention.bias", -7, 0, TRUE)],
    "imagegpt": [("h.0.attn.bias", -P, 0, TRUE)],
    "openai_gpt": [("h.0.attn.bias", -P, 0, ONE_F32)],
    "bark": [("layers.0.attn.bias", -P, 0, TRUE)],
    "clvp": [("layers.0.attn.bias", -P, 0, TRUE)],
}
# what else in these classes is not on the fused path, and why
OPAQUE = {
    "gpt_bigcode": set(), "gpt_neo": set(), "imagegpt": set(), "openai_gpt": set(), "bark": set(),
    "clvp": set(),
}


def band_segments(info):
    return [s for s in info["segments"] if s["source"] == "band"]


@pytest.mark.parametrize("name", sorted(MODELS))
def test_transformers_masks_are_bands(name):
    torch.manual_seed(0)
    r = plan_report(deferred_init(MODELS[name]))
    for key, lo, hi, bits in MASKS[name]:
        info = r[key]
        assert (info["source"], info["fusible"]) == ("band", True), (key, info["source"], info["first_unfusable_op"])
        (s,) = info["segments"]
        assert (s["band_rows"], s["band_cols"], s["band_lo"], s["band_hi"], s["band_in"], s["band_out"]) == \
            (P, P, lo, hi, bits, 0), (key, s)
    opaque = {k for k, v in r.items() if not v["fusible"]}
    assert opaque == OPAQUE[name], {k: r[k]["first_unfusable_op"] for k in opaque}


MAX = {"gpt_bigcode": 8192, "gpt_neo": 2048}


@pytest.mark.parametrize("name", sorted(MAX))
def test_from_module_plans_full_size_masks_without_embedding_them(tmp_path, name):
    """StarCoder's 8192^2 mask (64 MiB) and GPT-Neo's 2048^2 masks (4 MiB each) were over the 1 MiB a plan
    embeds: such models had no plan.  The masks are band entries now, with no value bytes."""
    n = MAX[name]
    cfg = (T.GPTBigCodeConfig(vocab_size=64, n_positions=n, n_embd=32, n_layer=1, n_head=2) if name == "gpt_bigcode"
           else T.GPTNeoConfig(vocab_size=64, max_position_embeddings=n, hidden_size=32, num_layers=2, num_heads=2,
                               attention_types=[[["global", "local"], 1]], window_size=256))
    cls = T.GPTBigCodeModel if name == "gpt_bigcode" else T.GPTNeoModel
    plan = InitPlan.from_module(deferred_init(cls, cfg))
    masks = [e for e in plan.entries if e.name.endswith("bias") and e.dtype == "Bool"]
    assert masks and all(e.source == "band" and e.value == "" for e in masks), [(e.name, e.source) for e in masks]
    assert plan.uses_band()
    plan.save(str(tmp_path / "p.json"))
    assert json.load(open(tmp_path / "p.json"))["format"] == FORMAT_BAND
    assert all(e.source == "band" for e in InitPlan.load(str(tmp_path / "p.json")).entries if e.name in
               {m.name for m in masks})


def test_plans_without_a_mask_keep_their_format(tmp_path):
    plan = InitPlan.from_module(deferred_init(nn.Linear, 8, 8))
    plan.save(str(tmp_path / "p.json"))
    assert json.load(open(tmp_path / "p.json"))["format"] == FORMAT and not plan.uses_band()


class Negatives(nn.Module):
    def __init__(self):
        super().__init__()
        n = 32
        self.register_buffer("rng", torch.tril(torch.randn(n, n)))  # tril of a random program
        self.register_buffer("index", torch.tril(torch.arange(n * n, dtype=torch.float32).view(n, n)))
        nonzero_out = torch.full((n, n), float("-inf")).triu(1)  # OUT is 0, IN -inf: tril of it folds ...
        self.register_buffer("ok", torch.tril(nonzero_out, 4))
        shifted = torch.tril(torch.ones(n, n)) + 1.0  # ... a band with OUT = 1 under tril does not
        self.register_buffer("shifted", torch.tril(shifted))
        a = torch.tril(torch.ones((n, n), dtype=torch.bool))
        o = torch.ones((n, n), dtype=torch.bool)
        self.register_buffer("crossing", torch.bitwise_xor(torch.tril(o, 2), torch.triu(o, -3)))  # not nested
        self.register_buffer("other_shape", torch.bitwise_xor(a[:16], torch.tril(torch.ones((16, n), dtype=torch.bool))))
        self.register_buffer("cumsum", torch.ones(n, n).cumsum(0))
        self.register_buffer("transposed", torch.tril(torch.ones(n, 2 * n).t()))  # a non-contiguous argument
        self.register_buffer("scaled", torch.tril(torch.ones(n, n)) * 2.0)  # a step on a band
        self.register_buffer("small", torch.tril(torch.ones(8, 8)))  # under 16 x 16: as before


def test_negatives_stay_opaque_and_replay_the_right_values():
    r = plan_report(deferred_init(Negatives))
    for name in ("rng", "index", "shifted", "crossing", "other_shape", "cumsum", "transposed", "scaled", "small"):
        assert r[name]["source"] == "opaque" and not r[name]["fusible"], (name, r[name]["source"])
    assert r["ok"]["source"] == "band"
    (s,) = r["ok"]["segments"]
    assert (s["band_lo"], s["band_hi"], s["band_out"]) == (1, 4, 0)
    # (a CPU module replays through ATen, the `rng` draw included)
    m = deferred_init(Negatives)
    torch.manual_seed(0)
    materialize_module(m)
    torch.manual_seed(0)
    eager = Negatives()
    for name, buf in eager.named_buffers():
        assert torch.equal(getattr(m, name), buf), name


def test_closing_casts_and_in_place_forms():
    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.register_buffer("as_bool", torch.tril(torch.ones(16, 24)).bool())
            self.register_buffer("bf16", torch.full((2, 16, 16), float("-inf")).triu(1).to(torch.bfloat16))
            x = torch.ones(16, 16, dtype=torch.int64)
            x.tril_(-2)
            self.register_buffer("inplace", x)
            self.register_buffer("empty", torch.triu(torch.ones(16, 16), 16))  # no diagonal left: zeros
            self.register_buffer("clone", torch.tril(torch.ones(16, 16, dtype=torch.bool)).view(1, 16, 16).clone())

    r = plan_report(deferred_init(M))
    seg = lambda k: r[k]["segments"][0]
    assert r["as_bool"]["source"] == "band" and (seg("as_bool")["band_in"], seg("as_bool")["band_rows"],
                                                 seg("as_bool")["band_cols"]) == (1, 16, 24)
    assert r["bf16"]["source"] == "band" and (seg("bf16")["band_in"], seg("bf16")["band_lo"]) == (0xFF80, 1)
    assert r["inplace"]["source"] == "band" and (seg("inplace")["band_hi"], seg("inplace")["band_in"]) == (-2, 1)
    assert r["empty"]["source"] == "const"
    assert r["clone"]["source"] == "band"


def test_library_validates_the_band_descriptor():
    good = dict(dtype=C.TDX_RAW8, src=C.TDX_SRC_BAND, elem_count=64, band_rows=8, band_cols=8, band_lo=-8,
                band_hi=0, band_in=1)
    assert C.prepare([C.make_desc(1 << 20, **good)]) > 0
    for dt in (C.TDX_RAW16, C.TDX_RAW32, C.TDX_RAW64, C.TDX_F32, C.TDX_BF16, C.TDX_F16, C.TDX_I64):
        assert C.prepare([C.make_desc(1 << 20, **dict(good, dtype=dt))]) > 0
    bad = [dict(good, band_rows=0), dict(good, band_cols=0), dict(good, band_rows=1 << 31),
           dict(good, band_cols=1 << 31), dict(good, band_lo=1, band_hi=0), dict(good, epi=[(C.TDX_EPI_MUL, 2.0)]),
           dict(good, algo=C.TDX_ALGO_BM32), dict(good, flags=C.TDX_FLAG_WINDOW),
           dict(good, flags=C.TDX_FLAG_SRC_NOROUND), dict(good, dtype=7)]
    for kw in bad:
        with pytest.raises(RuntimeError, match="TDX_SRC_BAND|unknown dtype"):
            C.prepare([C.make_desc(1 << 20, **kw)])


class Masks(nn.Module):
    """The replicas' masks at sizes that exercise every line shape of the restatement."""

    def __init__(self):
        super().__init__()
        self.bigcode = R.BigCodeMask(64)
        self.neo_global = R.NeoAttentionMask(48)
        self.neo_local = R.NeoAttentionMask(48, 5)
        self.openai = R.OpenAIMask(40)
        self.additive = R.AdditiveMask(24)
        self.additive16 = R.AdditiveMask(20, torch.bfloat16)
        self.wide = nn.Parameter(torch.triu(torch.ones(36, 17)), requires_grad=False)
        self.int64 = nn.Parameter(torch.tril(torch.ones((3, 19, 21), dtype=torch.int64), 3), requires_grad=False)


def test_plan_round_trip_and_cpu_restatement(tmp_path):
    m = deferred_init(Masks)
    plan = InitPlan.from_module(m)
    assert all(e.source == "band" for e in plan.entries), [(e.name, e.source) for e in plan.entries]
    p = tmp_path / "masks.json"
    plan.save(str(p))
    assert json.load(open(p))["format"] == FORMAT_BAND
    plan = InitPlan.load(str(p))
    eager = dict(Masks().named_parameters())
    eager.update(dict(Masks().named_buffers()))
    got, _, _ = O.evaluate_plan(plan, 7, 0)
    assert set(got) == set(eager)
    for name, want in eager.items():
        assert got[name].dtype == want.dtype and torch.equal(got[name], want.detach()), name
    # parameters in shards: torch.chunk of the whole (a band is indexed by the global element)
    for world in (2, 3, 5):
        parts = [O.evaluate_plan(plan, 7, 0, shard=(r, world))[0] for r in range(world)]
        for name in ("wide", "int64"):
            assert torch.equal(torch.cat([q[name] for q in parts]), got[name]), (name, world)
    # odd element ranges of every entry: a range starting mid-row, of any length
    for e in plan.entries:
        dtype = eager[e.name].dtype
        flat = eager[e.name].detach().reshape(-1)
        for begin, count in ((1, 7), (13, 29), (flat.numel() - 3, 3), (5, flat.numel() - 9)):
            descs = entry_descriptors(e, 0, begin, count, 7, [])
            part = torch.cat([R.as_tensor(O.generate(d), dtype) for d in descs])
            assert torch.equal(part, flat[begin:begin + count]), (e.name, begin, count)
