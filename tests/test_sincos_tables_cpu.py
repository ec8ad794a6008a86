"""Sinusoidal position tables (Whisper, M2M100 / NLLB, GPT-J, CodeGen, MusicGen) on the fused path,
without a GPU: planner verdicts on the transformers classes and on replicas of their builders, the
negatives that stay opaque, InitPlan for models whose tables could not be planned before, and the
host chain InitPlan -> JSON -> descriptors -> CPU restatement of the kernel (oracle/tdx_oracle.c)
against the eager CPU construction."""
import json
import math
import warnings

import pytest
import torch
import transformers as T
from torch import nn

import sincos_replicas as R
from oracle import tdx_oracle as O
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, plan_report
from torchdistx_b200.plan import FORMAT, FORMAT_SINCOS, InitPlan

warnings.filterwarnings("ignore", module="transformers")

_ENC_DEC = dict(d_model=64, encoder_layers=1, decoder_layers=1, encoder_attention_heads=4, decoder_attention_heads=4,
                encoder_ffn_dim=64, decoder_ffn_dim=64, vocab_size=256)
MODELS = {
    "whisper": (lambda: T.WhisperModel(T.WhisperConfig(
        **_ENC_DEC, max_source_positions=30, max_target_positions=32, pad_token_id=0, decoder_start_token_id=1,
        bos_token_id=1, eos_token_id=2)), ["encoder.embed_positions.weight"]),
    "m2m100": (lambda: T.M2M100Model(T.M2M100Config(**_ENC_DEC, max_position_embeddings=32)),
               ["encoder.embed_positions.weights", "decoder.embed_positions.weights"]),
    "gptj": (lambda: T.GPTJForCausalLM(T.GPTJConfig(n_embd=64, n_layer=2, n_head=4, rotary_dim=16, vocab_size=256,
                                                    n_positions=64)),
             ["transformer.h.0.attn.embed_positions", "transformer.h.1.attn.embed_positions"]),
    "codegen": (lambda: T.CodeGenForCausalLM(T.CodeGenConfig(n_embd=64, n_layer=2, n_head=4, rotary_dim=16,
                                                             vocab_size=256, n_positions=64, n_ctx=64)),
                ["transformer.h.0.attn.embed_positions", "transformer.h.1.attn.embed_positions"]),
    "musicgen": (lambda: T.MusicgenForCausalLM(T.MusicgenDecoderConfig(
        hidden_size=64, num_hidden_layers=1, num_attention_heads=4, ffn_dim=64, vocab_size=64,
        max_position_embeddings=64, num_codebooks=2)), ["model.decoder.embed_positions.weights"]),
}


def sincos_segments(info):
    return [s for s in info["segments"] if s["source"] == "sincos"]


@pytest.mark.parametrize("name", sorted(MODELS))
def test_transformers_tables_fold(name):
    build, tables = MODELS[name]
    r = plan_report(deferred_init(build))
    total = sum(v["numel"] for v in r.values())
    fused = sum(v["numel"] for v in r.values() if v["fusible"])
    assert fused / total == 1.0, {k: v["first_unfusable_op"] for k, v in r.items() if not v["fusible"]}
    for t in tables:
        info = r[t]
        assert info["source"] == "sincos" and info["fusible"], (t, info)
        segs = sincos_segments(info)
        padded = name == "m2m100"  # the padding row splits the table into three segments
        assert len(info["segments"]) == (3 if padded else 1) and len(segs) == (2 if padded else 1), info["segments"]
        W = info["sizes"][1]
        assert all(s["sincos_half"] * 2 == W for s in segs)
        assert all(s["sincos_cos_first"] == (name == "musicgen") for s in segs)


def test_replicas_fold():
    r = plan_report(deferred_init(R.WhisperPositions, 30, 64))["embed_positions.weight"]
    assert (r["source"], r["fusible"], r["rng_ops"]) == ("sincos", True, 2)  # two dead normal_ passes
    (s,) = r["segments"]
    assert (s["sincos_half"], s["sincos_cos_first"], s["p0"], s["p1"]) == (32, False, 0.0, 1.0)
    r = plan_report(deferred_init(R.M2M100Positions, 30, 64, 1))["weights"]
    assert [g["source"] for g in r["segments"]] == ["sincos", "const", "sincos"]
    assert [(g["begin"], g["end"]) for g in r["segments"]] == [(0, 64), (64, 128), (128, 32 * 64)]
    r = plan_report(deferred_init(R.MusicgenPositions, 30, 64))["weights"]
    assert r["source"] == "sincos" and r["segments"][0]["sincos_cos_first"]
    r = plan_report(deferred_init(R.GPTJAttentionPositions, 64, 16))["embed_positions"]
    assert r["source"] == "sincos" and r["segments"][0]["sincos_half"] == 8 and len(r["epilogue"]) == 4


class Negatives(nn.Module):
    def __init__(self):
        super().__init__()
        rows = torch.arange(12).float()[:, None]
        cols = torch.exp(torch.arange(4).float() * -0.5)[None, :]
        o = rows * cols
        self.register_buffer("outer", o)  # the product alone
        self.register_buffer("sin_only", torch.sin(o))
        self.register_buffer("dim0", torch.cat([torch.sin(o), torch.cos(o)], dim=0))
        other = rows * torch.exp(torch.arange(4).float() * -0.25)[None, :]
        self.register_buffer("two_products", torch.cat([torch.sin(o), torch.cos(other)], dim=1))
        self.register_buffer("sin_sin", torch.cat([torch.sin(o), torch.sin(o)], dim=1))
        self.register_buffer("rng_sin", torch.sin(torch.randn(8, 8)))
        self.register_buffer("sin_1d", torch.sin(torch.arange(40, dtype=torch.float32)))
        self.register_buffer("mask", torch.tril(torch.ones(8, 8)))
        self.register_buffer("odd", R.m2m100_embedding(12, 9, 1))  # a zero column appended by a second cat
        self.register_buffer("rows_from_1", torch.cat([torch.sin((rows + 1) * cols), torch.cos((rows + 1) * cols)], 1))
        t = torch.cat([torch.sin(o), torch.cos(o)], dim=1)
        self.register_buffer("scaled", t * 2.0)  # nothing folds onto a table but a final cast


def test_negatives_stay_opaque():
    r = plan_report(deferred_init(Negatives))
    for name in ("outer", "sin_only", "dim0", "two_products", "sin_sin", "rng_sin", "sin_1d", "mask", "odd",
                 "rows_from_1", "scaled"):
        assert r[name]["source"] == "opaque" and not r[name]["fusible"], (name, r[name]["source"])


class Tables(nn.Module):
    """The four builders at real sizes: Whisper large-v3, NLLB (padding_idx 1), GPT-J, MusicGen."""

    def __init__(self):
        super().__init__()
        self.whisper = R.WhisperPositions(1500, 1280)
        self.nllb = R.M2M100Positions(1024, 1024, 1)
        self.gptj = R.GPTJAttentionPositions(2048, 64)
        self.musicgen = R.MusicgenPositions(2048, 1024)


def test_from_module_plans_whisper_and_a_large_m2m100_table():
    # Whisper's dead normal_ passes made its table a random program a plan could not embed, and the
    # NLLB table (4.2 MB) was over the 1 MB embedding limit
    for cls, args in ((R.WhisperPositions, (1500, 1280)), (R.M2M100Positions, (1024, 1024, 1))):
        plan = InitPlan.from_module(deferred_init(cls, *args))
        assert [e.source for e in plan.entries] == ["sincos"], [(e.name, e.source) for e in plan.entries]
        assert plan.uses_sincos()


# The column program of each table, run eagerly on the CPU.
COLUMNS = {
    "whisper.embed_positions.weight": lambda: torch.exp(-(math.log(10000) / 639) * torch.arange(640)),
    "nllb.weights": lambda: torch.exp(torch.arange(512, dtype=torch.int64).float() * -(math.log(10000) / 511)),
    "gptj.embed_positions": lambda: 1.0 / (10000 ** (torch.arange(0, 64, 2, dtype=torch.int64) / 64)),
    "musicgen.weights": lambda: torch.exp(torch.arange(512, dtype=torch.int64).float() * -(math.log(10000) / 511)),
}


def _check(name, entry, got, want):
    """The restatement against the eager CPU table: within 4 * 2^-24 in fp32 (sinf / cosf of libm and
    of ATen's CPU kernels differ by an ulp or two), identical or one ulp apart in bf16 / fp16.  That
    bar holds where the two column programs agree.  ATen's vectorised CPU exp / pow and libm's expf /
    powf differ in the last bit for a few column values (the kernel computes them as ATen's CUDA
    kernels do: tests/test_sincos_tables_gpu.py is bit-exact), and float(r) * f carries that
    difference times the row index: those columns are held to the bound it implies."""
    seg = next(g for g in entry.segments if g["source"] == "sincos")
    half = seg["sincos_half"]
    col = C.make_desc(0, dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_count=half, p0=seg["p0"], p1=seg["p1"],
                      epi=seg["epilogue"])
    f_o = R.as_tensor(O.generate(col), torch.float32).double()
    f_e = COLUMNS[name]().double()
    differ = f_o != f_e
    assert int(differ.sum()) <= max(1, half // 50), (name, int(differ.sum()))
    rows = got.shape[0]
    slack = torch.where(differ, (rows - 1) * (2 * (f_o - f_e).abs() + f_e.abs() * 2.0 ** -23), torch.zeros(half))
    slack = torch.cat([slack, slack])[None, :]
    err = (got.double() - want.double()).abs()
    if got.dtype == torch.float32:
        return bool((err <= 4 * 2.0 ** -24 + slack).all())
    ulps = (got.view(torch.int16).int() - want.view(torch.int16).int()).abs()
    ulp16 = (want.double().abs() * 2.0 ** -7).clamp(min=2.0 ** -24)  # (at least one ulp of either dtype)
    return bool(((ulps <= 1) | ((slack > 0) & (err <= slack + ulp16))).all())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_plan_round_trip_and_cpu_restatement(tmp_path, dtype):
    torch.manual_seed(0)
    m = deferred_init(lambda: Tables().to(dtype))
    plan = InitPlan.from_module(m)
    p = tmp_path / "tables.json"
    plan.save(str(p))
    assert json.load(open(p))["format"] == FORMAT_SINCOS
    plan = InitPlan.load(str(p))
    got, end, _ = O.evaluate_plan(plan, 7, 0)
    eager = {
        "whisper.embed_positions.weight": R.sinusoids(1500, 1280),
        "nllb.weights": R.m2m100_embedding(1026, 1024, 1),
        "gptj.embed_positions": R.create_sinusoidal_positions(2048, 64),
        "musicgen.weights": R.musicgen_embedding(2048, 1024),
    }
    assert set(got) == set(eager)
    for name, want in eager.items():
        want = want.to(dtype)
        assert got[name].dtype == dtype and got[name].shape == want.shape, name
        entry = next(e for e in plan.entries if e.name == name)
        assert _check(name, entry, got[name], want), (name, dtype)
    assert torch.equal(got["nllb.weights"][1], torch.zeros(1024, dtype=dtype))
    # the Whisper parameter's two dead normal_ passes still move the generator
    assert end > 0
    # shards of the parameter are torch.chunk of the whole
    for world in (2, 3, 8):
        parts = [O.evaluate_plan(plan, 7, 0, shard=(r, world))[0] for r in range(world)]
        whole = torch.cat([q["whisper.embed_positions.weight"] for q in parts])
        assert torch.equal(whole.view(torch.uint8), got["whisper.embed_positions.weight"].view(torch.uint8)), world


def test_plans_without_a_table_keep_their_format(tmp_path):
    plan = InitPlan.from_module(deferred_init(nn.Linear, 8, 8))
    plan.save(str(tmp_path / "p.json"))
    assert json.load(open(tmp_path / "p.json"))["format"] == FORMAT and not plan.uses_sincos()


def test_library_validates_the_table_descriptor():
    good = dict(dtype=C.TDX_F32, src=C.TDX_SRC_SINCOS, elem_count=64, sincos_half=8)
    assert C.prepare([C.make_desc(1 << 20, **good)]) > 0
    assert list(C.make_desc(0, **dict(good, sincos_cos_first=True)).fill_bits) == [8, C.TDX_SINCOS_COS_FIRST]
    bad = [C.make_desc(1 << 20, **dict(good, sincos_half=0)), C.make_desc(1 << 20, **dict(good, dtype=C.TDX_I64)),
           C.make_desc(1 << 20, **dict(good, elem_begin=16 << 24))]  # (row 2^24: float(r) is no longer exact)
    d = C.make_desc(1 << 20, **good)
    d.fill_bits[1] = 2  # an undefined flag bit
    bad.append(d)
    for d in bad:
        with pytest.raises(RuntimeError, match="TDX_SRC_SINCOS|TDX_I64 is IOTA-only"):
            C.prepare([d])
    # the last row below 2^24 is accepted
    assert C.prepare([C.make_desc(1 << 20, **dict(good, elem_begin=16 * ((1 << 24) - 1), elem_count=16))]) > 0
