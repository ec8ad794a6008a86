"""CPU-side checks: the oracle is pinned to golden vectors, the C-ABI library loads and exports
every symbol include/tdx_init.h declares (no compute calls without a GPU), and the oracle's
transforms have the distributions they claim."""
import ctypes
import json
import math
import os
import re

import numpy as np
import pytest

from oracle import tdx_oracle as O
from torchdistx_b200 import _cabi as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_philox_matches_golden_vectors():
    kat = json.load(open(os.path.join(ROOT, "tests", "golden", "philox_kat.json")))
    assert len(kat["vectors"]) >= 32
    assert sum(v["source"].startswith("random123") for v in kat["vectors"]) == 3
    for v in kat["vectors"]:
        assert O.philox4x32(v["ctr"], v["key"]) == v["out"], v


def test_oracle_stream_matches_golden_vectors():
    """The normative stream (uniform / normal in fp32, bf16, fp16, the fp32 stream rounded, epilogues,
    index programs, fills) at three (seed, offset, first element) points each: the restatement may
    only change together with tests/golden/stream_vectors.json (make_stream_vectors.py)."""
    doc = json.load(open(os.path.join(ROOT, "tests", "golden", "stream_vectors.json")))
    assert doc["abi_version"] == C.load().tdx_abi_version() and len(doc["vectors"]) >= 50
    names = set()
    for v in doc["vectors"]:
        kw = dict(v["desc"])
        kw["epi"] = [tuple(e) for e in kw.get("epi", [])]
        d = C.make_desc(0, elem_count=v["elem_count"], elem_begin=v["elem_begin"], seed=v["seed"], offset=v["offset"], **kw)
        assert O.generate(d).tobytes().hex() == v["out_hex"], (v["name"], v["seed"], v["offset"], v["elem_begin"])
        names.add(v["name"])
    assert {"uniform_f32", "normal_bf16", "normal_bf16_from_the_fp32_stream", "trunc_normal_bf16", "rotary_inv_freq_f32",
            "rotary_inv_freq_bf16", "arange_i64", "fill_bool"} <= names
    # and the vectors mean what their names say (decoded, against the parameters they were made with)
    by = {(v["name"], v["elem_begin"]): v for v in doc["vectors"]}  # (0: the vector at seed 0, offset 0, first element 0)
    u = np.frombuffer(bytes.fromhex(by[("uniform_f32", 0)]["out_hex"]), dtype=np.float32)
    assert u.min() >= np.float32(-0.05) and u.max() < np.float32(0.03)
    t = np.frombuffer(bytes.fromhex(by[("trunc_normal_f32", 0)]["out_hex"]), dtype=np.float32)
    assert t.min() >= np.float32(-0.04) and t.max() <= np.float32(0.06)
    a = np.frombuffer(bytes.fromhex(by[("arange_i64", 0)]["out_hex"]), dtype=np.int64)
    assert a.tolist() == [5 + 3 * i for i in range(40)]
    f = np.frombuffer(bytes.fromhex(by[("rotary_inv_freq_f32", 0)]["out_hex"]), dtype=np.float32)
    exp = 1.0 / (500000.0 ** (np.arange(0, 80, 2, dtype=np.float64) / 64.0))  # 1 / base ** (arange(0, d, 2) / d), d = 64
    np.testing.assert_allclose(f, exp, rtol=1e-6)
    assert np.frombuffer(bytes.fromhex(by[("fill_bf16_one", 0)]["out_hex"]), dtype=np.uint16).tolist() == [0x3F80] * 40


def test_abi_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "tdx_init.h")).read()
    declared = set(re.findall(r"TDX_C_API\s+[\w\s\*]+?\b(tdx_\w+)\s*\(", header))
    assert declared == set(C.EXPORTED_SYMBOLS), declared ^ set(C.EXPORTED_SYMBOLS)
    lib = C.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.tdx_abi_version() == 2
    assert ctypes.sizeof(C.TdxInitDesc) == 128 and ctypes.sizeof(C.TdxPlan) == 4096
    assert lib.tdx_init_workspace_bytes(100) >= 100 * 128
    assert lib.tdx_elems_per_block(C.TDX_BF16, C.TDX_SRC_NORMAL, 0) == 8
    assert lib.tdx_elems_per_block(C.TDX_F32, C.TDX_SRC_UNIFORM, 0) == 4


def test_abi_rejects_bad_descriptors_without_touching_the_gpu():
    lib = C.load()
    d = C.make_desc(0x1000, dtype=C.TDX_RAW32, src=C.TDX_SRC_UNIFORM, elem_count=4)
    arr = (C.TdxInitDesc * 1)(d)
    assert lib.tdx_init_launch(arr, 1, None, 0, None) == -1  # TDX_E_BADARG
    assert b"raw dtypes" in lib.tdx_last_error()
    d = C.make_desc(0x1001, dtype=C.TDX_F32, src=C.TDX_SRC_UNIFORM, elem_count=4)
    arr = (C.TdxInitDesc * 1)(d)
    assert lib.tdx_init_launch(arr, 1, None, 0, None) == -1
    assert b"aligned" in lib.tdx_last_error()
    # algo bits that name no shipped kernel: flags outside the algorithm nibble and TDX_ALGO_NOLUT, and
    # algorithm 3 on a 16-bit normal
    for algo in (0x10, C.TDX_ALGO_ICDF16 | 0x10, 3):
        d = C.make_desc(0x1000, dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=4, algo=algo)
        arr = (C.TdxInitDesc * 1)(d)
        assert lib.tdx_init_launch(arr, 1, None, 0, None) == -1, algo
    assert lib.tdx_init_launch(None, 0, None, 0, None) == 0  # nothing to do is not an error


def bits_to_float(a, dtype):
    if dtype == C.TDX_F32:
        return a.view(np.float32).astype(np.float64)
    if dtype == C.TDX_BF16:
        return (a.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return a.view(np.float16).astype(np.float64)


@pytest.mark.parametrize("dtype", [C.TDX_F32, C.TDX_BF16, C.TDX_F16])
def test_oracle_uniform_distribution_and_bounds(dtype):
    n = 1 << 18
    d = C.make_desc(0, dtype=dtype, src=C.TDX_SRC_UNIFORM, elem_count=n, seed=3, offset=4, p0=-0.5, p1=0.25)
    x = bits_to_float(O.generate(d), dtype)
    assert x.min() >= -0.5 and x.max() < 0.25
    assert abs(x.mean() - (-0.125)) < 5 * (0.75 / 12 ** 0.5) / n ** 0.5 + 1e-3
    assert abs(x.std() / (0.75 / 12 ** 0.5) - 1) < 0.01


@pytest.mark.parametrize("dtype", [C.TDX_F32, C.TDX_BF16, C.TDX_F16])
def test_oracle_normal_distribution(dtype):
    from scipy import stats

    n = 1 << 18
    d = C.make_desc(0, dtype=dtype, src=C.TDX_SRC_NORMAL, elem_count=n, seed=11, offset=0, p0=1.0, p1=0.5)
    x = bits_to_float(O.generate(d), dtype)
    assert abs(x.mean() - 1.0) < 5 * 0.5 / n ** 0.5 + 2e-3
    assert abs(x.std() / 0.5 - 1) < 5 / (2 * n) ** 0.5 + 4e-3
    # two-sample Kolmogorov-Smirnov (alpha = 1e-3) against exact N(1, 0.5^2) draws rounded to the
    # same dtype (the rounding grid is coarse enough to matter for 16-bit types)
    import torch

    tdt = {C.TDX_F32: torch.float32, C.TDX_BF16: torch.bfloat16, C.TDX_F16: torch.float16}[dtype]
    ref = torch.from_numpy(np.random.default_rng(0).normal(1.0, 0.5, n)).to(tdt).double().numpy()
    assert stats.ks_2samp(x, ref).pvalue > 1e-3


def test_oracle_icdf16_tail_bins_reach_beyond_the_grid():
    # k == 0 has probability 2^-16 per element: 2^22 elements hold ~64 of them
    n = 1 << 22
    d = C.make_desc(0, dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=n, seed=5, offset=0, p0=0.0, p1=1.0)
    x = bits_to_float(O.generate(d), C.TDX_BF16)
    assert np.isfinite(x).all()
    grid_max = 4.17  # Phi^-1(1 - 2^-17)
    assert 20 <= (np.abs(x) > grid_max).sum() <= 140
    assert np.abs(x).max() < 8.5


def test_oracle_is_shard_invariant_and_offsets_disjoint():
    full = C.make_desc(0, dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=1000, seed=9, offset=16, p1=0.02)
    a = O.generate(full)
    parts = []
    for b, c in ((0, 123), (123, 500), (623, 377)):
        parts.append(O.generate(C.make_desc(0, dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_begin=b,
                                            elem_count=c, seed=9, offset=16, p1=0.02)))
    assert np.array_equal(a, np.concatenate(parts))
    other = O.generate(C.make_desc(0, dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=1000, seed=9,
                                   offset=20, p1=0.02))
    assert (a != other).mean() > 0.9


def test_prepare_lays_out_extreme_plans_within_the_workspace_bound():
    """tdx_init_prepare is host-only: the plan image (descriptor table, prefix sums, the table
    kernels' guided work lists) must fit tdx_init_workspace_bytes(n) for any mix -- one 180 GB tensor,
    thousands of table-eligible descriptors in every table family at once, nothing at all."""
    import ctypes

    lib = C.load()

    def prepare(descs):
        arr = (C.TdxInitDesc * len(descs))(*descs)
        need = ctypes.c_size_t(0)
        rc = lib.tdx_init_prepare(arr, len(descs), ctypes.byref(need))
        assert rc == 0, lib.tdx_last_error()
        assert need.value <= lib.tdx_init_workspace_bytes(len(descs))
        return need.value

    base = 0x7F0000000000  # never dereferenced: prepare does not touch the device
    # one huge tensor (90 G bf16 elements = 180 GB): the grab cap grows so that the list stays bounded
    big = prepare([C.make_desc(base, dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=90 * (1 << 30), seed=1, offset=0,
                               p0=0.0, p1=0.02)])
    assert big < 400 << 10
    # every table family at once (normal / uniform x bf16 / f16 x with / without epilogue), 700 descriptors each
    epi = [(C.TDX_EPI_MUL, 0.5)]
    descs = []
    for dt in (C.TDX_BF16, C.TDX_F16):
        for src in (C.TDX_SRC_NORMAL, C.TDX_SRC_UNIFORM):
            for e in ([], epi):
                for i in range(700):
                    descs.append(C.make_desc(base + 4096 * len(descs), dtype=dt, src=src,
                                             elem_count=(1 << 18) + 8 * (i % 5) + (1 << 20) * (i % 3), seed=7,
                                             offset=16 * len(descs), p0=0.0 if src == C.TDX_SRC_NORMAL else -1.0,
                                             p1=0.02 + 0.001 * (i % 7), epi=e))
    many = prepare(descs)
    assert many > len(descs) * 128  # the table is in there
    # a Llama-3-8B-like mix: 291 descriptors, a few sizes
    llama = []
    for layer in range(32):
        for n in (4096 * 4096, 1024 * 4096, 1024 * 4096, 4096 * 4096, 14336 * 4096, 14336 * 4096, 4096 * 14336):
            llama.append(C.make_desc(base, dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=n, seed=3,
                                     offset=64 * len(llama), p0=0.0, p1=0.02))
    llama += [C.make_desc(base, dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=128256 * 4096, seed=3, offset=1 << 30,
                          p0=0.0, p1=0.02)] * 2
    assert 40 << 10 < prepare(llama) < 400 << 10  # (291 descriptors x 128 B + a work list of ~1000 grabs)
    # nothing to do
    assert prepare([C.make_desc(base, dtype=C.TDX_F32, src=C.TDX_SRC_NORMAL, elem_count=0, seed=1, offset=0)]) >= 0
    # submit without a device must fail cleanly, not crash (there is no GPU in the CPU test run)
    need = ctypes.c_size_t(0)
    arr = (C.TdxInitDesc * 1)(llama[0])
    assert lib.tdx_init_prepare(arr, 1, ctypes.byref(need)) == 0 and need.value > 0
    assert lib.tdx_init_submit(None, 0, None) != 0


def test_oracle_iota_matches_torch_on_the_cpu():
    """TDX_SRC_IOTA in the CPU restatement: arange exactly, the rotary inv_freq program to fp32 rounding."""
    import numpy as np
    import torch

    n = 64
    d = C.make_desc(0, dtype=C.TDX_I64, src=C.TDX_SRC_IOTA, elem_begin=5, elem_count=n, p0=-4, p1=3)
    assert np.array_equal(O.generate(d).view(np.int64), (-4 + 3 * (5 + np.arange(n))))
    epi = [(C.TDX_EPI_MUL, 1.0 / 128), (C.TDX_EPI_RPOW, 500000.0), (C.TDX_EPI_RECIP, 0.0), (C.TDX_EPI_MUL, 1.0)]
    d = C.make_desc(0, dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_count=n, p0=0, p1=2, epi=epi)
    got = torch.from_numpy(O.generate(d).view(np.float32).copy())
    ref = 1.0 / (500000.0 ** (torch.arange(0, 2 * n, 2, dtype=torch.int64).float() / 128))
    torch.testing.assert_close(got, ref, rtol=4 * 2.0 ** -23, atol=0.0)
    # 16-bit outputs (`inv_freq.to(torch.bfloat16)`): the SAME fp32 program, rounded once at the store
    for dt, tdt in ((C.TDX_BF16, torch.bfloat16), (C.TDX_F16, torch.float16)):
        d16 = C.make_desc(0, dtype=dt, src=C.TDX_SRC_IOTA, elem_count=n, p0=0, p1=2, epi=epi)
        got16 = torch.from_numpy(O.generate(d16).view(np.int16).copy())
        assert torch.equal(got16, got.to(tdt).view(torch.int16))


@pytest.mark.parametrize("dtype", [C.TDX_F32, C.TDX_BF16, C.TDX_F16])
def test_clamp_keeps_a_nan(dtype):
    """`uniform_(-2, 2).erfinv_().clamp_(-1, 1)`: erfinv of |x| > 1 is NaN, and ATen's clamp_ returns a
    NaN input unchanged -- it does not become the lower bound."""
    kw = dict(dtype=dtype, src=C.TDX_SRC_UNIFORM, elem_count=4096, seed=8, offset=4, p0=-2.0, p1=2.0)
    raw = O.generate(C.make_desc(0, **kw))
    out = O.generate(C.make_desc(0, epi=[(C.TDX_EPI_ERFINV,), (C.TDX_EPI_CLAMP, -1.0, 1.0)], **kw))
    for lo, hi in ((-1.0, math.inf), (-math.inf, 1.0)):  # clamp_(min=) and clamp_(max=)
        one = O.generate(C.make_desc(0, epi=[(C.TDX_EPI_ERFINV,), (C.TDX_EPI_CLAMP, lo, hi)], **kw))
        assert np.array_equal(np.isnan(_floats(one, dtype)), np.isnan(_floats(out, dtype)))
    x, y = _floats(raw, dtype), _floats(out, dtype)
    outside = np.abs(x) > 1
    assert 1000 < outside.sum() < 3000
    assert np.isnan(y[outside]).all() and not np.isnan(y[~outside]).any()
    assert (np.abs(y[~outside]) <= 1).all()


def _floats(bits, dtype):
    if dtype == C.TDX_F32:
        return bits.view(np.float32).astype(np.float64)
    if dtype == C.TDX_BF16:
        return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return bits.view(np.float16).astype(np.float64)
