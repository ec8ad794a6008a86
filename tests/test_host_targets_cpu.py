"""Host destinations without a device: the cut tdx_init_submit_host makes of a descriptor table.

The tables are tests/submission_fuzz.py's (every source kind, dtype, epilogue class, window and ATen
stream), cut for staging buffers from the smallest the library accepts up to a few MiB, odd sizes
included.  For every cut:
  * the pieces of each descriptor cover its local elements exactly once, in order;
  * every pass's pieces fit in the staging buffer, apart, above the plan workspace the pass's table
    needs (laid out by tdx_init_prepare);
  * each piece sits at its destination's address mod 16;
  * on tables shrunk to a few thousand elements per descriptor, the pieces' descriptors, evaluated by the
    C restatement (oracle/tdx_oracle.c; ATen's stream: its unit draws) and concatenated, equal the uncut
    descriptor byte for byte.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import submission_fuzz as F  # noqa: E402
from oracle import tdx_oracle as O  # noqa: E402
from torchdistx_b200 import _cabi as C  # noqa: E402

HOST = 0x7F00_0000_0000  # where the fake host arena starts (16-byte aligned; nothing is written there)
STAGING = 0x7E00_0000_0000


def min_staging(descs) -> int:
    """The smallest staging buffer the library accepts for the table (found by bisection)."""
    lo, hi = 16, 1 << 16
    while lo < hi:
        mid = (lo + hi) // 2
        try:
            C.host_cut(descs, mid)
            hi = mid
        except RuntimeError as e:
            assert "staging buffer smaller" in str(e), e
            lo = mid + 1
    return lo


def check_cut(descs, staging_bytes):
    """The structural properties of one cut; returns (pieces, passes)."""
    pieces, passes = C.host_cut(descs, staging_bytes)
    covered = [0] * len(descs)
    by_pass = {}
    for p in pieces:
        d = descs[p.desc]
        isz = F.ISZ[d.dtype]
        assert p.elem_count > 0 and p.elem_first == covered[p.desc], (p.desc, p.elem_first, covered[p.desc])
        covered[p.desc] += p.elem_count
        assert (p.staging_off - (d.dst + p.elem_first * isz)) % 16 == 0
        assert p.staging_off + p.elem_count * isz <= staging_bytes
        by_pass.setdefault(p.pass_, []).append(p)
    assert covered == [int(d.elem_count) for d in descs]
    assert sorted(by_pass) == list(range(passes))
    assert [p.pass_ for p in pieces] == sorted(p.pass_ for p in pieces)
    for q, ps in by_pass.items():
        spans = sorted((p.staging_off, p.staging_off + p.elem_count * F.ISZ[descs[p.desc].dtype]) for p in ps)
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), f"pass {q}: pieces overlap"
        table = [x for p in ps for x in C.piece_descs(descs[p.desc], p, STAGING)]
        ws = C.prepare(table)
        assert ws <= spans[0][0], f"pass {q}: a workspace of {ws} bytes reaches the piece at {spans[0][0]}"
    return pieces, passes


@pytest.mark.parametrize("seed", range(2))
def test_the_cut_of_every_fuzz_table(seed):
    for t in F.tables(seed, forced=seed % 2 == 0, n_random=2):
        descs = t.descs(HOST, 0x1000)
        if not descs or sum(d.elem_count for d in descs) == 0:
            continue
        small = min_staging(descs)
        # (a table of up to 1 GiB: no staging below 3 MiB, or the cut has hundreds of thousands of pieces)
        for staging in ((3 << 20) + 4093, 16 << 20):
            pieces, passes = check_cut(descs, max(staging, small))
            total = sum(int(d.elem_count) * F.ISZ[d.dtype] for d in descs)
            assert passes >= -(-total // staging)


def evaluate(d):
    """What the kernels write for descriptor `d`, as bytes (ATen's stream: the unit draws of its elements)."""
    return (O.aten_units(d) if F.is_aten(dict(algo=int(d.algo))) else O.generate(d)).view(np.uint8)


def shrunk(seed):
    """The seed's tables with every descriptor cut down to at most a few thousand elements."""
    r = np.random.default_rng(50_000 + seed)
    out = []
    for t in F.tables(seed, forced=seed % 2 == 0, n_random=2):
        specs = []
        for s in t.specs:
            w = s.kw.get("window_width") or 0
            hi = 3 * w + 7 if w and w < 1000 else 3000
            specs.append(F._resize(r, s, int(r.integers(1, hi))))
        out.append(F.layout(r, specs, t.name + " shrunk"))
    return out


KEYS = ("philox_seed", "philox_offset", "p0", "p1", "dtype", "src", "n_epi")


@pytest.mark.parametrize("seed", range(2))
def test_pieces_evaluate_to_their_uncut_descriptors(seed):
    r = np.random.default_rng(seed)
    for t in shrunk(seed):
        host_source = r.integers(0, 256, t.source_bytes, dtype=np.uint8)
        descs = t.descs(HOST, host_source.ctypes.data)
        whole = [evaluate(d) for d in descs]
        small = min_staging(descs)
        for staging in (small, small + 16, small + 37, small + 4096 + 5, 1 << 20):
            pieces, _ = check_cut(descs, staging)
            got = [[] for _ in descs]
            for p in pieces:
                d = descs[p.desc]
                parts = C.piece_descs(d, p, STAGING)
                isz = F.ISZ[d.dtype]
                at = STAGING + p.staging_off
                for x in parts:
                    assert x.dst == at, "a piece's descriptors are back to back in local order"
                    at += int(x.elem_count) * isz
                    for k in KEYS:
                        assert getattr(x, k) == getattr(d, k), k
                    assert bytes(x.epi) == bytes(d.epi) and (x.algo, x.reserved & ~C.TDX_FLAG_WINDOW) == \
                        (d.algo, d.reserved & ~C.TDX_FLAG_WINDOW)
                    got[p.desc].append(evaluate(x))
                assert at == STAGING + p.staging_off + p.elem_count * isz
            for i, (d, w) in enumerate(zip(descs, whole)):
                cat = np.concatenate(got[i]) if got[i] else np.empty(0, np.uint8)
                if not np.array_equal(cat, w):
                    bad = int(np.flatnonzero(cat != w)[0])
                    raise AssertionError(f"{t.name}, staging {staging}: descriptor {i} {t.specs[i].kw}: "
                                         f"byte {bad} of the pieces differs from the uncut descriptor")


def test_a_window_cut_inside_its_runs():
    """A Shard(1) window cut inside a run: a partial first run, whole runs (windowed), a partial last run."""
    d = C.make_desc(HOST, dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=10 * 7, elem_begin=3, seed=5, offset=8,
                    p0=0.0, p1=0.02, flags=C.TDX_FLAG_WINDOW)
    d.fill_bits[0], d.fill_bits[1] = 7, 19
    p = C.TdxHostPiece(0, 0, 5, 20, 16 + 10)
    parts = C.piece_descs(d, p, 0)
    assert [(x.elem_begin, x.elem_count, bool(x.reserved & C.TDX_FLAG_WINDOW)) for x in parts] == \
        [(3 + 5, 2, False), (3 + 19, 14, True), (3 + 3 * 19, 4, False)]  # (local 5..6, 7..20, 21..24)
    assert [x.dst for x in parts] == [26, 26 + 2 * 2, 26 + 16 * 2]
    assert (parts[0].fill_bits[0], parts[0].fill_bits[1]) == (0, 0) and (parts[1].fill_bits[0], parts[1].fill_bits[1]) == (7, 19)


def test_refusals_before_any_launch():
    lib = C.load()
    d = C.make_desc(HOST, dtype=C.TDX_F32, src=C.TDX_SRC_UNIFORM, elem_count=1000, seed=1)
    arr = (C.TdxInitDesc * 1)(d)
    n, passes = ctypes.c_int(0), ctypes.c_int(0)
    # a staging buffer below one vector plus a one-descriptor pass's workspace
    assert lib.tdx_init_host_cut(arr, 1, 64, None, 0, ctypes.byref(n), ctypes.byref(passes)) == C.TDX_E_BADARG
    assert b"staging buffer smaller" in lib.tdx_last_error()
    # a descriptor the library refuses anyway
    bad = (C.TdxInitDesc * 1)(C.make_desc(HOST + 2, dtype=C.TDX_F32, src=C.TDX_SRC_UNIFORM, elem_count=4))
    assert lib.tdx_init_host_cut(bad, 1, 1 << 20, None, 0, ctypes.byref(n), ctypes.byref(passes)) == C.TDX_E_BADARG
    assert b"aligned" in lib.tdx_last_error()
    # null and unaligned staging buffers never reach the device
    assert lib.tdx_init_submit_host(arr, 1, None, 1 << 20, None) == C.TDX_E_BADARG
    assert lib.tdx_init_submit_host(arr, 1, 0x1008, 1 << 20, None) == C.TDX_E_BADARG
    assert b"staging" in lib.tdx_last_error()
    # nothing to do is not an error
    assert lib.tdx_init_host_cut(None, 0, 1 << 20, None, 0, ctypes.byref(n), ctypes.byref(passes)) == 0
    assert (n.value, passes.value) == (0, 0)
