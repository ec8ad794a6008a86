"""Descriptors past 2^31 local elements and 4 GiB, on the host: the cases tests/test_large_tensors_gpu.py
launches, and the host side of them that needs no device.

The cases (`family_cases`, `window_cases`, `mixed_table`) are one descriptor of every kernel family row
tests/submission_fuzz.py can build, ATen's stream excepted (its kernels never see a launch of 2^31
elements: planner_eval.cc replays such draws through ATen).  Each crosses 2^31 local elements and 2^32
bytes where its element size allows, starts at a global element that is not a multiple of its vector and
writes to an address that is not 16-byte aligned, so its ragged head and tail lie at large offsets too.

Without a device:
  * every case and the mixed table prepare (tdx_init_prepare, fake addresses) within
    tdx_init_workspace_bytes(n), and route to the row they are named for; their launch counts follow from
    submission_fuzz.route, whose Python integers are exact at any size;
  * the host cut (tdx_init_host_cut) of a 17.6 GB FSDP1 flat shard (rank 0 of 8 of Llama-3-70B in bf16)
    and of a windowed Shard(2) block of a fused-expert weight, through 256 MiB and 1 MiB + 13 of staging:
    the structural checks of tests/test_host_targets_cpu.py, at least ceil(bytes / staging) passes, and
    the first and last 4096 elements of the pieces that hold local elements 2^31 and 2^32, evaluated by
    the C restatement, equal the uncut descriptor there.
"""
import ctypes
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import submission_fuzz as F  # noqa: E402
from oracle import tdx_oracle as O  # noqa: E402
from test_host_targets_cpu import STAGING, check_cut  # noqa: E402
from torchdistx_b200 import _cabi as C  # noqa: E402

U, N = F.U, F.N
DT_NAME = {C.TDX_F32: "f32", C.TDX_BF16: "bf16", C.TDX_F16: "f16"}
SEED = 0x5EED
ARENA, SOURCE = 1 << 44, 1 << 43  # fake addresses (16-byte aligned; nothing is written there)
ANCHOR = 4096

# elements of a large case by element size: past 2^31 elements and 2^32 bytes (8-byte elements: past 2^32
# bytes; the 2^31-element int64 case is LARGE_I64)
ODD = 7
COUNT = {1: (1 << 32) + (1 << 20) + ODD, 2: (1 << 31) + (1 << 20) + ODD, 4: (1 << 31) + (1 << 20) + ODD,
         8: (1 << 29) + (1 << 20) + ODD}
LARGE_I64 = (1 << 31) + (1 << 20) + ODD


class Case:
    """One descriptor at byte `head` of an arena (`head` % 16 != 0 unless `aligned`), with a staged copy
    source of `source_elems` elements for TDX_SRC_GATHER."""

    def __init__(self, name, spec, row, head=None, source_elems=0):
        self.name, self.spec, self.row = name, spec, row
        isz = F.ISZ[spec.kw["dtype"]]
        self.head = isz if head is None else head  # (element-aligned, not 16-byte aligned)
        self.source_elems = source_elems

    @property
    def isz(self):
        return F.ISZ[self.spec.kw["dtype"]]

    @property
    def nbytes(self):
        return self.spec.nbytes

    def desc(self, arena, source=0, **over):
        self.spec.off = self.head
        if self.spec.kw["src"] == C.TDX_SRC_GATHER:
            self.spec.src_off = 0
        return self.spec.desc(arena, source, **over)

    def __repr__(self):
        return self.name


# a global start that is not a multiple of any element's vector (an odd one)
UNALIGNED_BEGIN = (1 << 20) * 3 + 5


def rng_case(r, gen, epi, table, aligned=False, params=None):
    src, dt, algo = gen
    isz = F.ISZ[dt]
    spec = F.rng_spec(r, gen, epi, False, COUNT[isz], [SEED], nolut=not table)
    if params is not None:
        spec.kw["p0"], spec.kw["p1"] = params
    epv = 16 // isz
    spec.kw["elem_begin"] = (1 << 20) * epv * 3 if aligned else UNALIGNED_BEGIN
    row = F.family(spec.kw)
    tag = "lut" if table else "direct"
    name = f"{tag}-{'u' if src == U else 'n'}-{DT_NAME[dt]}-algo{algo}-{epi}" + ("-aligned" if aligned else "")
    if params is not None:
        name += f"-{params[0]}-{params[1]}"
    return Case(name, spec, row, head=0 if aligned else None)


def family_cases():
    """One large descriptor of every non-ATen, non-window family row, with variants inside some rows:
    vector-aligned starts, mirrored and unmirrored tables, every fill width, broadcast index programs."""
    r = np.random.default_rng(31)
    out = []
    for gen in F.GENERATORS:
        for epi in ("none", "basic", "ext"):
            out.append(rng_case(r, gen, epi, table=False))
        # (the vector-aligned start and destination: the direct kernels' hot path at large offsets)
        out.append(rng_case(r, gen, "none", table=False, aligned=True))
    for row in F.LUT_ROWS:
        gen, epi = (row[1], row[2], row[3]), row[4]
        if row[1] == N and epi == "none":
            # mirrored (mean +0, std != 0, no epilogue) and unmirrored
            out.append(rng_case(r, gen, epi, table=True, params=(0.0, 0.02)))
            out.append(rng_case(r, gen, epi, table=True, params=(1.5, 0.25)))
            out.append(rng_case(r, gen, epi, table=True, aligned=True, params=(0.0, 0.02)))
        else:
            out.append(rng_case(r, gen, epi, table=True))
    for dt, bits in ((C.TDX_RAW8, 0xA5), (C.TDX_RAW16, 0x3F80), (C.TDX_RAW32, 0x8000_0001),
                     (C.TDX_RAW64, 0x0123_4567_89AB_CDEF)):
        isz = F.ISZ[dt]
        out.append(Case(f"fill-{isz * 8}", F.Spec(dict(dtype=dt, src=C.TDX_SRC_CONST, elem_count=COUNT[isz],
                                                       fill_bits=bits, fill_itemsize=isz)), ("fill",)))
    iota = lambda dt, n, **kw: F.Spec(dict(dtype=dt, src=C.TDX_SRC_IOTA, elem_count=n, elem_begin=5, **kw))
    out.append(Case("iota-f32", iota(C.TDX_F32, COUNT[4], p0=-3.0, p1=1.0, epi=[(C.TDX_EPI_MUL, 0.5)]), ("iota",)))
    out.append(Case("iota-bf16", iota(C.TDX_BF16, COUNT[2], p0=2.0, p1=1.0), ("iota",)))
    out.append(Case("iota-i64", iota(C.TDX_I64, COUNT[8], p0=-9.0, p1=3.0), ("iota",)))
    out.append(Case("iota-f32-broadcast", iota(C.TDX_F32, COUNT[4], p0=1.0, p1=1.0, iota_period=4099, iota_repeat=3,
                                               epi=[(C.TDX_EPI_MUL, 0.25)]), ("iota+ext",)))
    out.append(Case("iota-bf16-broadcast", iota(C.TDX_BF16, COUNT[2], p0=0.0, p1=2.0, iota_period=257, iota_repeat=0),
                    ("iota+ext",)))
    half = 256
    out.append(Case("sincos-bf16", F.Spec(dict(dtype=C.TDX_BF16, src=C.TDX_SRC_SINCOS, elem_count=COUNT[2], p0=0.0,
                                               p1=1.0, sincos_half=half, elem_begin=3,
                                               epi=[(C.TDX_EPI_MUL, -math.log(10000.0) / half), (C.TDX_EPI_EXP,)])),
                    ("sincos",)))
    n = 65537
    out.append(Case("band-bool-65537", F.Spec(dict(dtype=C.TDX_RAW8, src=C.TDX_SRC_BAND, elem_count=n * n, band_rows=n,
                                                   band_cols=n, band_lo=-n, band_hi=0, band_in=1, band_out=0,
                                                   elem_begin=5)), ("band",)))
    n = 46341  # (46341^2 > 2^31)
    out.append(Case("band-bf16-46341", F.Spec(dict(dtype=C.TDX_BF16, src=C.TDX_SRC_BAND, elem_count=n * n,
                                                   band_rows=n, band_cols=n, band_lo=-3, band_hi=5, band_in=0x3F80,
                                                   band_out=0xFF80, elem_begin=3)), ("band",)))
    period = 4099
    out.append(Case("gather-bf16-periodic", F.Spec(dict(dtype=C.TDX_BF16, src=C.TDX_SRC_GATHER, elem_count=COUNT[2],
                                                        gather_period=period, gather_repeat=3, elem_begin=11,
                                                        epi=[(C.TDX_EPI_MUL, 0.5)])), ("gather",),
                    source_elems=period))
    return out


def large_i64_cases():
    """Past 2^31 elements of 8 bytes (16 GiB): the int64 index program and the 64-bit fill."""
    return [Case("iota-i64-2^31", F.Spec(dict(dtype=C.TDX_I64, src=C.TDX_SRC_IOTA, elem_count=LARGE_I64, elem_begin=5,
                                              p0=-9.0, p1=3.0)), ("iota",)),
            Case("fill-64-2^31", F.Spec(dict(dtype=C.TDX_RAW64, src=C.TDX_SRC_CONST, elem_count=LARGE_I64,
                                             fill_bits=0xFEDC_BA98_7654_3210, fill_itemsize=8)), ("fill",))]


MAVERICK_W, MAVERICK_P = 8192, 16384  # Shard(2) of a [128, 5120, 16384] fused-expert weight at TP = 2


def window_case(r, gen, epi, path, count=None):
    """A windowed descriptor of > 2^31 local elements: on the whole-vector path (Maverick's geometry, rank 1,
    16-byte aligned) or on the element path (W not a multiple of the vector, an odd start, an unaligned
    destination)."""
    src, dt, algo = gen
    isz = F.ISZ[dt]
    count = count or COUNT[isz]
    spec = F.rng_spec(r, gen, epi, True, count, [SEED], nolut=False)
    if path == "whole":
        w, p, begin, head = MAVERICK_W, MAVERICK_P, MAVERICK_W, 0
    else:
        w, p = 8191, 16387
        begin, head = 3 * p + 5, isz
    spec.kw.update(window_width=w, window_pitch=p, elem_begin=begin)
    name = f"window-{'u' if src == U else 'n'}-{DT_NAME[dt]}-algo{algo}-{epi}-{path}"
    return Case(name, spec, F.family(spec.kw), head=head)


def window_cases():
    r = np.random.default_rng(32)
    return [window_case(r, gen, epi, path) for gen in F.GENERATORS for epi in ("none", "ext")
            for path in ("whole", "element")]


def huge_window_case():
    """A bf16 block of more than 2^31 vectors (32 GiB): the only launch whose tiles start past 2^31 local
    vectors, where the window kernel divides in 64 bits."""
    r = np.random.default_rng(33)
    return window_case(r, (N, C.TDX_BF16, C.TDX_ALGO_ICDF16), "none", "whole", count=(1 << 34) + (1 << 20) + ODD)


def mixed_table():
    """One submission: a direct fp32 uniform with an epilogue and a bf16 Shard(2) window (two families of
    > 2^31 elements), a table-kernel bf16 normal of > 2^31 elements, and small riders: a fill and an index
    program (they ride in the table kernel's work list), a rotary inv_freq program and a band mask.
    Returns the specs with their byte offsets in one arena."""
    r = np.random.default_rng(34)
    a = F.rng_spec(r, (U, C.TDX_F32, 0), "basic", False, COUNT[4], [SEED], nolut=True)
    a.kw.update(elem_begin=UNALIGNED_BEGIN, p0=-0.5, p1=0.5, epi=[(C.TDX_EPI_MUL, 2.0), (C.TDX_EPI_ADD, 1.0)])
    b = window_case(r, (N, C.TDX_BF16, C.TDX_ALGO_ICDF16), "none", "whole").spec
    c = F.rng_spec(r, (N, C.TDX_BF16, C.TDX_ALGO_ICDF16), "none", False, COUNT[2], [0x1234_5678_9ABC_DEF0], nolut=False)
    c.kw.update(elem_begin=UNALIGNED_BEGIN, p0=0.0, p1=0.02)
    riders = [F.Spec(dict(dtype=C.TDX_RAW32, src=C.TDX_SRC_CONST, elem_count=100_003, fill_bits=0x3F80_0000,
                          fill_itemsize=4)),
              F.Spec(dict(dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_count=50_001, p0=0.0, p1=1.0,
                          epi=[(C.TDX_EPI_MUL, 0.5)])),
              F.Spec(dict(dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_count=64, p0=0.0, p1=2.0,
                          epi=[(C.TDX_EPI_MUL, -math.log(500000.0) / 128), (C.TDX_EPI_EXP,)])),
              F.Spec(dict(dtype=C.TDX_RAW8, src=C.TDX_SRC_BAND, elem_count=2048 * 2048, band_rows=2048,
                          band_cols=2048, band_lo=-2048, band_hi=0, band_in=1, band_out=0))]
    specs = [a, b, c] + riders
    cur = 3
    for s in specs:
        isz = F.ISZ[s.kw["dtype"]]
        cur = -(-cur // isz) * isz
        if s is b:
            cur = -(-cur // 16) * 16  # (the window on its whole-vector path)
        elif cur % 16 == 0:  # (the rest off 16-byte alignment)
            cur += isz
        s.off = cur
        cur += s.nbytes
    return specs, cur + 64


# ---- without a device ------------------------------------------------------------------------------

def prepare(descs):
    lib = C.load()
    arr = (C.TdxInitDesc * len(descs))(*descs)
    need = ctypes.c_size_t(0)
    rc = lib.tdx_init_prepare(arr, len(descs), ctypes.byref(need))
    assert rc == 0, lib.tdx_last_error().decode()
    assert 0 < need.value <= lib.tdx_init_workspace_bytes(len(descs)), need.value
    return int(need.value)


ALL = family_cases() + large_i64_cases() + window_cases() + [huge_window_case()]


def test_every_large_case_crosses_2_to_31_elements_and_4_gib():
    for c in ALL:
        n = c.spec.count
        assert n * c.isz > (1 << 32), c
        assert n > (1 << 31) or c.isz == 8, c
        assert c.head % 16 or "aligned" in c.name or c.name.endswith("-whole"), c
    # every non-ATen family row has a case
    rows = {c.row for c in ALL}
    want = {row for row in F.ROW_ORDER if row[0] != "aten"}
    assert want <= rows, want - rows


@pytest.mark.parametrize("case", ALL, ids=repr)
def test_large_cases_prepare_and_route(case):
    assert F.route([case.spec]) == [case.row] and F.launches([case.spec]) == 1, (case, F.route([case.spec]))
    prepare([case.desc(ARENA, SOURCE)])
    # (the pieces the GPU test compares against: small, on the direct kernel where the family has one)
    alone = F.alone(case.spec)
    assert F.family(alone.kw)[0] != "lut"


def test_the_mixed_table_prepares_and_routes():
    specs, _ = mixed_table()
    fam = F.route(specs)
    lut = ("lut", N, C.TDX_BF16, C.TDX_ALGO_ICDF16, "none")
    assert fam[2] == lut and fam[3] == lut and fam[4] == lut, fam  # (the fill and the index program ride)
    assert fam[0][0] == "direct" and fam[1][0] == "window" and fam[5] == ("iota+ext",) and fam[6] == ("band",)
    assert F.launches(specs) == 5
    prepare([s.desc(ARENA) for s in specs])


# ---- the host cut at these sizes -------------------------------------------------------------------

LLAMA3_70B = dict(vocab=128256, hidden=8192, inter=28672, layers=80, heads=64, kv_heads=8)


def flat_shard_table(rank=0, world=8, align=8):
    """The descriptors of FSDP1's flat shard of Llama-3-70B in bf16 (HF parameter order, `align_numel`
    gaps as zero fills): rank `rank` of `world`, 17.6 GB for rank 0 of 8.  Normals of std 0.02, norms
    filled with ones; one seed, consecutive offsets."""
    m = LLAMA3_70B
    h, kv = m["hidden"], m["hidden"] // m["heads"] * m["kv_heads"]
    params = [("normal", m["vocab"] * h)]
    for _ in range(m["layers"]):
        params += [("normal", h * h), ("normal", kv * h), ("normal", kv * h), ("normal", h * h),
                   ("normal", m["inter"] * h), ("normal", m["inter"] * h), ("normal", h * m["inter"]), ("ones", h),
                   ("ones", h)]
    params += [("ones", h), ("normal", m["vocab"] * h)]
    starts, cur = [], 0
    for _, n in params:
        cur = -(-cur // align) * align
        starts.append(cur)
        cur += n
    chunk = -(-cur // world)
    lo, hi = rank * chunk, min((rank + 1) * chunk, cur)
    descs, offset = [], 0
    for (kind, n), s in zip(params, starts):
        a, b = max(s, lo), min(s + n, hi)
        offset += 4 * (-(-n // 4))  # (each draw's own slice of the stream)
        if a >= b:
            continue
        dst = ARENA + (a - lo) * 2
        if kind == "normal":
            descs.append(C.make_desc(dst, dtype=C.TDX_BF16, src=N, elem_count=b - a, elem_begin=a - s, seed=SEED,
                                     offset=offset, p0=0.0, p1=0.02))
        else:
            descs.append(C.make_desc(dst, dtype=C.TDX_BF16, src=C.TDX_SRC_CONST, elem_count=b - a, fill_bits=0x3F80,
                                     fill_itemsize=2))
    return descs, (hi - lo) * 2


def sub_desc(d, x, k):
    """The descriptor of local elements [x, x + k) of `d` (a window: whole runs shifted into elem_begin,
    then the elements of the last run before x kept and dropped again by `evaluate_sub`)."""
    e = C.TdxInitDesc.from_buffer_copy(d)
    isz = F.ISZ[d.dtype]
    e.dst = (d.dst or 0) + x * isz
    if d.reserved & C.TDX_FLAG_WINDOW:
        w, p = int(d.fill_bits[0]), int(d.fill_bits[1])
        e.elem_begin = d.elem_begin + (x // w) * p
        e.elem_count = x % w + k
        return e, x % w
    if d.src != C.TDX_SRC_CONST:
        e.elem_begin = d.elem_begin + x
    e.elem_count = k
    return e, 0


def evaluate_sub(d, x, k):
    e, skip = sub_desc(d, x, k)
    isz = F.ISZ[d.dtype]
    return O.generate(e).view(np.uint8)[skip * isz:]


def check_pieces_at_large_offsets(descs, staging):
    pieces, passes = check_cut(descs, staging)
    total = sum(int(d.elem_count) * F.ISZ[d.dtype] for d in descs)
    assert passes >= -(-total // staging), (passes, total, staging)
    checked = 0
    for i, d in enumerate(descs):
        for local in (1 << 31, 1 << 32):
            if local >= d.elem_count:
                continue
            p = next(q for q in pieces if q.desc == i and q.elem_first <= local < q.elem_first + q.elem_count)
            isz = F.ISZ[d.dtype]
            parts = C.piece_descs(d, p, STAGING)
            assert sum(int(x.elem_count) for x in parts) == p.elem_count
            # the piece's own descriptors, evaluated over their first and last elements, in local order
            k = min(ANCHOR, p.elem_count)
            for x0 in sorted({0, p.elem_count - k}):
                got, at = [], 0
                for x in parts:
                    n = int(x.elem_count)
                    a, b = max(x0, at), min(x0 + k, at + n)
                    if a < b:
                        got.append(evaluate_sub(x, a - at, b - a))
                    at += n
                got = np.concatenate(got)
                want = evaluate_sub(d, p.elem_first + x0, k)
                assert got.size == k * isz and np.array_equal(got, want), (i, local, x0, staging)
                checked += 1
    return checked


@pytest.mark.parametrize("staging", [256 << 20, (1 << 20) + 13])
def test_the_host_cut_of_a_17_gb_flat_shard(staging):
    descs, nbytes = flat_shard_table()
    assert nbytes > 17_500_000_000 and sum(int(d.elem_count) for d in descs) > (1 << 33)
    # (descriptors of > 2^31 elements: the embedding's 1.05e9 is below; the cut's offsets are not)
    assert check_pieces_at_large_offsets(descs, staging) == 0
    # the pieces at flat element 2^31 and 2^32 of the shard: a descriptor of the whole shard's span
    whole = C.make_desc(ARENA + 2, dtype=C.TDX_BF16, src=N, elem_count=nbytes // 2, elem_begin=3, seed=SEED,
                        offset=16, p0=0.0, p1=0.02)
    assert check_pieces_at_large_offsets([whole], staging) == 4


@pytest.mark.parametrize("staging", [256 << 20, (1 << 20) + 13])
def test_the_host_cut_of_a_windowed_fused_expert_block(staging):
    """Rank 1's Shard(2) block of Llama-4 Maverick's [128, 5120, 16384] experts at TP = 2: 5.4e9 elements."""
    d = C.make_desc(ARENA, dtype=C.TDX_BF16, src=N, elem_count=128 * 5120 * MAVERICK_W, elem_begin=MAVERICK_W,
                    seed=SEED, offset=64, p0=0.0, p1=0.02, flags=C.TDX_FLAG_WINDOW)
    d.fill_bits[0], d.fill_bits[1] = MAVERICK_W, MAVERICK_P
    e = C.make_desc(ARENA + 2 * d.elem_count + 4, dtype=C.TDX_F32, src=U, elem_count=COUNT[4], elem_begin=16387 * 3 + 5,
                    seed=SEED, offset=8, p0=-1.0, p1=1.0, flags=C.TDX_FLAG_WINDOW, epi=[(C.TDX_EPI_MUL, 0.5)])
    e.fill_bits[0], e.fill_bits[1] = 8191, 16387
    assert check_pieces_at_large_offsets([d, e], staging) == 6  # (e: 2^31 only)
