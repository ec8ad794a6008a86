"""Seeded descriptor tables that mix the kernel families the way a materialize_module submission does.

`tables(seed)` gives the tables of one seed: a few random mixes plus the forced regimes, the tables just
below and just above every decision the host scheduler (csrc/kernels/tdx_init_host.cu build_plan,
launch_groups) takes from the whole table rather than per descriptor:
  * the table threshold: a 16-bit family takes the table kernel only if its launch holds 2^25 elements
    (2^26 for the uniform); below that, its direct twin;
  * riders: constant fills and index programs join the largest table group when they are at most 1/16 of
    its bytes;
  * the pre-assigned work list: at least 16 table-kernel tiles per SM;
  * static grabs: at most kStaticTilesPerCta (8) tiles per resident CTA of a direct kernel;
  * one descriptor (the inline plan);
  * 47 kernel families (one plan header) and 48 or more (two), and every one of the 80 family rows.

A table is a list of `Spec`s: the arguments of `_cabi.make_desc` without the addresses, and the byte
offset of the destination in one arena.  Destinations are packed back to back at element alignment
(not 16 bytes), after a random head shift and with optional gaps, so neighbours of different families
share 16-byte lines.  Copies read a staged source buffer of their own.

`route(specs)` restates the routing -- family_of, the table threshold and the twin fallback, the rider
rule -- and gives the kernel family of every descriptor; `launches(specs)` the launch count that follows;
`oracle_bits(spec, d)` what the CPU restatement holds a descriptor's first elements to.  Nothing here
needs a GPU.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field, replace
from typing import Dict, List, Optional

import numpy as np

from oracle import tdx_oracle as O
from torchdistx_b200 import _cabi as C

SM = 132  # the host's assumption without a device (H100 SXM); the GPU tests pass the device's own count
MAX_GROUPS = 47  # kernel families one plan header holds
LUT_MIN_LAUNCH = 1 << 25
LUT_MIN_ELEMS = 1 << 18
LUT_TILE_ELEMS = 8192 * 8  # table kernel: 8192 vectors of eight 16-bit elements
LUT_TILE_VECS = 8192
DIRECT16_TILE_ELEMS = 1024 * 8  # 16-bit direct kernels: 1024 vectors
STATIC_TILES_PER_CTA = 8
MAX_TABLE_BYTES = 1 << 30

ISZ = C.ITEMSIZE
U, N = C.TDX_SRC_UNIFORM, C.TDX_SRC_NORMAL
FLOATS = (C.TDX_F32, C.TDX_BF16, C.TDX_F16)
WIDE = C.TDX_ALGO_WIDE32
EXT_OPS = {C.TDX_EPI_EXP, C.TDX_EPI_LOG, C.TDX_EPI_EXPM1, C.TDX_EPI_INV_SOFTPLUS, C.TDX_EPI_MULADD}

# (src, dtype, algo) of the ten generators, as the library resolves them (tdx_init_host.cu resolve_algo)
GENERATORS = [(U, C.TDX_F32, 0), (U, C.TDX_BF16, 0), (U, C.TDX_F16, 0), (N, C.TDX_F32, C.TDX_ALGO_BM32),
              (N, C.TDX_BF16, C.TDX_ALGO_ICDF16), (N, C.TDX_F16, C.TDX_ALGO_ICDF16), (U, C.TDX_BF16, WIDE),
              (U, C.TDX_F16, WIDE), (N, C.TDX_BF16, C.TDX_ALGO_BM32), (N, C.TDX_F16, C.TDX_ALGO_BM32)]
# ATen's stream: (src, dtype, algo) of its eight rows (a wide normal is the native one)
ATEN = [(U, dt, C.TDX_ALGO_ATEN) for dt in FLOATS] + [(U, dt, C.TDX_ALGO_ATEN_WIDE) for dt in FLOATS[1:]] + \
       [(N, dt, C.TDX_ALGO_ATEN) for dt in FLOATS]
# the table kernel's rows, in the library's row order (the rider host is the first of the largest)
LUT_ROWS = [("lut", N, C.TDX_BF16, 1, "none"), ("lut", N, C.TDX_F16, 1, "none"), ("lut", U, C.TDX_BF16, 0, "none"),
            ("lut", U, C.TDX_F16, 0, "none"), ("lut", N, C.TDX_BF16, 1, "basic"), ("lut", N, C.TDX_F16, 1, "basic"),
            ("lut", U, C.TDX_BF16, 0, "basic"), ("lut", U, C.TDX_F16, 0, "basic")]
# every family row of the library, in its order (plans take groups in this order, 47 to a plan)
_GEN_EPI = [("direct",) + g + (e,) for g in GENERATORS for e in ("none", "basic")]
ROW_ORDER = ([("fill",), ("iota",)] + _GEN_EPI + LUT_ROWS + [("iota+ext",)] +
             [("direct",) + g + ("ext",) for g in GENERATORS] + [("sincos",), ("gather",), ("band",)] +
             [("window",) + g + (e,) for g in GENERATORS for e in (False, True)] +
             [("aten",) + g + (e,) for g in ATEN for e in (False, True)])
assert len(ROW_ORDER) == 80 and len(set(ROW_ORDER)) == 80

# parameters: a small pool, so that equal parameters meet (sorting, table reuse); the signed-zero pairs of
# tests/generator_edges.py ZERO_SIGN and normal_(+-0, 0) among them
UNIFORM_PARAMS = [(-0.5, 0.5), (0.0, 1.0), (-0.0, -0.0), (-0.0, 0.0), (-1.0, -1e-3), (0.25, 4.0)]
NORMAL_PARAMS = [(0.0, 0.02), (0.0, 1.0), (-0.0, 0.0), (0.0, 0.0), (1.5, 0.25)]
SEEDS = [0x5EED, 0x1234_5678_9ABC_DEF0, 7]
BASIC = [[(C.TDX_EPI_MUL, 0.5)], [(C.TDX_EPI_ADD, -0.25)], [(C.TDX_EPI_MUL, -0.0)],
         [(C.TDX_EPI_MUL, 2.0), (C.TDX_EPI_ADD, 1.0)], [(C.TDX_EPI_CLAMP, -0.5, 0.5)]]
EXT = [[(C.TDX_EPI_EXP,)], [(C.TDX_EPI_MULADD, 2.0, 1.0)], [(C.TDX_EPI_MUL, 0.5), (C.TDX_EPI_EXPM1,)],
       [(C.TDX_EPI_MULADD, 1.0, -0.0)]]
# uniform over (0, 1) only: the trunc_normal_ chain and the state-space steps that need a positive x
TRUNC = [(C.TDX_EPI_ERFINV,), (C.TDX_EPI_MUL, 0.02 * math.sqrt(2.0)), (C.TDX_EPI_ADD, 0.0), (C.TDX_EPI_CLAMP, -0.04, 0.04)]
POSITIVE_EXT = [[(C.TDX_EPI_LOG,)], [(C.TDX_EPI_INV_SOFTPLUS,)], [(C.TDX_EPI_MUL, 4.0), (C.TDX_EPI_LOG,)]]


@dataclass
class Spec:
    kw: dict  # make_desc arguments, without dst (and without gather_src: `src_off` is its offset)
    off: int = 0  # byte offset of the destination in the arena
    src_off: Optional[int] = None  # copies: byte offset of the source in the staged source buffer

    @property
    def count(self) -> int:
        return self.kw.get("elem_count", 0)

    @property
    def nbytes(self) -> int:
        return self.count * ISZ[self.kw["dtype"]]

    def desc(self, arena: int, source: int = 0, **over) -> "C.TdxInitDesc":
        kw = dict(self.kw, **over)
        if self.src_off is not None:
            kw["gather_src"] = source + self.src_off
        d = C.make_desc(arena + self.off, **kw)
        if kw.get("flags", 0) & C.TDX_FLAG_WINDOW and not is_aten(kw):  # {W, P}
            d.fill_bits[0], d.fill_bits[1] = kw["window_width"], kw["window_pitch"]
        return d


@dataclass
class Table:
    name: str
    specs: List[Spec]
    arena_bytes: int = 0
    source_bytes: int = 0
    sm: int = SM
    tags: List[str] = field(default_factory=list)

    def descs(self, arena: int, source: int = 0):
        return [s.desc(arena, source) for s in self.specs]


# ---- the restatement of the routing ----------------------------------------------------------------

def is_aten(kw) -> bool:
    return kw.get("algo", 0) & 0x0F in (C.TDX_ALGO_ATEN, C.TDX_ALGO_ATEN_WIDE)


def epi_class(kw) -> str:
    if kw["src"] == C.TDX_SRC_IOTA and kw.get("iota_period", 0):
        return "ext"
    steps = kw.get("epi", ())
    if any(st[0] & 0xFF in EXT_OPS for st in steps):
        return "ext"
    return "basic" if steps else "none"


def resolve_algo(kw) -> int:
    src, dt, a = kw["src"], kw["dtype"], kw.get("algo", 0) & 0x0F
    if a in (C.TDX_ALGO_ATEN, C.TDX_ALGO_ATEN_WIDE):
        return a if a == C.TDX_ALGO_ATEN_WIDE and src == U and dt != C.TDX_F32 else C.TDX_ALGO_ATEN
    if src == N:
        return a if a else (C.TDX_ALGO_BM32 if dt == C.TDX_F32 else C.TDX_ALGO_ICDF16)
    return WIDE if src == U and dt != C.TDX_F32 and a == WIDE else 0


def family(kw, table: bool = True) -> tuple:
    """The kernel family a descriptor runs in (tdx_init_host.cu family_of), as a key."""
    src = kw["src"]
    if src == C.TDX_SRC_CONST:
        return ("fill",)
    if src == C.TDX_SRC_IOTA:
        return ("iota+ext",) if epi_class(kw) == "ext" else ("iota",)
    if src in (C.TDX_SRC_SINCOS, C.TDX_SRC_GATHER, C.TDX_SRC_BAND):
        return ({C.TDX_SRC_SINCOS: "sincos", C.TDX_SRC_GATHER: "gather", C.TDX_SRC_BAND: "band"}[src],)
    dt, algo, epi = kw["dtype"], resolve_algo(kw), epi_class(kw)
    if algo in (C.TDX_ALGO_ATEN, C.TDX_ALGO_ATEN_WIDE):  # (one row serves plain ranges and windows)
        return ("aten", src, dt, algo, epi != "none")
    if kw.get("flags", 0) & C.TDX_FLAG_WINDOW:
        return ("window", src, dt, algo, epi != "none")
    key = ("lut", src, dt, algo, epi)
    if table and not kw.get("algo", 0) & C.TDX_ALGO_NOLUT and kw.get("elem_count", 0) >= LUT_MIN_ELEMS and \
            key in LUT_ROWS:
        return key
    return ("direct", src, dt, algo, epi)


def route(specs: List[Spec]) -> List[tuple]:
    """The family of every descriptor of one submission: family_of, then the table threshold over the
    whole launch (a table family below it falls back to its direct twin), then the riders."""
    fam = [family(s.kw) for s in specs]
    lut_elems: Dict[tuple, int] = {}
    for f, s in zip(fam, specs):
        if f[0] == "lut":
            lut_elems[f] = lut_elems.get(f, 0) + s.count
    for i, (f, s) in enumerate(zip(fam, specs)):
        if f[0] == "lut" and lut_elems[f] < LUT_MIN_LAUNCH * (2 if f[1] == U else 1):
            fam[i] = family(s.kw, table=False)
    rides = [f in (("fill",), ("iota",)) for f in fam]
    bytes_of: Dict[tuple, int] = {}
    for f, s in zip(fam, specs):
        bytes_of[f] = bytes_of.get(f, 0) + s.nbytes
    host, host_bytes = None, 0
    for row in LUT_ROWS:
        if row in bytes_of and bytes_of[row] > host_bytes:
            host, host_bytes = row, bytes_of[row]
    ride_bytes = sum(s.nbytes for r, s in zip(rides, specs) if r)
    if any(rides) and host is not None and ride_bytes * 16 <= host_bytes:
        fam = [host if r else f for r, f in zip(rides, fam)]
    return fam


def tiles_of(spec: Spec, dst: int, tile_vecs: int) -> int:
    """Tiles of one descriptor in a group of tile_vecs-vector tiles (tdx_init_host.cu tiles_of); `dst` is
    its destination address (fills and bands count the 16-byte lines they touch)."""
    kw, n = spec.kw, spec.count
    if n == 0:
        return 0
    isz = ISZ[kw["dtype"]]
    epv = 16 // isz
    begin = kw.get("elem_begin", 0)
    if kw["src"] in (C.TDX_SRC_CONST, C.TDX_SRC_BAND):
        end = dst + n * isz
        nvec = (end - (dst & ~15) + 15) // 16
    elif is_aten(kw) and not kw.get("flags", 0) & C.TDX_FLAG_WINDOW:
        S = kw["aten_stride"]
        nvec = 4 * ((begin + n - 1) // (4 * S) - begin // (4 * S) + 1) * (S // epv)
    elif kw["src"] in (C.TDX_SRC_IOTA, C.TDX_SRC_SINCOS, C.TDX_SRC_GATHER) or kw.get("flags", 0) & C.TDX_FLAG_WINDOW:
        nvec = -(-n // epv)
    else:
        nvec = (begin + n - 1) // epv - begin // epv + 1
    return -(-nvec // tile_vecs)


def groups(specs: List[Spec]) -> int:
    """Kernel families of the submission (plan groups, with empty descriptors)."""
    return len(set(route(specs)))


def launches(specs: List[Spec]) -> int:
    """Kernel launches of the submission: one per family with any element to write."""
    return len({f for f, s in zip(route(specs), specs) if s.count})


def alone(spec: Spec) -> Spec:
    """The descriptor for a launch of its own, on the direct kernel where it has one (TDX_ALGO_NOLUT: the
    same bits, by the library's contract)."""
    kw = dict(spec.kw)
    if kw["src"] in (U, N) and resolve_algo(kw) not in (C.TDX_ALGO_ATEN, C.TDX_ALGO_ATEN_WIDE):
        kw["algo"] = kw.get("algo", 0) | C.TDX_ALGO_NOLUT
    return replace(spec, kw=kw)


def oracle_bits(spec: Spec, d) -> Optional[np.ndarray]:
    """The restatement's element bits of the first elements of `d` (`spec`'s descriptor, cut short), or
    None where no bar applies."""
    kw = spec.kw
    if is_aten(kw):  # (its unit uniform draws only)
        if kw["src"] != U or kw["dtype"] != C.TDX_F32 or kw.get("epi") or (kw["p0"], kw["p1"]) != (0.0, 1.0):
            return None
        return O.aten_units(d).view(np.uint32)
    if kw["src"] == C.TDX_SRC_SINCOS or (kw["src"] == N and kw.get("epi")):
        # (sincos: its restatement's bar grows with the row index -- held bit for bit to ATen's CUDA
        # construction in tests/test_sincos_tables_gpu.py; a normal through an epilogue carries the
        # generator's ulp into every step -- held to ATen on the same draws in tests/test_epilogue_aten_gpu.py)
        return None
    return O.generate(d)


# ---- drawing descriptors ---------------------------------------------------------------------------

def _pick(r: np.random.Generator, seq):
    return seq[int(r.integers(len(seq)))]


def _epb(kw) -> int:
    return 4 if kw["dtype"] == C.TDX_F32 or resolve_algo(kw) == WIDE or \
        (kw["src"] == N and resolve_algo(kw) == C.TDX_ALGO_BM32) else 8


def _size(r: np.random.Generator, hi: int) -> int:
    """Log-uniform over [0, hi] elements (0 now and then)."""
    if hi <= 0 or r.random() < 0.04:
        return 0
    return int(min(hi, math.floor(math.exp(r.uniform(0.0, math.log(hi + 1))))))


def _begin(r: np.random.Generator, kw, count: int, limit: int = 1 << 62) -> int:
    """0, a random start, or one that crosses the 2^32-block boundary of the Philox counter."""
    u = r.random()
    if u < 0.4:
        return 0
    if u < 0.7 or limit < (1 << 36):
        return int(r.integers(0, max(1, min(limit - count, 1 << 30))))
    edge = (1 << 32) * _epb(kw)
    return edge - int(r.integers(1, max(2, min(count, 1 << 16) + 1)))


def rng_spec(r: np.random.Generator, gen, epi_kind: str, window: bool, count: int, seeds, nolut=None) -> Spec:
    src, dt, algo = gen
    p0, p1 = _pick(r, UNIFORM_PARAMS if src == U else NORMAL_PARAMS)
    if epi_kind == "none":
        epi = []
    elif epi_kind == "basic":
        epi = list(_pick(r, BASIC + ([TRUNC] if src == U else [])))
    else:
        epi = list(_pick(r, EXT + (POSITIVE_EXT if src == U else [])))
    if src == U and epi and (epi == TRUNC or epi in POSITIVE_EXT):
        p0, p1 = (0.0, 1.0) if epi != TRUNC else (2 * 0.0227501 - 1, 2 * 0.9772499 - 1)
    kw = dict(dtype=dt, src=src, algo=algo, elem_count=count, seed=_pick(r, seeds), p0=p0, p1=p1, epi=epi,
              offset=4 * int(r.integers(0, 1 << 20)))
    aten = algo in (C.TDX_ALGO_ATEN, C.TDX_ALGO_ATEN_WIDE)
    if not aten and (r.random() < 0.25 if nolut is None else nolut):
        kw["algo"] = algo | C.TDX_ALGO_NOLUT
    if window:
        w = int(r.integers(1, 4097))
        pitch = w + int(r.integers(0, 3 * w + 1))
        kw.update(flags=C.TDX_FLAG_WINDOW, window_width=w, window_pitch=pitch)
    if aten:  # ATen's grid stride; every global element below 2^31
        kw["aten_stride"] = 256 * _pick(r, [1, 37, 132 * 8, 4096])
        span = ((count - 1) // kw["window_width"]) * kw["window_pitch"] + kw["window_width"] if window and count \
            else count
        kw["elem_begin"] = int(r.integers(0, max(1, (1 << 31) - span))) if r.random() < 0.5 else 0
        if not window:
            kw["window_width"] = kw["window_pitch"] = 0
    else:
        kw["elem_begin"] = _begin(r, kw, count)
    return Spec(kw)


def det_spec(r: np.random.Generator, kind: str, count: int) -> Spec:
    if kind == "fill":
        dt = _pick(r, [C.TDX_F32, C.TDX_BF16, C.TDX_F16, C.TDX_RAW8, C.TDX_RAW16, C.TDX_RAW32, C.TDX_RAW64])
        isz = ISZ[dt]
        bits = _pick(r, [0, (1 << (8 * isz)) - 1, 0x3F80_0000 & ((1 << (8 * isz)) - 1), 1 << (8 * isz - 1),
                         int(r.integers(0, 1 << min(8 * isz, 62)))])
        return Spec(dict(dtype=dt, src=C.TDX_SRC_CONST, elem_count=count, fill_bits=bits, fill_itemsize=isz))
    if kind in ("iota", "iota+ext"):
        if kind == "iota" and r.random() < 0.3:
            return Spec(dict(dtype=C.TDX_I64, src=C.TDX_SRC_IOTA, elem_count=count, p0=float(r.integers(-9, 9)),
                             p1=float(r.integers(0, 4)), elem_begin=int(r.integers(0, 1 << 20))))
        dt = _pick(r, FLOATS)
        kw = dict(dtype=dt, src=C.TDX_SRC_IOTA, elem_count=count, p0=float(r.integers(-4, 5)), p1=1.0,
                  elem_begin=int(r.integers(0, 64)))
        if kind == "iota":
            kw["epi"] = _pick(r, [[], [(C.TDX_EPI_MUL, 0.5)], [(C.TDX_EPI_MUL, 2.0), (C.TDX_EPI_ADD, -1.0)]])
        elif r.random() < 0.5:  # broadcast geometry
            kw.update(iota_period=int(r.integers(1, 300)), iota_repeat=int(r.integers(0, 5)),
                      epi=_pick(r, [[], [(C.TDX_EPI_MUL, 0.25)]]))
        else:
            kw.update(p0=1.0, epi=_pick(r, [[(C.TDX_EPI_LOG,)], [(C.TDX_EPI_MUL, -0.01), (C.TDX_EPI_EXP,)]]))
        return Spec(kw)
    if kind == "sincos":
        half = int(r.integers(1, 257))
        return Spec(dict(dtype=_pick(r, FLOATS), src=C.TDX_SRC_SINCOS, elem_count=count, p0=0.0, p1=1.0,
                         sincos_half=half, sincos_cos_first=bool(r.random() < 0.3),
                         epi=[(C.TDX_EPI_MUL, -math.log(10000.0) / half), (C.TDX_EPI_EXP,)],
                         elem_begin=int(r.integers(0, 4 * half))))
    if kind == "band":
        dt = _pick(r, list(ISZ))
        isz = ISZ[dt]
        cols, rows = int(r.integers(1, 300)), int(r.integers(1, 300))
        lo = int(r.integers(-rows, cols + 1))
        hi = int(r.integers(lo, cols + 1))
        full = (1 << (8 * isz)) - 1
        return Spec(dict(dtype=dt, src=C.TDX_SRC_BAND, elem_count=count, band_rows=rows, band_cols=cols,
                         band_lo=lo, band_hi=hi, band_in=_pick(r, [1, full, 0x3F80 & full]),
                         band_out=_pick(r, [0, full & ~0x7, 0xFF80 & full]), elem_begin=int(r.integers(0, 1 << 20))))
    if kind == "gather":
        dt = _pick(r, [C.TDX_F32, C.TDX_BF16, C.TDX_F16, C.TDX_I64])
        kw = dict(dtype=dt, src=C.TDX_SRC_GATHER, elem_count=count)
        if dt != C.TDX_I64 and r.random() < 0.4:
            kw["epi"] = _pick(r, [[(C.TDX_EPI_MUL, 0.5)], [(C.TDX_EPI_EXP,)]])
        if r.random() < 0.5:
            kw.update(gather_period=int(r.integers(1, 500)), gather_repeat=int(r.integers(0, 4)),
                      elem_begin=int(r.integers(0, 1 << 20)))
        else:
            kw["elem_begin"] = int(r.integers(0, 64))
        return Spec(kw)
    raise ValueError(kind)


DET_KINDS = ["fill", "iota", "iota+ext", "sincos", "band", "gather"]


def every_key(r: np.random.Generator, count: int, seeds) -> List[Spec]:
    """One descriptor of every combination the ABI accepts: the deterministic sources, and (src, dtype,
    algo) x epilogue class x window for the generators and ATen's stream."""
    out = [det_spec(r, k, count) for k in DET_KINDS]
    for gen in GENERATORS + ATEN:
        for epi in ("none", "basic", "ext"):
            for window in (False, True):
                out.append(rng_spec(r, gen, epi, window, count, seeds, nolut=False))
    return out


# ---- tables ----------------------------------------------------------------------------------------

def layout(r: np.random.Generator, specs: List[Spec], name: str, sm: int = SM, tags=()) -> Table:
    """Packs the destinations back to back at element alignment after a random head shift, with gaps now
    and then, and stages the copies' sources."""
    cur = int(r.integers(0, 16))
    src_cur = 0
    for s in specs:
        isz = ISZ[s.kw["dtype"]]
        if r.random() < 0.3:
            cur += int(r.integers(1, 40))
        cur = -(-cur // isz) * isz
        s.off = cur
        cur += s.nbytes
        if s.kw["src"] == C.TDX_SRC_GATHER:
            need = s.kw.get("gather_period") or (s.kw.get("elem_begin", 0) + s.count)
            src_cur = -(-src_cur // 16) * 16
            s.src_off = src_cur
            src_cur += max(need, 1) * isz
    t = Table(name, specs, arena_bytes=cur + 64, source_bytes=src_cur + 64, sm=sm, tags=list(tags))
    assert t.arena_bytes <= MAX_TABLE_BYTES + 4096, (name, t.arena_bytes)
    return t


def random_table(r: np.random.Generator, name: str, sm: int = SM, budget: int = 64 << 20) -> Table:
    seeds = SEEDS[:1] if r.random() < 0.5 else SEEDS
    n = int(r.integers(1, 40))
    specs, used = [], 0
    for _ in range(n):
        u = r.random()
        if u < 0.3:
            kind = _pick(r, DET_KINDS)
            cap = {"sincos": 1 << 20, "gather": 1 << 18, "band": 1 << 22}.get(kind, 1 << 27)
            spec = det_spec(r, kind, 0)
        else:
            gen = _pick(r, GENERATORS if u < 0.8 else ATEN)
            spec = rng_spec(r, gen, _pick(r, ["none", "basic", "ext"]), r.random() < 0.25, 0, seeds)
            cap = 1 << 27
        isz = ISZ[spec.kw["dtype"]]
        count = _size(r, min(cap, (budget - used) // isz))
        spec = _resize(r, spec, count)
        used += spec.nbytes
        specs.append(spec)
    return layout(r, specs, name, sm, ["random"])


def _resize(r: np.random.Generator, spec: Spec, count: int) -> Spec:
    kw = dict(spec.kw, elem_count=count)
    if kw["src"] == C.TDX_SRC_SINCOS:  # rows below 2^24
        kw["elem_begin"] = min(kw.get("elem_begin", 0), (1 << 24) * 2 * kw["sincos_half"] - count)
    if kw.get("algo", 0) & 0x0F in (C.TDX_ALGO_ATEN, C.TDX_ALGO_ATEN_WIDE):
        w, p = kw.get("window_width") or 0, kw.get("window_pitch") or 0
        span = ((count - 1) // w) * p + w if w and count else count
        kw["elem_begin"] = min(kw.get("elem_begin", 0), max(0, (1 << 31) - span))
    return replace(spec, kw=kw)


def _lut_split(r, gen, epi, total: int, seeds, parts: int = 3) -> List[Spec]:
    """`total` elements of one table family in at most `parts` descriptors, each a whole number of table
    tiles (but the last) and at least 2^18 elements."""
    q, unit = total // LUT_TILE_ELEMS, LUT_MIN_ELEMS // LUT_TILE_ELEMS
    parts = max(1, min(parts, q // unit))
    sizes = [unit] * parts
    for _ in range(q - unit * parts):
        sizes[int(r.integers(parts))] += 1
    sizes = [x * LUT_TILE_ELEMS for x in sizes]
    sizes[-1] += total - sum(sizes)
    assert sum(sizes) == total and min(sizes) >= LUT_MIN_ELEMS
    return [rng_spec(r, gen, epi, False, x, seeds, nolut=False) for x in sizes]


def forced_tables(r: np.random.Generator, sm: int = SM) -> List[Table]:
    """The tables just below and just above every threshold of the scheduler."""
    out = []
    seeds = SEEDS
    nb = (N, C.TDX_BF16, C.TDX_ALGO_ICDF16)
    ub = (U, C.TDX_F16, 0)

    def small(avoid=None):
        """Four small descriptors of random generators, none of them in the family `avoid`."""
        out = []
        while len(out) < 4:
            s = rng_spec(r, _pick(r, GENERATORS), _pick(r, ["none", "basic", "ext"]), r.random() < 0.3,
                         int(r.integers(1, 5000)), seeds)
            if family(s.kw) != avoid:
                out.append(s)
        return out

    # the table threshold (x2 for the uniform): 2^25 - 8 / 2^25 normal elements, 2^26 - 8 / 2^26 uniform
    for gen, need, epi in ((nb, LUT_MIN_LAUNCH, "none"), (ub, 2 * LUT_MIN_LAUNCH, "basic")):
        for total, tag in ((need - 8, "table-below"), (need, "table-at")):
            specs = _lut_split(r, gen, epi, total, [SEEDS[0]], parts=int(r.integers(1, 4))) + small()
            specs.insert(int(r.integers(len(specs))), det_spec(r, "fill", 1000))
            out.append(layout(r, specs, f"{tag}:{gen[0]}", sm, [tag]))
    # the rider ratio: constant fills and index programs of 1/16 of the host's bytes ride, one byte more not.
    # Riders of every width and index programs with TDX_I64 and a basic epilogue; hundreds of tiles each.
    host_elems = LUT_MIN_LAUNCH * 8 if r.random() < 0.5 else LUT_MIN_LAUNCH  # (riders of 32 MiB or 4 MiB)
    for extra, tag in ((0, "riders-at"), (1, "riders-above")):
        host = _lut_split(r, nb, "none", host_elems, [SEEDS[0]], parts=2)
        budget = host_elems * 2 // 16 + extra
        riders = [Spec(dict(dtype=C.TDX_I64, src=C.TDX_SRC_IOTA, elem_count=budget // 8 // 4, p0=3.0, p1=1.0)),
                  det_spec(r, "iota", 0), det_spec(r, "fill", 0), det_spec(r, "fill", 0)]
        riders[1] = Spec(dict(dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_count=budget // 4 // 4, p0=0.0, p1=1.0,
                              epi=[(C.TDX_EPI_MUL, 0.5)]))
        riders[2] = Spec(dict(dtype=C.TDX_RAW64, src=C.TDX_SRC_CONST, elem_count=budget // 8 // 4,
                              fill_bits=0x0123_4567_89AB_CDEF, fill_itemsize=8))
        rest = budget - sum(x.nbytes for x in riders[:3])
        riders[3] = Spec(dict(dtype=C.TDX_RAW8, src=C.TDX_SRC_CONST, elem_count=rest, fill_bits=0x5A, fill_itemsize=1))
        specs = host + riders + small()
        r.shuffle(specs)
        out.append(layout(r, specs, tag, sm, [tag]))
    # the pre-assigned work list: 16 table tiles per SM, one tile less and exactly (no rider: a fill in the
    # table group would add its own tiles; the small descriptors are direct-kernel families)
    for tiles, tag in ((16 * sm - 1, "preassigned-below"), (16 * sm, "preassigned-at")):
        specs = _lut_split(r, nb, "none", tiles * LUT_TILE_ELEMS, SEEDS, parts=3)
        for s in specs:
            s.kw["elem_begin"] = 0  # (tile counts as planned)
        out.append(layout(r, specs + small(), tag, sm, [tag]))
    # static grabs: kStaticTilesPerCta tiles per resident CTA of a direct kernel, exactly and one tile more,
    # for every occupancy a 256-thread kernel can have on an SM of 2048 threads (1 to 8 CTAs): one of them is
    # the kernel's own.  The small descriptors stay out of that family.
    direct_nb = ("direct",) + nb + ("none",)
    for per_sm in range(1, 9):
        for delta in (0, 1):
            tiles = STATIC_TILES_PER_CTA * sm * per_sm + delta
            spec = rng_spec(r, nb, "none", False, tiles * DIRECT16_TILE_ELEMS, [SEEDS[0]], nolut=True)
            spec.kw["elem_begin"] = 0
            out.append(layout(r, [spec] + small(avoid=direct_nb), f"static-grabs:{per_sm}x{delta}", sm,
                              ["static-grabs"]))
    # one descriptor: the inline plan, from one element to a table-kernel launch
    for count in (1, 4097, int(r.integers(1, 1 << 22)), LUT_MIN_LAUNCH):
        gen = nb if count == LUT_MIN_LAUNCH else _pick(r, GENERATORS)
        out.append(layout(r, [rng_spec(r, gen, "none" if count == LUT_MIN_LAUNCH else _pick(r, ["none", "basic", "ext"]),
                                       False, count, seeds, nolut=False if count == LUT_MIN_LAUNCH else None)],
                          f"one:{count}", sm, ["one"]))
    # one plan header's worth of families and more: 47, 48 (the 48th family alone in the second plan, as
    # one descriptor), a random number past 47 and every one of the 80 rows
    by_family: Dict[tuple, List[Spec]] = {}
    for s in every_key(r, 0, seeds):
        by_family.setdefault(family(s.kw), []).append(s)
    fams = sorted(by_family)
    for want, tag in ((47, "families-47"), (48, "families-48"), (int(r.integers(49, len(fams) + 1)), "families-wide")):
        pick = [fams[i] for i in sorted(r.choice(len(fams), want, replace=False).tolist())]
        specs = [_resize(r, _pick(r, by_family[f]), int(r.integers(1, 20000))) for f in pick]
        # (48: one descriptor per family, so the second plan is one group of one descriptor, launched inline)
        if want != 48 and r.random() < 0.5:  # more descriptors in the families already there
            specs += [_resize(r, _pick(r, by_family[f]), int(r.integers(1, 5000))) for f in pick[: want // 2]]
        assert groups(specs) == want, (tag, groups(specs))
        out.append(layout(r, specs, tag, sm, ["wide" if want > MAX_GROUPS else "families-47"]))
    out.append(every_row(r, sm))
    return out


def every_row(r: np.random.Generator, sm: int = SM) -> Table:
    """A descriptor of every one of the 80 family rows in one table: the eight table-kernel rows each carry
    their family's threshold (768 MiB in all)."""
    specs = [_resize(r, s, int(r.integers(1, 3000))) for s in every_key(r, 0, SEEDS)]
    for row in LUT_ROWS:
        gen = (row[1], row[2], row[3])
        specs += _lut_split(r, gen, row[4], LUT_MIN_LAUNCH * (2 if row[1] == U else 1), [SEEDS[0]], parts=1)
    # fills and index programs of more than 1/16 of the largest table group: they keep their own rows
    specs.append(Spec(dict(dtype=C.TDX_RAW8, src=C.TDX_SRC_CONST, elem_count=(LUT_MIN_LAUNCH * 4) // 16 + 1,
                           fill_bits=0xA5, fill_itemsize=1)))
    r.shuffle(specs)
    return layout(r, specs, "every-row", sm, ["every-row", "wide"])


def tables(seed: int, sm: int = SM, forced: bool = True, n_random: int = 4) -> List[Table]:
    r = np.random.default_rng(seed)
    out = [random_table(r, f"random {i}", sm) for i in range(n_random)]
    if forced:
        out += forced_tables(r, sm)
    for t in out:
        t.name = f"seed {seed} {t.name}"
    return out


# ---- a module whose tensor-parallel submission spans more than one plan ---------------------------

def spec_of(d) -> Spec:
    """The Spec of a descriptor (enough of it for `family` and `route`)."""
    kw = dict(dtype=int(d.dtype), src=int(d.src), algo=int(d.algo), elem_count=int(d.elem_count),
              epi=[(int(d.epi[i].op), d.epi[i].a, d.epi[i].b) for i in range(int(d.n_epi))], flags=int(d.reserved))
    if d.src == C.TDX_SRC_IOTA:
        kw["iota_period"] = int(d.fill_bits[0])
    return Spec(kw)


def mixed_precision_model(device="cuda"):
    """fp32, bf16 and fp16 Linear pairs (Colwise / Rowwise under MIXED_PLAN) drawn with uniform, normal,
    trunc_normal_, kaiming, randn * s + m and exp / log chains, the 16-bit ones also built in fp32 and cast
    with .to(); a Mamba-style A_log, a causal mask, a sinusoid table, a host-built buffer, rotary inv_freq
    and a padding_idx embedding."""
    import torch
    from torch import nn

    inits = {
        "kaiming": lambda w: None,  # (nn.Linear's own kaiming_uniform_)
        "normal": lambda w: nn.init.normal_(w, 0.0, 0.02),
        "trunc": lambda w: nn.init.trunc_normal_(w, std=0.02),
        "affine": lambda w: nn.init.normal_(w).mul_(0.5).add_(0.125),  # randn * s + m
        "uexp": lambda w: nn.init.uniform_(w, 0.5, 2.0).log_(),
        "nexp": lambda w: nn.init.normal_(w, -2.0, 0.5).exp_(),
    }

    class Mixed(nn.Module):
        def __init__(self):
            super().__init__()
            for dt in (torch.float32, torch.bfloat16, torch.float16):
                for cast in (False, True) if dt != torch.float32 else (False,):
                    for name, init in inits.items():
                        for side, shape in (("col", (96, 40)), ("row", (40, 96))):
                            lin = nn.Linear(shape[1], shape[0], bias=side == "col", dtype=dt, device=device)
                            if cast:  # drawn on fp32, then .to(dt): the wide families
                                w = nn.Linear(shape[1], shape[0], bias=False, device=device).weight
                                with torch.no_grad():
                                    init(w)
                                lin.weight = nn.Parameter(w.detach().to(dt))
                                lin.register_buffer("master", w.detach())  # (the fp32 draw stays observable)
                            else:
                                with torch.no_grad():
                                    init(lin.weight)
                            setattr(self, f"{str(dt)[6:]}{'_cast' if cast else ''}_{name}_{side}", lin)
            self.A_log = nn.Parameter(torch.log(torch.arange(1, 17, dtype=torch.float32, device=device)).repeat(24, 1))
            self.emb = nn.Embedding(100, 48, padding_idx=0, dtype=torch.bfloat16, device=device)
            self.register_buffer("mask", torch.tril(torch.ones(64, 64, dtype=torch.bool, device=device)))
            pos = torch.arange(64, dtype=torch.float32, device=device)[:, None] * torch.exp(
                torch.arange(0, 32, dtype=torch.float32, device=device) * (-math.log(10000.0) / 32))[None, :]
            self.register_buffer("sinus", torch.cat([pos.sin(), pos.cos()], dim=1))
            self.register_buffer("host", torch.from_numpy(np.linspace(-1.0, 1.0, 200, dtype=np.float32)).to(device, torch.float16))
            self.register_buffer("inv_freq", 1.0 / (10000 ** (torch.arange(0, 64, 2, dtype=torch.int64, device=device).float() / 64)))

    return Mixed


def mixed_precision_plan(module):
    from torch.distributed.tensor.parallel import ColwiseParallel, RowwiseParallel

    return {n: ColwiseParallel() if n.endswith("_col") else RowwiseParallel()
            for n, _ in module.named_children() if n.endswith(("_col", "_row"))}
