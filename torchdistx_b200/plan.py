"""Serialisable initialisation plans (SURVEY.md section 8f item 4).

The reference's recording cannot leave the process: every op holds a ``std::function`` over the
dispatcher and an ``OperatorHandle&`` (reference src/cc/torchdistx/deferred_init.cc:159, 217-225),
so re-materialising a model -- elastic restart, a new rank joining, another seed -- means
re-running the Python constructor under ``deferred_init``.  Here the planner's verdict per tensor
is plain data (source, parameters, epilogue, RNG passes on the chain), so it can be written to
disk and replayed later with nothing but the C ABI:

    plan = InitPlan.from_module(deferred_model)        # works without a GPU
    plan.save("llama3-8b.init.json")
    ...
    tensors = InitPlan.load("llama3-8b.init.json").materialize(device="cuda", shard=(rank, world))

Under the same generator state ``InitPlan.materialize`` produces exactly the bits
``materialize_module`` produces (tests/test_plan_gpu.py): same traversal order, same Philox
offset bookkeeping, same kernels.  Tensors whose program is not fusible (tiny ``arange``-style
buffers such as rotary ``inv_freq``) are evaluated once when the plan is built and stored by
value (refused above ``max_embedded_bytes``).  Building a plan therefore MATERIALISES those few
tensors on the recording (on their recorded device); it does so under a forked RNG state, so the
caller's generators are left as they were, and it refuses programs that draw random numbers
(embedding one sample would freeze it).

``InitPlan.from_module(module, rng="aten")`` builds a plan whose draws take ATen's own CUDA stream, as
``materialize_module(rng="aten")`` draws them (InitPlan/7): PyTorch's own bits and generator offsets,
through ``materialize``, ``apply`` and ``init_sharded_module`` alike.
"""
from __future__ import annotations

import base64
import json
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
from torch.nn import Module

from . import _C, _cabi

_DTYPES = {
    "Float": torch.float32, "BFloat16": torch.bfloat16, "Half": torch.float16, "Double": torch.float64,
    "Long": torch.int64, "Int": torch.int32, "Short": torch.int16, "Char": torch.int8,
    "Byte": torch.uint8, "Bool": torch.bool,
}
_TDX_DTYPE = {torch.float32: _cabi.TDX_F32, torch.bfloat16: _cabi.TDX_BF16, torch.float16: _cabi.TDX_F16}
_RAW = {1: _cabi.TDX_RAW8, 2: _cabi.TDX_RAW16, 4: _cabi.TDX_RAW32, 8: _cabi.TDX_RAW64}
_DTYPE_NAMES = {v: k for k, v in _DTYPES.items()}
FORMAT = "torchdistx_b200.InitPlan/2"
# Plans that need the state-space extension of the ABI (an epilogue step from TDX_EPI_EXP on, or a
# broadcast index) are written as version 3, so that readers without it reject them.
FORMAT_SSM = "torchdistx_b200.InitPlan/3"
_SSM_STEPS = range(_cabi.TDX_EPI_EXP, _cabi.TDX_EPI_MULADD + 1)
# Plans with a sinusoidal position table (a "sincos" segment, TDX_SRC_SINCOS) are version 4.
FORMAT_SINCOS = "torchdistx_b200.InitPlan/4"
# Plans with a copy of a host-built tensor (a "gather" segment, TDX_SRC_GATHER: the source's bytes
# are embedded in the plan) are version 5.
FORMAT_GATHER = "torchdistx_b200.InitPlan/5"
# Plans with a band mask (a "band" segment, TDX_SRC_BAND: a causal-mask buffer) are version 6.
FORMAT_BAND = "torchdistx_b200.InitPlan/6"
# Plans built for ATen's own CUDA stream (``from_module(rng="aten")``: TDX_ALGO_ATEN draws, ATen's generator
# offsets) are version 7, with a top-level ``"rng": "aten"``; each drawn segment records "aten_wide".
FORMAT_ATEN = "torchdistx_b200.InitPlan/7"
_FORMATS = (FORMAT_ATEN, FORMAT_BAND, FORMAT_GATHER, FORMAT_SINCOS, FORMAT_SSM, FORMAT, "torchdistx_b200.InitPlan/1")


# Staging for host targets: the engine's first submission size (planner_engine.cc), and never more than
# one pass of the table needs.
HOST_STAGING_BYTES = 256 << 20


def offset_increment(numel: int) -> int:
    """Generator offset one RNG pass over `numel` elements consumes (planner_engine.cc assign_rng)."""
    blocks = (numel + 3) // 4
    return ((blocks + 3) // 4) * 4 + 4


# `aten` below: the (multiprocessor count, max threads per multiprocessor) of the device an ``rng="aten"``
# plan is built on.  ATen's launch of a draw, and so its grid stride S and its generator offset increment,
# depend on them (``_C.aten_stream_policy``); None: the default stream.
DeviceProps = Optional[Tuple[int, int]]


def _aten_policy(numel: int, aten: Tuple[int, int]) -> Tuple[int, int]:
    """(S, offset increment) of ATen's launch of one draw of `numel` elements on a device `aten`."""
    return tuple(_C.aten_stream_policy(numel, aten[0], aten[1]))


@dataclass
class PlanEntry:
    name: str
    kind: str  # "param" | "buffer"
    sizes: List[int]
    dtype: str
    source: str  # "const" | "uniform" | "normal" | "uninit" | "iota" | "sincos" | "gather" | "band" | "value"
    p0: float = 0.0
    p1: float = 0.0
    epilogue: List[Tuple[int, float, float]] = field(default_factory=list)
    const_bytes: str = ""  # base64, one element
    value: str = ""  # base64 of the whole tensor for "value" entries
    rng_numels: List[int] = field(default_factory=list)
    requires_grad: bool = False
    alias_of: Optional[str] = None  # tied parameters: same tensor as an earlier entry
    wide: bool = False  # fp32 source cast to a 16-bit dtype (TDX_ALGO_WIDE32)
    src_noround: bool = False  # TDX_FLAG_SRC_NOROUND
    # Identity of every RNG pass of `rng_numels` inside the plan: a deepcopy / clone shares its
    # source's passes (the copy is bit-identical and consumes nothing of the generator).
    rng_ids: List[int] = field(default_factory=list)
    # The tensor as disjoint element ranges, each with its own source (`w.normal_();
    # w[padding_idx].zero_()` is three); empty = one segment described by the fields above.
    # {"begin", "end", "origin", "source", "p0", "p1", "epilogue", "const_bytes", "wide",
    #  "src_noround", "rng_pass" (index into rng_numels, -1: none), for broadcast "iota"
    #  segments "iota_period", "iota_repeat" (absent: 0), and for "sincos" segments (a sinusoidal
    #  position table [R, 2H]; p0, p1 and the epilogue are its column program) "sincos_half" (H)
    #  and "sincos_cos_first" (the [cos | sin] order), and for "gather" segments (a copy of a
    #  host-built tensor) "gather_bytes" (base64 of the source, in the entry's dtype),
    #  "gather_period", "gather_repeat" (its broadcast geometry, 0 / 0: a plain copy), and for "band"
    #  segments (a band mask of an [..., R, C] tensor) "band_rows", "band_cols", "band_lo", "band_hi"
    #  and "band_in", "band_out" (the element bits inside and outside the band, as integers), and in an
    #  ``rng="aten"`` plan, for "uniform" / "normal" segments, "aten_wide" (the draw ran on fp32 and is
    #  rounded at the store: TDX_ALGO_ATEN_WIDE; such a plan lists every entry with a draw as segments)}
    segments: List[dict] = field(default_factory=list)

    def segment_list(self) -> List[dict]:
        if self.segments:
            return self.segments
        numel = 1
        for d in self.sizes:
            numel *= d
        return [dict(begin=0, end=numel, origin=0, source=self.source, p0=self.p0, p1=self.p1,
                     epilogue=self.epilogue, const_bytes=self.const_bytes, wide=self.wide,
                     src_noround=self.src_noround, rng_pass=len(self.rng_numels) - 1)]


def _prod(xs) -> int:
    n = 1
    for x in xs:
        n *= x
    return n


Steps = List[Tuple[int, int, int]]


def chunk_steps(e: "PlanEntry", shard: Optional[Tuple[int, int]], dim: Optional[int] = 0) -> Steps:
    """`shard` = (rank, world) along `dim` as chunk steps (:func:`block_ranges`): ``[(dim, rank, world)]``
    for a parameter, ``[]`` (whole) for a buffer, a 0-d tensor, one rank, no shard or `dim` None
    (replicated) -- the layout of ``materialize_module(shard=...)``, FSDP2's ``Shard(0)`` and a
    tensor-parallel ``Shard(dim)``."""
    if shard is None or shard[1] <= 1 or e.kind != "param" or not e.sizes or dim is None:
        return []
    return [(dim, shard[0], shard[1])]


def block_ranges(sizes: List[int], steps: Steps) -> List[Tuple[int, int]]:
    """The block the chunk steps ``[(dim, index, count), ...]`` cut from a tensor of `sizes`, as a range
    ``[lo, hi)`` per dimension: each step is ``torch.chunk(x, count, dim)[index]`` of the block so far
    (ceil(n / count) rows per chunk; an index past the last chunk leaves no rows)."""
    ranges = [(0, s) for s in sizes]
    for dim, index, count in steps:
        lo, hi = ranges[dim]
        per = -(-(hi - lo) // count)
        start = min(hi - lo, index * per)
        ranges[dim] = (lo + start, lo + start + max(0, min(per, hi - lo - start)))
    return ranges


def _block(e: "PlanEntry", shard, dim, steps) -> Tuple[List[Tuple[int, int]], Optional[int]]:
    """(ranges, k): the block's ranges and the one dimension k >= 1 it restricts (None: at most dim 0)."""
    if steps is None:
        steps = chunk_steps(e, shard, dim)
    ranges = block_ranges(list(e.sizes), steps)
    cut = [d for d, r in enumerate(ranges) if d and r != (0, e.sizes[d])]
    if len(cut) > 1:
        raise ValueError(f"'{e.name}': the block {ranges} restricts more than dim 0 and one other dimension")
    return ranges, (cut[0] if cut else None)


def shard_range(e: "PlanEntry", shard: Optional[Tuple[int, int]] = None, dim: Optional[int] = 0,
                steps: Optional[Steps] = None) -> Tuple[int, int, List[int]]:
    """(first element, element count, sizes) of this rank's part of an entry: the block of the chunk
    `steps` (:func:`block_ranges`), or of `shard` along `dim` (:func:`chunk_steps`).  A block is rows
    [lo_0, hi_0) of dim 0 times at most one range [lo_k, hi_k) of a dim k >= 1; with such a k it is
    ``(hi_0 - lo_0) * prod(sizes[1:k])`` runs of count / runs elements, ``sizes[k] * prod(sizes[k + 1:])``
    apart, the first at the returned element (:func:`shard_window`)."""
    ranges, k = _block(e, shard, dim, steps)
    sizes = [hi - lo for lo, hi in ranges]
    if not sizes:
        return 0, 1, sizes
    begin = ranges[0][0] * _prod(e.sizes[1:])
    if k is not None:
        begin += ranges[k][0] * _prod(e.sizes[k + 1:])
    return begin, _prod(sizes), sizes


def shard_window(e: "PlanEntry", shard: Optional[Tuple[int, int]] = None, dim: Optional[int] = 0,
                 steps: Optional[Steps] = None) -> Optional[Tuple[int, int]]:
    """(W, P) of a block that restricts a dim k >= 1 (include/tdx_init.h TDX_FLAG_WINDOW), or None for a
    part that is one contiguous range."""
    ranges, k = _block(e, shard, dim, steps)
    if k is None or (ranges[0][1] - ranges[0][0]) * _prod(e.sizes[1:k]) <= 1:  # (one run: a plain range)
        return None
    inner = _prod(e.sizes[k + 1:])
    return (ranges[k][1] - ranges[k][0]) * inner, e.sizes[k] * inner


def _narrow(t: torch.Tensor, ranges: List[Tuple[int, int]]) -> torch.Tensor:
    for d, (lo, hi) in enumerate(ranges):
        if (lo, hi) != (0, t.shape[d]):
            t = t.narrow(d, lo, hi - lo)
    return t


def value_tensor(e: "PlanEntry", shard: Optional[Tuple[int, int]] = None, dim: Optional[int] = 0,
                 steps: Optional[Steps] = None) -> torch.Tensor:
    """A by-value entry as a CPU tensor: whole, or this rank's block of a parameter (what
    ``materialize_module`` does with a replayed parameter: narrow + clone)."""
    raw = torch.frombuffer(bytearray(base64.b64decode(e.value)), dtype=torch.uint8)
    t = raw.view(_DTYPES[e.dtype]).reshape(e.sizes)
    return _narrow(t, _block(e, shard, dim, steps)[0]).contiguous()


def narrowed(e: "PlanEntry", shard: Optional[Tuple[int, int]] = None, dim: Optional[int] = 0,
             steps: Optional[Steps] = None) -> bool:
    """Is this rank's part of the entry built whole and narrowed?  A block restricting a dim k >= 1 that
    is not one contiguous range, of a program with an index, table or copy segment: those have no
    windowed descriptor (the planner's rule: planner_engine.cc emit_from)."""
    return shard_window(e, shard, dim, steps) is not None and any(
        g["source"] in ("iota", "sincos", "gather", "band") for g in e.segment_list())


def assign_pass_offsets(e: "PlanEntry", assigned: Dict[int, int], offset: int,
                        aten: DeviceProps = None) -> Tuple[List[int], int]:
    """Philox offsets of the entry's RNG passes, and the generator offset after them.  Every pass on
    the chain takes its slice of the stream once per pass identity: a clone names its source's
    passes again (same stream, nothing consumed).  `aten`: each pass, dead ones included, advances the
    generator as ATen's launch of it does on that device."""
    ids = e.rng_ids if e.rng_ids else [None] * len(e.rng_numels)
    pass_offset = []
    for pid, n in zip(ids, e.rng_numels):
        if pid is not None and pid in assigned:
            pass_offset.append(assigned[pid])
            continue
        pass_offset.append(offset)
        if pid is not None:
            assigned[pid] = offset
        offset += _aten_policy(n, aten)[1] if aten else offset_increment(n)
    return pass_offset, offset


def gather_source(g: dict, dtype: torch.dtype) -> torch.Tensor:
    """The source of a "gather" segment as a 1-D CPU tensor of the entry's dtype."""
    return torch.frombuffer(bytearray(base64.b64decode(g["gather_bytes"])), dtype=torch.uint8).view(dtype)


def entry_descriptors(e: "PlanEntry", base: int, begin: int, count: int, seed: int,
                      pass_offset: List[int], gather_src=None, window: Optional[Tuple[int, int]] = None,
                      aten: DeviceProps = None) -> list:
    """The C-ABI descriptors that write elements [begin, begin + count) of an entry into a buffer
    whose first byte is at address `base` (plain data in, ``TdxInitDesc`` out: no device needed).
    `gather_src(segment)` gives the device address of a "gather" segment's source (default 0: the
    source is not on a device; a host restatement reads it from the segment).  `window` = (W, P): the
    part is count / W runs of W elements, P apart, from `begin` (a Shard(d >= 1) block): per segment,
    the partial runs at its ends are plain descriptors, its whole runs one windowed descriptor (RNG)
    or one fill (constants) -- what the planner emits (planner_engine.cc emit_window).  `aten`: the draws
    take ATen's stream on that device (TDX_ALGO_ATEN / TDX_ALGO_ATEN_WIDE, ``fill_bits[1]`` = its grid
    stride S, and a window in ``fill_bits[0]`` as ``W | P << 32``)."""
    dtype = _DTYPES[e.dtype]
    isz = torch.empty((), dtype=dtype).element_size()
    if window is not None:
        W, P = window
        descs = []
        for g in e.segment_list():
            if g["source"] == "uninit":
                continue
            one = dict(e.__dict__, segments=[g])
            o = 0 if g["begin"] <= begin else (g["begin"] - begin) // P
            while W and o < count // W:
                rb = begin + o * P
                if rb >= g["end"]:
                    break
                lo, hi = max(rb, g["begin"]), min(rb + W, g["end"])
                if lo >= hi:
                    o += 1
                    continue
                if (lo, hi) == (rb, rb + W):  # runs [o, last) lie inside the segment
                    last = min(count // W, (g["end"] - begin - W) // P + 1)
                    (d,) = entry_descriptors(PlanEntry(**one), base + o * W * isz, rb, W, seed, pass_offset, gather_src,
                                             aten=aten)
                    if last - o > 1:
                        d.elem_count = (last - o) * W  # (a constant's whole runs are contiguous: one fill)
                        if g["source"] != "const":
                            d.reserved |= _cabi.TDX_FLAG_WINDOW
                            if aten:  # (fill_bits[1] is ATen's grid stride)
                                d.fill_bits[0] = W | P << 32
                            else:
                                d.fill_bits[0], d.fill_bits[1] = W, P
                    descs.append(d)
                    o = last
                else:
                    descs += entry_descriptors(PlanEntry(**one), base + (o * W + lo - rb) * isz, lo, hi - lo,
                                               seed, pass_offset, gather_src, aten=aten)
                    o += 1
        return descs
    descs = []
    for g in e.segment_list():
        lo, hi = max(g["begin"], begin), min(g["end"], begin + count)
        if lo >= hi or g["source"] == "uninit":
            continue
        dst = base + (lo - begin) * isz
        if g["source"] == "const":
            descs.append(_cabi.make_desc(
                dst, dtype=_RAW[isz], src=_cabi.TDX_SRC_CONST, elem_count=hi - lo,
                fill_bits=int.from_bytes(base64.b64decode(g["const_bytes"]), "little"), fill_itemsize=isz))
        elif g["source"] == "iota":  # arange and the index programs built on it (rotary inv_freq)
            descs.append(_cabi.make_desc(
                dst, dtype=_cabi.TDX_I64 if dtype == torch.int64 else _TDX_DTYPE[dtype],
                src=_cabi.TDX_SRC_IOTA, elem_begin=lo - g["origin"], elem_count=hi - lo,
                p0=g["p0"], p1=g["p1"], epi=g["epilogue"], iota_period=g.get("iota_period", 0),
                iota_repeat=g.get("iota_repeat", 0)))
        elif g["source"] == "sincos":  # a sinusoidal position table, indexed like an arange
            descs.append(_cabi.make_desc(
                dst, dtype=_TDX_DTYPE[dtype], src=_cabi.TDX_SRC_SINCOS, elem_begin=lo - g["origin"],
                elem_count=hi - lo, p0=g["p0"], p1=g["p1"], epi=g["epilogue"], sincos_half=g["sincos_half"],
                sincos_cos_first=g["sincos_cos_first"]))
        elif g["source"] == "gather":  # a copy of a host-built tensor, indexed like an arange
            descs.append(_cabi.make_desc(
                dst, dtype=_cabi.TDX_I64 if dtype == torch.int64 else _TDX_DTYPE[dtype], src=_cabi.TDX_SRC_GATHER,
                elem_begin=lo - g["origin"], elem_count=hi - lo, epi=g["epilogue"],
                gather_src=gather_src(g) if gather_src else 0, gather_period=g["gather_period"],
                gather_repeat=g["gather_repeat"]))
        elif g["source"] == "band":  # a band mask, indexed like an arange; any element width
            descs.append(_cabi.make_desc(
                dst, dtype=_RAW[isz], src=_cabi.TDX_SRC_BAND, elem_begin=lo - g["origin"], elem_count=hi - lo,
                band_rows=g["band_rows"], band_cols=g["band_cols"], band_lo=g["band_lo"], band_hi=g["band_hi"],
                band_in=g["band_in"], band_out=g["band_out"]))
        else:
            if aten:  # (the draw's dtype, whether or not the fp32 tensor is observable: it changes bits)
                algo = _cabi.TDX_ALGO_ATEN_WIDE if g["aten_wide"] else _cabi.TDX_ALGO_ATEN
                stride = _aten_policy(e.rng_numels[g["rng_pass"]], aten)[0]
            else:
                algo, stride = (_cabi.TDX_ALGO_WIDE32 if g["wide"] else 0), 0
            descs.append(_cabi.make_desc(
                dst, dtype=_TDX_DTYPE[dtype],
                src=_cabi.TDX_SRC_UNIFORM if g["source"] == "uniform" else _cabi.TDX_SRC_NORMAL,
                elem_begin=lo - g["origin"], elem_count=hi - lo, seed=seed,
                offset=pass_offset[g["rng_pass"]], p0=g["p0"], p1=g["p1"],
                epi=g["epilogue"], algo=algo, aten_stride=stride,
                flags=_cabi.TDX_FLAG_SRC_NOROUND if g["src_noround"] else 0))
    return descs


class InitPlan:
    def __init__(self, entries: List[PlanEntry], rng: str = "fused"):
        if rng not in ("fused", "aten"):
            raise ValueError(f'rng must be "fused" or "aten", got "{rng}"')
        self.entries = entries
        self.rng = rng  # the stream the plan's draws take: materialize_module's `rng`

    # ------------------------------------------------------------------------------------- build
    @classmethod
    def from_module(cls, module: Module, max_embedded_bytes: int = 1 << 20, rng: str = "fused") -> "InitPlan":
        """Builds the plan of a module created by ``deferred_init``.  Traversal order is the one
        ``materialize_module`` uses (children first, then own parameters, then own buffers).

        `rng="aten"`: the plan's draws take ATen's own CUDA stream, as ``materialize_module(rng="aten")``
        draws them: after the same ``torch.manual_seed`` its tensors and the generator's offset are
        eager CUDA's.  Each drawn segment records whether the draw ran on fp32 (rounded at the store);
        the grid stride S of each draw is not recorded, it is the materialising device's.  A tensor
        whose random program ATen's stream cannot take (a draw through a non-contiguous view, one that
        needs 64-bit indexing, a step the kernels do not compute as ATen does) raises ``ValueError``:
        ``materialize_module`` replays such a tensor through ATen, a plan cannot."""
        from .deferred_init import materialize_tensor

        if rng not in ("fused", "aten"):
            raise ValueError(f'rng must be "fused" or "aten", got "{rng}"')

        entries: List[PlanEntry] = []
        seen: Dict[int, str] = {}

        def visit(mod: Module, prefix: str) -> None:
            for cname, child in mod._modules.items():
                if child is not None:
                    visit(child, f"{prefix}{cname}.")
            for kind, group in (("param", mod._parameters), ("buffer", mod._buffers)):
                for key, t in group.items():
                    if t is None:
                        continue
                    name = prefix + key
                    if id(t) in seen:
                        entries.append(PlanEntry(name, kind, list(t.shape), _DTYPE_NAMES[t.dtype], "alias", alias_of=seen[id(t)]))
                        continue
                    seen[id(t)] = name
                    info = dict(_C.plan_info(t, rng))
                    if info.get("aten_refusal"):
                        raise ValueError(f"'{name}' has a random initialisation program ATen's stream cannot take "
                                         f"({info['aten_refusal']}); an rng=\"aten\" plan cannot hold it")
                    if info["source"] in ("const", "uniform", "normal", "uninit", "iota", "sincos", "gather", "band") \
                            and info["fusible"]:
                        segs = [dict(begin=g["begin"], end=g["end"], origin=g["origin"], source=g["source"],
                                     p0=g["p0"], p1=g["p1"], epilogue=[tuple(e) for e in g["epilogue"]],
                                     const_bytes=base64.b64encode(g["const_bytes"]).decode(),
                                     wide=bool(g["wide"]), src_noround=bool(g["src_noround"]),
                                     rng_pass=int(g["rng_pass"])) for g in info["segments"]]
                        for s, g in zip(segs, info["segments"]):
                            for k in ("iota_period", "iota_repeat"):
                                if g[k]:
                                    s[k] = int(g[k])
                            if g["source"] == "sincos":
                                s["sincos_half"] = int(g["sincos_half"])
                                s["sincos_cos_first"] = bool(g["sincos_cos_first"])
                            if g["source"] == "gather":
                                s["gather_bytes"] = base64.b64encode(g["gather_bytes"]).decode()
                                s["gather_period"] = int(g["gather_period"])
                                s["gather_repeat"] = int(g["gather_repeat"])
                            if g["source"] == "band":
                                for k in ("band_rows", "band_cols", "band_lo", "band_hi", "band_in", "band_out"):
                                    s[k] = int(g[k])
                            if rng == "aten" and g["source"] in ("uniform", "normal"):
                                s["aten_wide"] = bool(g["aten_wide"])
                        # (broadcast, table and band geometry, gather sources and the draw dtype of ATen's
                        # stream only live in the segment list)
                        only_listed = any("iota_period" in s or "aten_wide" in s or s["source"] in ("sincos", "gather", "band")
                                          for s in segs)
                        entries.append(PlanEntry(
                            name, kind, list(info["sizes"]), info["dtype"], info["source"], info["p0"], info["p1"],
                            [tuple(e) for e in info["epilogue"]],
                            base64.b64encode(info["const_bytes"]).decode(), "", list(info["rng_numels"]),
                            bool(info["requires_grad"]), None, bool(info["wide"]), bool(info["src_noround"]),
                            [int(i) for i in info["rng_op_ids"]], segs if len(segs) > 1 or only_listed else []))
                        continue
                    # not fusible (or already real): evaluate now and store by value -- under a forked
                    # RNG state, and never a program that draws random numbers (one frozen sample)
                    if info["deferred"]:
                        if any(n.startswith(("aten::rand", "aten::normal", "aten::uniform", "aten::bernoulli",
                                             "aten::multinomial", "aten::dropout"))
                               for n in (h.split(" ")[0] for h in _C.storage_history(t))):
                            raise ValueError(
                                f"'{name}' has a random initialisation program the planner cannot fold "
                                f"(first unfusable op: {info['first_unfusable_op'] or 'n/a'}); a plan cannot embed it")
                        devs = [torch.device(info["device"])] if info["device"].startswith("cuda") and torch.cuda.is_available() else []
                        with torch.random.fork_rng(devices=devs):
                            before = [torch.get_rng_state()] + [torch.cuda.get_rng_state(d) for d in devs]
                            real = materialize_tensor(t)
                            after = [torch.get_rng_state()] + [torch.cuda.get_rng_state(d) for d in devs]
                        # (the names above only see this tensor's own storage: `randn(n).sub_(c) * 2 + 3` draws
                        # its numbers in a dependency.  A generator that moved says so whatever the program is.)
                        if any(not torch.equal(a, b) for a, b in zip(before, after)):
                            raise ValueError(
                                f"'{name}' has a random initialisation program the planner cannot fold "
                                f"(first unfusable op: {info['first_unfusable_op'] or 'n/a'}); a plan cannot embed it")
                    else:
                        real = t
                    nbytes = real.numel() * real.element_size()
                    if nbytes > max_embedded_bytes:
                        raise ValueError(
                            f"'{name}' ({nbytes} bytes) has an initialisation program the planner cannot fold "
                            f"(first unfusable op: {info['first_unfusable_op'] or 'n/a'}) and is too large to embed")
                    raw = real.detach().cpu().contiguous().reshape(-1).view(torch.uint8).numpy().tobytes()
                    entries.append(PlanEntry(name, kind, list(real.shape), _DTYPE_NAMES[real.dtype],
                                             "value", value=base64.b64encode(raw).decode(),
                                             requires_grad=bool(real.requires_grad)))

        visit(module, "")
        return cls(entries, rng)

    # --------------------------------------------------------------------------------------- io
    def save(self, path: str) -> None:
        with open(path, "w") as f:
            if self.rng == "aten":
                doc = {"format": FORMAT_ATEN, "rng": "aten"}
            else:
                doc = {"format": FORMAT_BAND if self.uses_band() else FORMAT_GATHER if self.uses_gather()
                       else FORMAT_SINCOS if self.uses_sincos() else FORMAT_SSM if self.uses_ssm() else FORMAT}
            json.dump({**doc, "entries": [e.__dict__ for e in self.entries]}, f)

    def uses_band(self) -> bool:
        """Does the plan hold a band mask (written as InitPlan/6)?"""
        return any(g["source"] == "band" for e in self.entries for g in e.segments)

    def uses_gather(self) -> bool:
        """Does the plan hold a copy of a host-built tensor (written as InitPlan/5)?"""
        return any(g["source"] == "gather" for e in self.entries for g in e.segments)

    def uses_sincos(self) -> bool:
        """Does the plan hold a sinusoidal position table (written as InitPlan/4)?"""
        return any(g["source"] == "sincos" for e in self.entries for g in e.segments)

    def uses_ssm(self) -> bool:
        """Does the plan need the state-space extension (written as InitPlan/3)?"""
        for e in self.entries:
            if any(st[0] & 0xFF in _SSM_STEPS for st in e.epilogue):
                return True
            for g in e.segments:
                if g.get("iota_period") or any(st[0] & 0xFF in _SSM_STEPS for st in g["epilogue"]):
                    return True
        return False

    @classmethod
    def load(cls, path: str) -> "InitPlan":
        with open(path) as f:
            doc = json.load(f)
        if doc.get("format") not in _FORMATS:
            raise ValueError(f"{path}: not an {FORMAT} file")
        rng = doc.get("rng", "fused")
        if (doc["format"] == FORMAT_ATEN) != (rng == "aten"):
            raise ValueError(f"{path}: a {doc['format']} file with rng {rng!r}")
        entries = []
        for d in doc["entries"]:
            d["epilogue"] = [tuple(e) for e in d.get("epilogue", [])]
            for g in d.get("segments", []):
                g["epilogue"] = [tuple(e) for e in g.get("epilogue", [])]
            entries.append(PlanEntry(**d))
        return cls(entries, rng)

    @property
    def num_params(self) -> int:
        n = 0
        for e in self.entries:
            if e.kind == "param" and e.source != "alias":
                k = 1
                for s in e.sizes:
                    k *= s
                n += k
        return n

    # ------------------------------------------------------------------------------ descriptors
    @staticmethod
    def _steps(e: PlanEntry, shard, placements, blocks) -> Steps:
        if blocks is not None:
            if shard is not None or placements is not None:
                raise ValueError("give either `blocks` or `shard` / `placements`")
            return list(blocks.get(e.name, []))
        return chunk_steps(e, shard, 0 if placements is None else placements.get(e.name))

    def descriptors(self, seed: int, offset: int, shard: Optional[Tuple[int, int]] = None, gather_src=None,
                    placements: Optional[Dict[str, Optional[int]]] = None, blocks: Optional[Dict[str, Steps]] = None,
                    device_props: DeviceProps = None):
        """The plan as the C ABI sees it, without a device: ``([(entry, sizes, descs)], offset after)``
        for the tensors :meth:`materialize` would build from generator state ``(seed, offset)`` on
        this rank.  ``descs`` address each tensor from byte 0 (``dst`` = byte offset inside it); value
        and alias entries have none.  A host that is not Python rebuilds exactly this table from the
        JSON file; tests evaluate it with the stream's CPU restatement.  `gather_src(segment)` gives
        the address of a "gather" segment's source (default: 0, none staged).

        `placements` (``{parameter name: d or None}``, :func:`torchdistx_b200.parallel.tp_placements`):
        a tensor-parallel layout instead of dim-0 chunks -- each listed parameter is this rank's
        ``Shard(d)`` block (``None``: replicated), every other entry is whole, as
        ``materialize_module(parallelize_plan=...)`` builds them.  An entry with an index, table or
        copy segment under ``Shard(d >= 1)`` is listed whole (sizes and descriptors); narrow it
        (:func:`narrowed`).

        `blocks` (``{entry name: chunk steps}``, :func:`torchdistx_b200.parallel.local_block`): any
        layout whose local blocks are rows of dim 0 times at most one range of another dimension, such
        as FSDP2 over tensor parallelism on a 2-D mesh -- each listed entry is its block
        (:func:`block_ranges`), every other entry is whole; not combined with `shard` / `placements`.
        Entries built whole and narrowed are listed whole, as above.

        `device_props` = (multiprocessor count, max threads per multiprocessor) of the device that will
        run the table: required for an ``rng="aten"`` plan, whose draws take ATen's launch on that device
        (each drawn descriptor carries its grid stride S in ``fill_bits[1]``, and each pass advances
        the generator by ATen's increment); ignored otherwise."""
        aten = self._aten_props(device_props)
        assigned: Dict[int, int] = {}
        table = []
        for e in self.entries:
            steps = self._steps(e, shard, placements, blocks)
            if e.source in ("alias", "value"):  # (a by-value parameter is chunked like any other: value_tensor)
                table.append((e, shard_range(e, steps=steps)[2] if e.source == "value" else list(e.sizes), []))
                continue
            if narrowed(e, steps=steps):
                steps = []
            begin, count, sizes = shard_range(e, steps=steps)
            pass_offset, offset = assign_pass_offsets(e, assigned, offset, aten)
            table.append((e, sizes, entry_descriptors(e, 0, begin, count, seed, pass_offset, gather_src,
                                                      shard_window(e, steps=steps), aten)))
        return table, offset

    def _aten_props(self, device_props: DeviceProps) -> DeviceProps:
        if self.rng != "aten":
            return None
        if device_props is None:
            raise ValueError('an rng="aten" plan needs the device\'s (multiprocessor count, max threads per '
                             'multiprocessor) as `device_props`: its draws take ATen\'s launch on that device')
        sm, tps = (int(x) for x in device_props)
        return sm, tps

    # ------------------------------------------------------------------------------ materialise
    def materialize(self, device="cuda", shard: Optional[Tuple[int, int]] = None,
                    generator: Optional[torch.Generator] = None,
                    into: Optional[Dict[str, torch.Tensor]] = None,
                    placements: Optional[Dict[str, Optional[int]]] = None,
                    blocks: Optional[Dict[str, Steps]] = None,
                    staging_bytes: int = HOST_STAGING_BYTES) -> Dict[str, torch.Tensor]:
        """Builds every tensor of the plan on `device` through libtdx_init and returns
        ``{name: tensor}`` (parameters as ``torch.nn.Parameter``).  Consumes the CUDA generator
        exactly like ``materialize_module`` would.

        `into`: write into caller-owned CUDA buffers instead of allocating (``{name: tensor}``; each
        must be contiguous, of the plan's dtype and hold at least this rank's elements).  This is
        the FSDP hand-off of SURVEY 8f.1: after ``fully_shard(meta_model)`` / ``to_empty`` the
        local shards FSDP owns are initialised in place, no unsharded tensor, no copy
        (:func:`init_sharded_module`).

        An `into` buffer may also be a contiguous CPU tensor, pinned or pageable: a CPU-offloaded shard
        (FSDP2's ``CPUOffloadPolicy``, FSDP1's ``offload_params``).  Its descriptors are built on `device`
        all the same and copied to host memory in passes through a staging buffer of at most
        `staging_bytes` (``tdx_init_submit_host``), after the table of device targets; by-value entries
        and entries built whole and narrowed are built on the device and copied into it.  The bits and
        the generator offsets are those of CUDA targets.  The call returns once every host target holds
        its values.

        `placements`: a tensor-parallel layout, as for :meth:`descriptors` (the tensors are this
        rank's local blocks; entries built whole and narrowed are narrowed here, on the device).

        `blocks`: each listed entry is its block of chunk steps, every other entry whole, as for
        :meth:`descriptors` (the FSDP x TP hand-off of :func:`init_sharded_module`).

        An ``rng="aten"`` plan draws from ATen's stream as laid out for `device` (its multiprocessor
        count and threads per multiprocessor), under every layout above.
        """
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError("InitPlan.materialize drives the CUDA kernels; there is no CPU path")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        gen = generator or torch.cuda.default_generators[device.index]
        seed, offset = gen.initial_seed(), gen.get_offset()
        aten = None
        if self.rng == "aten":
            props = torch.cuda.get_device_properties(device)
            aten = props.multi_processor_count, props.max_threads_per_multi_processor
        out: Dict[str, torch.Tensor] = {}
        descs = []
        host_descs = []  # descriptors whose destination is a CPU `into` buffer
        host_written = False
        staged: List[torch.Tensor] = []  # gather sources on the device: alive until the launch is queued

        def gather_src(g: dict) -> int:
            staged.append(gather_source(g, _DTYPES[e.dtype]).to(device))
            return staged[-1].data_ptr()

        assigned: Dict[int, int] = {}  # RNG pass identity -> the offset it was given
        narrow = []  # (entry, block ranges) of entries built whole and narrowed after the launch
        with torch.cuda.device(device):
            for e in self.entries:
                if e.source == "alias":
                    out[e.name] = out[e.alias_of]
                    continue
                dtype = _DTYPES[e.dtype]
                target = None if into is None else into.get(e.name)
                steps = self._steps(e, shard, placements, blocks)
                if e.source == "value":
                    t = value_tensor(e, steps=steps).to(device)
                    if target is not None:
                        target.copy_(t)
                        host_written |= target.device.type == "cpu"
                        t = target
                    out[e.name] = t if target is not None else _wrap(t, e)
                    continue
                if narrowed(e, steps=steps):
                    narrow.append((e, block_ranges(list(e.sizes), steps)))
                    steps, target = [], None  # (the whole tensor is a temporary)
                begin, count, sizes = shard_range(e, steps=steps)
                if target is not None and target.device.type == "cpu":
                    if not (target.is_contiguous() and target.dtype == dtype and target.numel() >= count):
                        raise ValueError(f"'{e.name}': a CPU `into` buffer must be a contiguous {dtype} tensor "
                                         f"with at least {count} elements")
                    t = target
                elif target is not None:
                    if not (target.is_cuda and target.is_contiguous() and target.dtype == dtype
                            and target.numel() >= count):
                        raise ValueError(f"'{e.name}': `into` buffer must be a contiguous CUDA {dtype} tensor "
                                         f"with at least {count} elements")
                    t = target
                else:
                    t = torch.empty(sizes, dtype=dtype, device=device)
                pass_offset, offset = assign_pass_offsets(e, assigned, offset, aten)
                table = host_descs if t.device.type == "cpu" else descs
                table += entry_descriptors(e, t.data_ptr(), begin, count, seed, pass_offset, gather_src,
                                           shard_window(e, steps=steps), aten)
                out[e.name] = t if target is not None else _wrap(t, e)
            if descs:
                ws_bytes = _cabi.prepare(descs)  # exactly what this table needs (not the ~1.6 MB upper bound)
                if ws_bytes:
                    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
                    _cabi.submit(ws.data_ptr(), ws_bytes, torch.cuda.current_stream(device).cuda_stream)
            if host_descs:
                submit_host(host_descs, device, staging_bytes)
                host_written = True
            for e, ranges in narrow:
                t = _narrow(out[e.name].detach(), ranges).contiguous()
                target = None if into is None else into.get(e.name)
                if target is not None:
                    target.view(-1)[: t.numel()].copy_(t.view(-1))
                    host_written |= target.device.type == "cpu"
                out[e.name] = target if target is not None else _wrap(t, e)
            gen.set_offset(offset)
            if host_written:  # (pinned copies are asynchronous: the host reads these tensors next)
                torch.cuda.current_stream(device).synchronize()
        return out

    def apply(self, module: Module, **kw) -> None:
        """Materialises the plan into `module` (e.g. one built under ``torch.device("meta")``):
        every parameter / buffer named in the plan is replaced."""
        tensors = self.materialize(**kw)
        for name, t in tensors.items():
            owner, _, key = name.rpartition(".")
            mod = module.get_submodule(owner) if owner else module
            group = mod._parameters if key in mod._parameters else mod._buffers
            group[key] = t


def host_staging_bytes(descs, staging_bytes: int = HOST_STAGING_BYTES) -> int:
    """The staging buffer :func:`submit_host` allocates for `descs`: `staging_bytes`, or less when the
    whole table (its bytes, each piece's alignment and the workspace of one pass) fits in less."""
    data = sum(int(d.elem_count) * _cabi.ITEMSIZE[int(d.dtype)] + 16 for d in descs)
    return min(int(staging_bytes), data + _cabi.load().tdx_init_workspace_bytes(3 * len(descs)))


def submit_host(descs, device: torch.device, staging_bytes: int = HOST_STAGING_BYTES) -> int:
    """Runs a table of host destinations through ``tdx_init_submit_host`` on `device`'s current stream,
    with a staging buffer from the caching allocator; returns the kernel launches over every pass.  The
    copies into pinned memory are asynchronous: synchronise the stream before reading the targets."""
    n = host_staging_bytes(descs, staging_bytes)
    stream = torch.cuda.current_stream(device)
    staging = torch.empty(n, dtype=torch.uint8, device=device)  # (freed in stream order after the copies)
    return _cabi.submit_host(descs, staging.data_ptr(), n, stream.cuda_stream)


def _wrap(t: torch.Tensor, e: PlanEntry) -> torch.Tensor:
    if e.kind == "param":
        return torch.nn.Parameter(t, requires_grad=e.requires_grad)
    return t


def init_sharded_module(module: Module, plan: InitPlan, rank: Optional[int] = None, world: Optional[int] = None,
                        device="cuda") -> None:
    """FSDP2 hand-off (SURVEY 8f.1): `module` has been through ``fully_shard`` (its parameters are
    ``DTensor``s sharded on dim 0 over `world` ranks, e.g. built on the meta device and
    ``to_empty(device=...)``'d).  Every rank fills the local shards FSDP owns, in place, with its
    slice of the plan -- no full tensor, no chunk/clone.  All ranks must hold the same generator
    state (:func:`torchdistx_b200.parallel.sync_rng`).

    Without `rank` and `world`, each parameter's layout is read from the parameter itself
    (:func:`torchdistx_b200.parallel.local_block`): ``parallelize_module`` over a ``tp`` mesh dimension
    and then ``fully_shard`` over ``dp`` (or HSDP), FSDP2 alone, or tensor parallelism alone.  Every
    ``to_local()`` block is filled in place in one call; buffers, which FSDP2 does not shard, are whole;
    FSDP2's padding past a block stays unwritten.  Every rank of the whole world draws the same
    generator offsets (they depend on global sizes only), so call ``sync_rng`` over the default group
    first.  Raises ``ValueError`` for a parameter the plan lacks or whose global shape or dtype differs
    from its entry, a local tensor smaller than its block, and a tied parameter whose names carry
    different layouts."""
    if (rank is None) != (world is None):
        raise ValueError("give both `rank` and `world`, or neither (layouts read from the parameters)")
    if rank is None:
        return _init_blocks(module, plan, device)
    into = {name: _local(t) for name, t in list(module.named_parameters()) + list(module.named_buffers())}
    with torch.no_grad():
        plan.materialize(device=device, shard=(rank, world), into=into)


def _local(t: torch.Tensor) -> torch.Tensor:
    local = t.to_local() if hasattr(t, "to_local") else t
    return local.data if hasattr(local, "data") else local


def _init_blocks(module: Module, plan: InitPlan, device) -> None:
    """:func:`init_sharded_module` with each parameter's layout read from its placements."""
    from .parallel import local_block

    entries = {e.name: e for e in plan.entries}
    params = dict(module.named_parameters(remove_duplicate=False))
    blocks: Dict[str, Steps] = {}
    into: Dict[str, torch.Tensor] = {}
    for name, p in params.items():
        e = entries.get(name)
        if e is None:
            raise ValueError(f"'{name}' is not in the plan")
        if list(p.shape) != list(e.sizes) or p.dtype != _DTYPES[e.dtype]:
            raise ValueError(f"'{name}' is {p.dtype} {list(p.shape)} in the module and "
                             f"{_DTYPES[e.dtype]} {list(e.sizes)} in the plan")
        steps = local_block(p, name)
        if e.source == "alias":  # (filled once, through the name the plan built it under)
            src = params.get(e.alias_of)
            if src is not p:
                other = "absent" if src is None else f"{tuple(getattr(src, 'placements', ()))}"
                raise ValueError(f"'{e.alias_of}' and '{name}' are one tied parameter in the plan, but the module "
                                 f"lays them out differently ({other} and {tuple(getattr(p, 'placements', ()))})")
            continue
        local = _local(p)
        count = shard_range(e, steps=steps)[1]
        if local.numel() < count:
            raise ValueError(f"'{name}': the local tensor holds {local.numel()} elements, its block "
                             f"{block_ranges(list(e.sizes), steps)} has {count}")
        blocks[name], into[name] = steps, local
    for name, b in module.named_buffers():  # (FSDP2 does not shard buffers: whole)
        into[name] = _local(b)
    with torch.no_grad():
        plan.materialize(device=device, into=into, blocks=blocks)
