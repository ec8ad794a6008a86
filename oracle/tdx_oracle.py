"""ctypes loader of oracle/tdx_oracle.c (TEST INFRASTRUCTURE: tests/, smoke(), bench cpu_baseline).

One library restates every descriptor of include/tdx_init.h (`generate`) and the unit draws of ATen's
stream (`aten_units`); `evaluate_plan` runs a whole InitPlan descriptor table through it."""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "_build", "libtdx_oracle.so")
# every file the library is built from (oracle/Makefile lists the same)
SOURCES = [os.path.join(HERE, f) for f in ("tdx_oracle.c", "tdx_philox.c")] + \
    [os.path.join(os.path.dirname(HERE), "include", "tdx_init.h")]


def build() -> str:
    subprocess.run(["make", "-s", "-C", HERE], check=True)
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(f) for f in SOURCES):
            build()
        _lib = ctypes.CDLL(SO)
        _lib.tdx_oracle_generate.restype = ctypes.c_int
        _lib.tdx_oracle_generate.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        _lib.tdx_oracle_aten_units.restype = ctypes.c_int
        _lib.tdx_oracle_aten_units.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        _lib.tdx_oracle_philox4x32.restype = None
        _lib.tdx_oracle_philox4x32.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        _lib.tdx_oracle_offset_increment.restype = ctypes.c_uint64
        _lib.tdx_oracle_offset_increment.argtypes = [ctypes.c_uint64]
    return _lib


def philox4x32(ctr, key, rounds=10):
    c = (ctypes.c_uint32 * 4)(*ctr)
    k = (ctypes.c_uint32 * 2)(*key)
    o = (ctypes.c_uint32 * 4)()
    lib().tdx_oracle_philox4x32(c, k, rounds, o)
    return [int(x) for x in o]


def generate(desc) -> np.ndarray:
    """Expected content (raw element bits as a numpy array) of the buffer a descriptor writes.
    `desc` is a torchdistx_b200._cabi.TdxInitDesc (only its bytes are read; a copy's source address
    is a host address)."""
    from torchdistx_b200 import _cabi as C

    isz = C.ITEMSIZE.get(int(desc.dtype), 1)  # (an unknown dtype: the library refuses it)
    out = np.empty(int(desc.elem_count), dtype={1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[isz])
    if lib().tdx_oracle_generate(ctypes.byref(desc), out.ctypes.data_as(ctypes.c_void_p)) != 0:
        raise ValueError("descriptor is outside the oracle's specification")
    return out


def aten_units(desc) -> np.ndarray:
    """The unit draws (float32) of an ATen-stream descriptor's elements, by their global index."""
    out = np.empty(int(desc.elem_count), dtype=np.float32)
    if lib().tdx_oracle_aten_units(ctypes.byref(desc), out.ctypes.data_as(ctypes.c_void_p)) != 0:
        raise ValueError("not a descriptor of ATen's stream the oracle restates")
    return out


def offset_increment(numel: int) -> int:
    return int(lib().tdx_oracle_offset_increment(numel))


def evaluate_plan(plan, seed, offset, *, shard=None, placements=None, blocks=None):
    """``({name: tensor}, generator offset after, windowed descriptor count)``: what
    ``plan.descriptors(seed, offset, ...)`` writes on this rank, by the restatement.

    Copies read their sources staged in host memory; every descriptor is placed at its ``dst`` and the
    descriptors must tile their tensor (but for entries with an uninitialised segment); entries listed
    whole are narrowed to this rank's block, as ``InitPlan.materialize`` does; by-value entries are
    ``value_tensor`` of the same block."""
    import torch

    from torchdistx_b200 import _cabi as C
    from torchdistx_b200.plan import _DTYPES, block_ranges, gather_source, narrowed, value_tensor

    keep = []  # (the sources of copy segments, staged in host memory for the call)

    def host_src(g):
        keep.append(gather_source(g, torch.uint8).clone())
        return keep[-1].data_ptr()

    table, end = plan.descriptors(seed, offset, shard, gather_src=host_src, placements=placements, blocks=blocks)
    out, windows = {}, 0
    for e, sizes, descs in table:
        if e.source == "alias":
            out[e.name] = out[e.alias_of]
            continue
        steps = plan._steps(e, shard, placements, blocks)
        if e.source == "value":
            out[e.name] = value_tensor(e, steps=steps)
            assert list(out[e.name].shape) == sizes, e.name
            continue
        dtype = _DTYPES[e.dtype]
        isz = torch.empty((), dtype=dtype).element_size()
        numel = int(np.prod(sizes)) if sizes else 1
        buf = np.zeros(numel * isz, dtype=np.uint8)
        hits = np.zeros(numel, dtype=np.int64)
        for d in descs:
            got = generate(d).view(np.uint8)
            at = int(d.dst or 0)  # (byte offset inside the tensor; ctypes reads address 0 back as None)
            assert got.size == d.elem_count * isz and at % isz == 0 and at + got.size <= buf.size, e.name
            buf[at: at + got.size] = got
            hits[at // isz: at // isz + int(d.elem_count)] += 1
            windows += bool(d.reserved & C.TDX_FLAG_WINDOW)
        uninit = e.source == "uninit" or any(g["source"] == "uninit" for g in e.segment_list())
        assert (hits <= 1).all() and (uninit or (hits == 1).all()), e.name  # the descriptors tile the tensor
        # (a trailing rank of an uneven split owns no rows)
        t = torch.from_numpy(buf).view(dtype).reshape(sizes) if numel else torch.empty(sizes, dtype=dtype)
        if narrowed(e, steps=steps):  # (listed whole: this rank narrows it)
            for k, (lo, hi) in enumerate(block_ranges(list(e.sizes), steps)):
                t = t.narrow(k, lo, hi - lo)
            t = t.contiguous()
        out[e.name] = t
    return out, end, windows

