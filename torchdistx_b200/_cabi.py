"""ctypes view of the C ABI declared in ``include/tdx_init.h`` (libtdx_init.so).

The product path (``torchdistx_b200._C``) links the library directly; this module exists
so that tests, the kernel sweep and ``bench.py`` can drive the kernels *through the C ABI*
with raw device pointers, exactly as a non-Python host (the reference's C++ runtime,
``src/cc/torchdistx/deferred_init.cc``) would.

There is deliberately no fallback: if the shared library is missing, importing the
loader raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Iterable, Optional, Sequence

_HERE = os.path.dirname(os.path.abspath(__file__))
# TDX_INIT_LIB: another build of the library (to compare two builds, or to check that a missing one is an
# error); the engine always uses the in-tree library
LIB_PATH = os.environ.get("TDX_INIT_LIB") or os.path.join(_HERE, "libtdx_init.so")

# enums of tdx_init.h
TDX_F32, TDX_BF16, TDX_F16, TDX_I64 = 0, 1, 2, 3
TDX_RAW8, TDX_RAW16, TDX_RAW32, TDX_RAW64 = 8, 9, 10, 11
# bytes per element of each dtype
ITEMSIZE = {TDX_F32: 4, TDX_BF16: 2, TDX_F16: 2, TDX_I64: 8, TDX_RAW8: 1, TDX_RAW16: 2, TDX_RAW32: 4, TDX_RAW64: 8}
TDX_SRC_CONST, TDX_SRC_UNIFORM, TDX_SRC_NORMAL, TDX_SRC_IOTA = 0, 1, 2, 3
TDX_SRC_SINCOS = 4
TDX_SRC_GATHER = 5
TDX_SRC_BAND = 6
TDX_SINCOS_COS_FIRST = 0x1
TDX_ALGO_DEFAULT, TDX_ALGO_ICDF16, TDX_ALGO_BM32 = 0, 1, 2
TDX_ALGO_WIDE32 = 2
TDX_ALGO_ATEN, TDX_ALGO_ATEN_WIDE = 3, 4
TDX_ALGO_NOLUT = 0x20
TDX_EPI_MUL, TDX_EPI_ADD, TDX_EPI_ERFINV, TDX_EPI_CLAMP, TDX_EPI_RPOW, TDX_EPI_RECIP = 1, 2, 3, 4, 5, 6
TDX_EPI_EXP, TDX_EPI_LOG, TDX_EPI_EXPM1, TDX_EPI_INV_SOFTPLUS, TDX_EPI_MULADD = 7, 8, 9, 10, 11
TDX_MAX_EPI = 4
TDX_EPI_NOROUND = 0x100
TDX_FLAG_SRC_NOROUND = 0x1
TDX_FLAG_WINDOW = 0x2
TDX_E_BADARG, TDX_E_WORKSPACE, TDX_E_NODEVICE = -1, -2, -3

EXPORTED_SYMBOLS = (
    "tdx_init_workspace_bytes",
    "tdx_init_launch",
    "tdx_init_prepare",
    "tdx_init_submit",
    "tdx_plan_upload",
    "tdx_plan_launch",
    "tdx_init_submit_host",
    "tdx_init_host_cut",
    "tdx_init_host_piece_descs",
    "tdx_last_host_copies",
    "tdx_last_launch_count",
    "tdx_last_upload_bytes",
    "tdx_elems_per_block",
    "tdx_abi_version",
    "tdx_last_error",
)


class TdxEpiStep(ctypes.Structure):
    _fields_ = [("op", ctypes.c_uint32), ("a", ctypes.c_float), ("b", ctypes.c_float)]


class TdxInitDesc(ctypes.Structure):
    _fields_ = [
        ("dst", ctypes.c_void_p),
        ("elem_begin", ctypes.c_uint64),
        ("elem_count", ctypes.c_uint64),
        ("philox_seed", ctypes.c_uint64),
        ("philox_offset", ctypes.c_uint64),
        ("p0", ctypes.c_double),
        ("p1", ctypes.c_double),
        ("fill_bits", ctypes.c_uint64 * 2),
        ("dtype", ctypes.c_uint8),
        ("src", ctypes.c_uint8),
        ("algo", ctypes.c_uint8),
        ("n_epi", ctypes.c_uint8),
        ("reserved", ctypes.c_uint32),
        ("epi", TdxEpiStep * TDX_MAX_EPI),
    ]


class TdxPlan(ctypes.Structure):
    _fields_ = [("opaque", ctypes.c_uint64 * 512)]


class TdxHostPiece(ctypes.Structure):
    _fields_ = [
        ("desc", ctypes.c_int32),
        ("pass_", ctypes.c_int32),
        ("elem_first", ctypes.c_uint64),
        ("elem_count", ctypes.c_uint64),
        ("staging_off", ctypes.c_uint64),
    ]


assert ctypes.sizeof(TdxInitDesc) == 128, ctypes.sizeof(TdxInitDesc)

_lib: Optional[ctypes.CDLL] = None


def load() -> ctypes.CDLL:
    """Loads libtdx_init.so (built by ``__graft_entry__.build()`` / ``build_kernels.sh``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: the CUDA kernel library has not been built "
            "(run `python -c 'import __graft_entry__ as g; g.build()'`). "
            "torchdistx_b200 has no CPU fallback for CUDA tensors."
        )
    lib = ctypes.CDLL(LIB_PATH)
    lib.tdx_init_workspace_bytes.restype = ctypes.c_size_t
    lib.tdx_init_workspace_bytes.argtypes = [ctypes.c_int]
    lib.tdx_init_prepare.restype = ctypes.c_int
    lib.tdx_init_prepare.argtypes = [ctypes.POINTER(TdxInitDesc), ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]
    lib.tdx_init_submit.restype = ctypes.c_int
    lib.tdx_init_submit.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.tdx_init_launch.restype = ctypes.c_int
    lib.tdx_init_launch.argtypes = [
        ctypes.POINTER(TdxInitDesc), ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.tdx_plan_upload.restype = ctypes.c_int
    lib.tdx_plan_upload.argtypes = [
        ctypes.POINTER(TdxInitDesc), ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
        ctypes.POINTER(TdxPlan)]
    lib.tdx_plan_launch.restype = ctypes.c_int
    lib.tdx_plan_launch.argtypes = [ctypes.POINTER(TdxPlan), ctypes.c_void_p, ctypes.c_void_p]
    lib.tdx_init_submit_host.restype = ctypes.c_int
    lib.tdx_init_submit_host.argtypes = [
        ctypes.POINTER(TdxInitDesc), ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.tdx_init_host_cut.restype = ctypes.c_int
    lib.tdx_init_host_cut.argtypes = [
        ctypes.POINTER(TdxInitDesc), ctypes.c_int, ctypes.c_size_t, ctypes.POINTER(TdxHostPiece), ctypes.c_int,
        ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    lib.tdx_init_host_piece_descs.restype = ctypes.c_int
    lib.tdx_init_host_piece_descs.argtypes = [
        ctypes.POINTER(TdxInitDesc), ctypes.POINTER(TdxHostPiece), ctypes.c_void_p, ctypes.POINTER(TdxInitDesc)]
    lib.tdx_last_host_copies.restype = ctypes.c_int
    lib.tdx_last_launch_count.restype = ctypes.c_int
    lib.tdx_last_upload_bytes.restype = ctypes.c_size_t
    lib.tdx_elems_per_block.restype = ctypes.c_int
    lib.tdx_elems_per_block.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.tdx_abi_version.restype = ctypes.c_int
    lib.tdx_last_error.restype = ctypes.c_char_p
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError(f"libtdx_init: error {rc}: {load().tdx_last_error().decode()}")


def fill_pattern(value_bits: int, itemsize: int) -> Sequence[int]:
    """16-byte store pattern: the element's bits replicated."""
    b = int(value_bits).to_bytes(itemsize, "little") * (16 // itemsize)
    return int.from_bytes(b[:8], "little"), int.from_bytes(b[8:], "little")


def make_desc(dst: int, *, dtype: int, src: int, elem_count: int, elem_begin: int = 0,
              seed: int = 0, offset: int = 0, p0: float = 0.0, p1: float = 1.0, algo: int = 0,
              fill_bits: int = 0, fill_itemsize: int = 0,
              epi: Iterable[tuple] = (), flags: int = 0, iota_period: int = 0,
              iota_repeat: int = 0, sincos_half: int = 0, sincos_cos_first: bool = False,
              gather_src: int = 0, gather_period: int = 0, gather_repeat: int = 0,
              band_rows: int = 0, band_cols: int = 0, band_lo: int = 0, band_hi: int = 0,
              band_in: int = 0, band_out: int = 0, aten_stride: int = 0, window_width: int = 0,
              window_pitch: int = 0) -> TdxInitDesc:
    d = TdxInitDesc()
    d.dst = dst
    d.elem_begin = elem_begin
    d.elem_count = elem_count
    d.philox_seed = seed & (2**64 - 1)
    d.philox_offset = offset
    d.p0, d.p1 = p0, p1
    d.dtype, d.src, d.algo = dtype, src, algo
    d.reserved = flags
    if src == TDX_SRC_CONST:
        lo, hi = fill_pattern(fill_bits, fill_itemsize)
        d.fill_bits[0], d.fill_bits[1] = lo, hi
    elif src == TDX_SRC_IOTA:  # broadcast geometry (include/tdx_init.h): 0, 0 = the plain arange
        d.fill_bits[0], d.fill_bits[1] = iota_period, iota_repeat
    elif src == TDX_SRC_SINCOS:  # {H, order}: p0, p1 and epi are the column program
        d.fill_bits[0], d.fill_bits[1] = sincos_half, TDX_SINCOS_COS_FIRST if sincos_cos_first else 0
    elif src == TDX_SRC_GATHER:  # {source address, P | R << 32}: {0, 0} geometry = the plain copy
        d.fill_bits[0], d.fill_bits[1] = gather_src, gather_period | (gather_repeat << 32)
    elif src == TDX_SRC_BAND:  # {C | R << 32, lo | hi << 32}; the IN / OUT bits ride in seed / offset
        d.fill_bits[0] = band_cols | (band_rows << 32)
        d.fill_bits[1] = (band_lo & 0xFFFFFFFF) | ((band_hi & 0xFFFFFFFF) << 32)
        d.philox_seed, d.philox_offset = band_in, band_out
    elif algo & 0x0F in (TDX_ALGO_ATEN, TDX_ALGO_ATEN_WIDE):  # {W | P << 32 (TDX_FLAG_WINDOW), S}
        d.fill_bits[0] = window_width | (window_pitch << 32)
        d.fill_bits[1] = aten_stride
    steps = list(epi)
    d.n_epi = len(steps)
    for i, st in enumerate(steps):
        d.epi[i].op = st[0]
        d.epi[i].a = st[1] if len(st) > 1 else 0.0
        d.epi[i].b = st[2] if len(st) > 2 else 0.0
    return d


def launch(descs: Sequence[TdxInitDesc], workspace_ptr: int, workspace_bytes: int,
           stream: int = 0) -> int:
    """tdx_init_launch over a Python list of descriptors; returns the number of kernel launches."""
    lib = load()
    arr = (TdxInitDesc * len(descs))(*descs)
    check(lib.tdx_init_launch(arr, len(descs), workspace_ptr, workspace_bytes, stream))
    return lib.tdx_last_launch_count()


def prepare(descs: Sequence[TdxInitDesc]) -> int:
    """tdx_init_prepare: lays the plan out on the host; returns the exact workspace size it needs
    (0: nothing to launch).  Follow with `submit` on the same thread."""
    lib = load()
    arr = (TdxInitDesc * len(descs))(*descs)
    need = ctypes.c_size_t(0)
    check(lib.tdx_init_prepare(arr, len(descs), ctypes.byref(need)))
    return int(need.value)


def submit(workspace_ptr: int, workspace_bytes: int, stream: int = 0) -> int:
    """tdx_init_submit of the plan `prepare` built; returns the number of kernel launches."""
    lib = load()
    check(lib.tdx_init_submit(workspace_ptr, workspace_bytes, stream))
    return lib.tdx_last_launch_count()


def submit_host(descs: Sequence[TdxInitDesc], staging_ptr: int, staging_bytes: int, stream: int = 0) -> int:
    """tdx_init_submit_host: runs a table of host destinations in passes through the device staging
    buffer; returns the number of kernel launches over every pass."""
    lib = load()
    arr = (TdxInitDesc * len(descs))(*descs)
    check(lib.tdx_init_submit_host(arr, len(descs), staging_ptr, staging_bytes, stream))
    return lib.tdx_last_launch_count()


def host_cut(descs: Sequence[TdxInitDesc], staging_bytes: int):
    """tdx_init_host_cut, without a device: ``(pieces, passes)`` of the cut tdx_init_submit_host makes of
    the table for a staging buffer of `staging_bytes` (``TdxHostPiece``s, pass by pass)."""
    lib = load()
    arr = (TdxInitDesc * len(descs))(*descs)
    n, passes = ctypes.c_int(0), ctypes.c_int(0)
    check(lib.tdx_init_host_cut(arr, len(descs), staging_bytes, None, 0, ctypes.byref(n), ctypes.byref(passes)))
    pieces = (TdxHostPiece * n.value)()
    check(lib.tdx_init_host_cut(arr, len(descs), staging_bytes, pieces, n.value, ctypes.byref(n), ctypes.byref(passes)))
    return list(pieces), passes.value


def piece_descs(desc: TdxInitDesc, piece: TdxHostPiece, staging_ptr: int = 0) -> list:
    """tdx_init_host_piece_descs: the descriptors that write `piece` of `desc` into a staging buffer at
    `staging_ptr`, in local order."""
    out = (TdxInitDesc * 3)()
    k = load().tdx_init_host_piece_descs(ctypes.byref(desc), ctypes.byref(piece), staging_ptr, out)
    if k < 0:
        check(k)
    return list(out[:k])
