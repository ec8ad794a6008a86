"""ATen's own CUDA stream (`rng="aten"`, TDX_ALGO_ATEN) without a GPU: ATen's launch policy, the C
restatement oracle/tdx_philox.c pinned to curand's own host code, the library's validation of the
descriptors, and the `rng=` option of the public calls."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

from torchdistx_b200 import _C
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, materialize_module, materialize_tensor

ORACLE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")
CUDA_INCLUDE = "/usr/local/cuda/include"


def policy(n, sm, tps):
    """DistributionTemplates.h calc_execution_policy, restated."""
    grid = min(sm * (tps // 256), (n + 255) // 256)
    s = 256 * grid
    return s, ((n - 1) // (4 * s) + 1) * 4


@pytest.mark.parametrize("sm", [132, 114])
def test_launch_policy_matches_aten(sm):
    s_max = 256 * sm * 8
    for n in (1, 255, 256, s_max - 1, s_max, 4 * s_max, 4 * s_max + 1, 2**31 - 2, 2**31 - 1, 10**7 + 7):
        assert tuple(_C.aten_stream_policy(n, sm, 2048)) == policy(n, sm, 2048), n
    assert tuple(_C.aten_stream_policy(0, sm, 2048))[1] == 0  # an empty tensor draws nothing


HARNESS = r"""
#include <cstdio>
#include <cmath>
#include <curand_kernel.h>
extern "C" {
#include "tdx_philox.c"
}
int main() {
  const unsigned long long seeds[3] = {0ull, 42ull, 0x123456789abcdefull};
  const unsigned long long offsets[3] = {0ull, 4ull, 1ull << 40};
  const unsigned S[2] = {256u * 132u * 8u, 512u};
  long bad_word = 0, bad_uniform = 0, bad_normal = 0, n = 0;
  for (auto seed : seeds) for (auto off : offsets) for (unsigned s : S)
    for (unsigned g = 0; g < 12u * s; g += (g % 977u) + 1u) {
      const unsigned t = g % s, q = g / s, k = q / 4, j = q % 4;
      curandStatePhilox4_32_10_t st, su, sn;
      curand_init(seed, t, off, &st);
      uint4 w;
      for (unsigned i = 0; i <= k; ++i) w = curand4(&st);
      curand_init(seed, t, off, &su);
      float4 u;
      for (unsigned i = 0; i <= k; ++i) u = curand_uniform4(&su);
      curand_init(seed, t, off, &sn);
      float4 z;
      for (unsigned i = 0; i <= k; ++i) z = curand_normal4(&sn);
      const unsigned wj = (&w.x)[j];
      const float uj = (&u.x)[j], zj = (&z.x)[j];
      bad_word += aten_word(seed, off, s, g) != wj;
      bad_uniform += aten_uniform01(seed, off, s, g) != uj;
      const float mine = aten_normal01(seed, off, s, g);
      const float ulp = std::nextafter(std::fabs(zj), INFINITY) - std::fabs(zj);
      bad_normal += std::fabs(mine - zj) > 4 * ulp;
      ++n;
    }
  std::printf("%ld %ld %ld %ld\n", n, bad_word, bad_uniform, bad_normal);
  return 0;
}
"""


@pytest.mark.skipif(shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INCLUDE, "curand_kernel.h")),
                    reason="needs g++ and the CUDA toolkit's curand headers")
def test_oracle_is_curand(tmp_path):
    """Words and uniform lanes equal curand's host code (built with contraction, as nvcc builds the
    device code); normals within 4 ulp (both through libm here, but curand's host path and the
    restatement may round -2 log(u) and the product differently)."""
    src = tmp_path / "h.cc"
    src.write_text(HARNESS)
    exe = tmp_path / "h"
    subprocess.run(["g++", "-O2", "-mfma", "-ffp-contract=fast", "-I", CUDA_INCLUDE, "-I", ORACLE, str(src), "-o", str(exe)],
                   check=True, capture_output=True)
    n, bad_word, bad_uniform, bad_normal = map(int, subprocess.run([str(exe)], check=True, capture_output=True,
                                                                   text=True).stdout.split())
    assert n > 1000 and bad_word == 0 and bad_uniform == 0 and bad_normal == 0, (n, bad_word, bad_uniform, bad_normal)


def aten_desc(**kw):
    args = dict(dtype=C.TDX_BF16, src=C.TDX_SRC_NORMAL, elem_count=4096, seed=7, offset=8, p0=0.0, p1=1.0,
                algo=C.TDX_ALGO_ATEN, aten_stride=256 * 132 * 8)
    args.update(kw)
    return C.make_desc(0x10000, **args)


def prepare(d):
    lib = C.load()
    need = ctypes.c_size_t(0)
    return lib.tdx_init_prepare(ctypes.byref(d), 1, ctypes.byref(need))


GOOD = [dict(dtype=dt, src=src, algo=algo) for dt in (C.TDX_F32, C.TDX_BF16, C.TDX_F16)
        for src in (C.TDX_SRC_UNIFORM, C.TDX_SRC_NORMAL) for algo in (C.TDX_ALGO_ATEN, C.TDX_ALGO_ATEN_WIDE)] + [
    dict(epi=[(C.TDX_EPI_MUL, 2.0), (C.TDX_EPI_ADD, 1.0)]),
    dict(flags=C.TDX_FLAG_WINDOW, window_width=100, window_pitch=1000, elem_count=1000),
    dict(elem_begin=2**31 - 4096), dict(aten_stride=256), dict(elem_count=0, elem_begin=2**40)]
BAD = {
    "stride_zero": dict(aten_stride=0), "stride_not_256": dict(aten_stride=300), "offset_not_4": dict(offset=6),
    "last_element_2^31": dict(elem_begin=2**31 - 4095), "window_last_element": dict(
        flags=C.TDX_FLAG_WINDOW, window_width=100, window_pitch=2**30, elem_count=300),
    "window_w0": dict(flags=C.TDX_FLAG_WINDOW, window_width=0, window_pitch=10),
    "window_p_lt_w": dict(flags=C.TDX_FLAG_WINDOW, window_width=10, window_pitch=5),
    "nolut": dict(algo=C.TDX_ALGO_ATEN | C.TDX_ALGO_NOLUT), "const": dict(src=C.TDX_SRC_CONST, dtype=C.TDX_RAW16, fill_itemsize=2),
    "iota": dict(src=C.TDX_SRC_IOTA), "i64": dict(dtype=C.TDX_I64), "raw16": dict(dtype=C.TDX_RAW16)}


@pytest.mark.parametrize("kw", GOOD, ids=[str(i) for i in range(len(GOOD))])
def test_library_accepts_aten_descriptors(kw):
    assert prepare(aten_desc(**kw)) == 0, C.load().tdx_last_error()


@pytest.mark.parametrize("case", sorted(BAD))
def test_library_rejects_bad_aten_descriptors(case):
    assert prepare(aten_desc(**BAD[case])) == -1  # TDX_E_BADARG


def test_rng_option_is_validated():
    m = deferred_init(lambda: torch.nn.Linear(4, 4))
    with pytest.raises(ValueError, match="rng"):
        materialize_module(m, rng="philox")
    t = deferred_init(lambda: torch.randn(8))
    with pytest.raises(ValueError, match="rng"):
        materialize_tensor(t, rng="ATen")
    with pytest.raises(ValueError, match="rng"):
        _C.materialize_tensors([t], rng="")


def test_aten_on_the_cpu_device_is_the_default():
    """CPU tensors replay ATen's mt19937 stream whatever `rng` says: both equal the eager run."""
    def build():
        return torch.nn.Sequential(torch.nn.Linear(64, 32), torch.nn.Embedding(10, 8, padding_idx=0),
                                   torch.nn.LayerNorm(8))

    torch.manual_seed(3)
    eager = build()
    got = {}
    for rng in ("fused", "aten"):
        torch.manual_seed(3)
        m = deferred_init(build)
        materialize_module(m, rng=rng)
        got[rng] = m
    for (k, a), b, c in zip(eager.state_dict().items(), got["fused"].state_dict().values(),
                            got["aten"].state_dict().values()):
        assert torch.equal(a, b) and torch.equal(a, c), k
