"""The C restatement (oracle/tdx_oracle.c) at the generators' edge parameters, without a GPU: the cases and
exact references of tests/generator_edges.py at 2^20 elements each (2^22 where every k must occur), through the native 16-bit stream, the
wide (fp32 stream) 16-bit forms and fp32, without an epilogue and with one that changes no bit.  This pins
the answers tests/test_generator_edges_gpu.py holds the kernels to, sign rules included.  (The superset
epilogue's steps are the kernels' alone: the restatement has none of them.)"""
import numpy as np
import pytest
import torch

import generator_edges as E
from oracle import tdx_oracle as O
from torchdistx_b200 import _cabi as C

SEED, OFFSET = 0x1234_5678_9ABC, 0x1_0000_0040
_streams = {}


def size(case):
    return 1 << 22 if case.kind == "range" else 1 << 20


def stream(n):
    if n not in _streams:
        _streams[n] = E.Stream(SEED, OFFSET, torch.arange(n, dtype=torch.int64))
    return _streams[n]


def draw(case, dtype, wide, steps, p0=None, p1=None):
    if wide:
        algo = C.TDX_ALGO_WIDE32
    else:
        algo = (C.TDX_ALGO_ICDF16 if dtype != torch.float32 else C.TDX_ALGO_BM32) if case.src == E.N else 0
    d = C.make_desc(0, dtype=E.TDX[dtype], src=case.src, elem_count=size(case), seed=SEED, offset=OFFSET,
                    p0=case.p0 if p0 is None else p0, p1=case.p1 if p1 is None else p1, algo=algo, epi=steps)
    out = O.generate(d)
    return torch.from_numpy(out.view(np.int32 if dtype == torch.float32 else np.int16))


PARAMS = [(dt, wide, c) for dt in E.DTYPES for wide in ((False, True) if dt != torch.float32 else (False,))
          for c in E.cases(dt) if not (wide and c.kind == "range")]


@pytest.mark.parametrize("dtype,wide,case", PARAMS,
                         ids=[f"{str(dt)[6:]}-{'wide' if w else 'native'}-{c.id}" for dt, w, c in PARAMS])
def test_restatement_gives_the_exact_answer(dtype, wide, case):
    for epi, steps in case.variants(("none", "basic")):
        bits = draw(case, dtype, wide, steps)
        raw = lambda p0, p1: draw(case, dtype, wide, [], p0, p1)  # noqa: E731
        E.check(case, dtype, wide, bits, stream(size(case)), raw, f"{dtype} {'wide' if wide else 'native'} {case.id} {epi}")

