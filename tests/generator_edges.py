"""The generators at edge parameters, where the answer is known exactly (TEST INFRASTRUCTURE, shared by
tests/test_generator_edges_cpu.py and tests/test_generator_edges_gpu.py).

Every case below has a bitwise reference -- signed zeros, infinities and subnormals included -- except the
fp16 normals whose magnitudes leave the normal range ("range" cases), which are held to the float64 bar
of tests/generator_domain.py plus exact signs and exact infinities.  The references:
  const     every element is one value: float32(p) rounded to the dtype.  normal_(m, +-0) and any std
            whose fp32 value is 0 give the mean (q x = +-0, q x + m = m; for m = +0, +-0 + +0 = +0);
            uniform_(a, a) gives a; trunc_normal_'s chain with its scale 0 gives +0 (+-0 + +0).
  signed    normal_(-0.0, 0): the zero takes the sign of the draw (+-0 + -0 keeps it).  16-bit stream:
            -0 iff 1 <= k < 32768, or k == 0 and the tail word's bit 31 is clear (the lower tail).  The
            Box-Muller families: the sign bit of normal_(-0.0, 1) of the same family, which is
            fma(r, d, -0) = r d with its sign, also where r d is an exact zero; and, independently of the
            kernel, the sign of a float64 Box-Muller value of the element's two words wherever that is
            clearly not 0.
  times0    normal_(0, 1).mul_(c), c = +-0: ATen's mul_ on the same family's draw without the step, and
            the sign of z xor that of c (16-bit stream: z(k) as above, +0 at k = 32768; Box-Muller: the
            float64 value).
  zero      uniform_(-0.0, -0.0) and uniform_(-0.0, +0.0): the value 0 with the sign ZERO_SIGN records
            for every family (ATen's CPU kernel gives +0, its CUDA kernel -0; no sign is promised).
  uniform   from + k (to - from) 2^-16 (16-bit stream) or from + float32(w) (to - from) 2^-32 (32-bit
            word w), both exact products, rounded once to fp32 (the kernels' one FMA), clamped to the
            largest value below `to` (of the dtype, or of fp32 for the 32-bit stream: OutTraits::prev),
            then rounded to the dtype.  So never +-0 when to = 0 except where a wide (fp32 stream) form
            rounds its fp32 value -2^-149 to the 16-bit dtype.
  range     fp16 normals that overflow to +-inf or land among the subnormals: the fp16 rounding of a
            value within the polynomial's stated error of float64 (generator_domain.py), +-inf exactly
            where that whole interval rounds beyond 65504, the sign of z(k) on every zero.
"""
import functools
import math

import numpy as np
import torch
from scipy.special import ndtri

import generator_domain as G
import philox_torch as PT
from torchdistx_b200 import _cabi as C

INT = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}
TDX = {torch.float32: C.TDX_F32, torch.bfloat16: C.TDX_BF16, torch.float16: C.TDX_F16}
DTYPES = (torch.float32, torch.bfloat16, torch.float16)
N, U = C.TDX_SRC_NORMAL, C.TDX_SRC_UNIFORM

# trunc_normal_(mean=0, std, a=-2, b=2) as recorded, with its scale std * sqrt(2) set to 0 (trunc_normal_
# itself divides by std): uniform_(2l - 1, 2u - 1), erfinv_, mul_(0), add_(0), clamp_(-2, 2)
TRUNC_L, TRUNC_U = math.erf(-2.0 / math.sqrt(2.0)), math.erf(2.0 / math.sqrt(2.0))
TRUNC0 = [(C.TDX_EPI_ERFINV,), (C.TDX_EPI_MUL, 0.0), (C.TDX_EPI_ADD, 0.0), (C.TDX_EPI_CLAMP, -2.0, 2.0)]
TIMES0 = [(C.TDX_EPI_MUL, 0.0)]
# mul_(-0.0): the sign of every z flipped, -0 at k = 32768 too
NEG_TIMES0 = [(C.TDX_EPI_MUL, -0.0)]
# The same programs through the superset-epilogue kernels: a MULADD step that changes no bit (x * 1 + -0
# is x for every x, +-0 included), or the chain's mul_ and add_ as one MULADD
EXT = {"trunc": [TRUNC0[0], (C.TDX_EPI_MULADD, 0.0, 0.0), TRUNC0[3]],
       "times0": TIMES0 + [(C.TDX_EPI_MULADD, 1.0, -0.0)], "neg_times0": NEG_TIMES0 + [(C.TDX_EPI_MULADD, 1.0, -0.0)]}
KEEP = {"basic": [(C.TDX_EPI_MUL, 1.0)], "ext": [(C.TDX_EPI_MULADD, 1.0, -0.0)]}

# The sign of uniform_(-0.0, to) with to = -0.0 / +0.0 in every generator: fminf(k * 0 + -0, to), and
# k * (+0) + -0 = +0, so the sign is the clamp's: min(+0, -0) = -0 (the minimum of two zeros is -0 on
# the H100's FMNMX and HMNMX2, and in the C library's fminf), min(+0, +0) = +0.  (from, to, sign bit)
ZERO_SIGN = [(-0.0, -0.0, 1), (-0.0, 0.0, 0)]


class Case:
    def __init__(self, kind, src, p0, p1, steps=None, ext=None, sign=None):
        self.kind, self.src, self.p0, self.p1, self.steps, self.ext = kind, src, p0, p1, steps, ext
        self.sign = sign  # `zero`: the sign bit every element has

    @property
    def id(self):
        s = {N: "normal", U: "uniform"}[self.src]
        tag = "" if not self.steps else "+trunc" if self.steps is TRUNC0 else f"+mul({self.steps[0][1]!r})"
        return f"{self.kind}-{s}({self.p0!r},{self.p1!r}){tag}"

    def variants(self, epis=("none", "basic", "ext")):
        """(name, steps): the case without an epilogue and through each epilogue family.  A case that is an
        epilogue program runs as that program (basic) and through the superset kernels (ext)."""
        if self.steps is not None:
            return [(e, self.steps if e == "basic" else self.ext) for e in epis if e != "none"]
        return [(e, [] if e == "none" else KEEP[e]) for e in epis]


def cases(dtype):
    big_n = 6e4 if dtype == torch.float16 else 1e38
    big_u = 65504.0 if dtype == torch.float16 else 1e38
    out = [Case("const", N, m, s) for m in (0.0, 0.25, -3.0, big_n) for s in (0.0, -0.0)]
    out += [Case("const", N, 0.0, 1e-50), Case("const", N, -3.0, 1e-50), Case("signed", N, -0.0, 0.0),
            Case("times0", N, 0.0, 1.0, TIMES0, EXT["times0"]),
            Case("times0", N, 0.0, 1.0, NEG_TIMES0, EXT["neg_times0"]),
            Case("const", U, TRUNC_L, TRUNC_U, TRUNC0, EXT["trunc"])]
    out += [Case("const", U, a, a) for a in (0.0, 0.75, -3.0, big_u)]
    out += [Case("zero", U, a, b, sign=s) for a, b, s in ZERO_SIGN]
    out += [Case("uniform", U, a, b) for a, b in ((-1e-3, 0.0), (-1.0, -0.0), (0.0, 1e-7))]
    if dtype == torch.float16:
        out += [Case("range", N, m, s) for m, s in ((0.0, 2e4), (6e4, 1e4), (0.0, 1e-8), (0.0, 1e-6))]
        out += [Case("uniform", U, a, b) for a, b in ((6e4, 65504.0), (-32000.0, 32000.0))]
    return out


def f32(x):
    return float(np.float32(x))


def const_value(case):
    """The one value of a `const` case, before the store's rounding."""
    if case.steps:  # the trunc chain: (+-0) + (+0)
        return 0.0
    return f32(case.p0)


def full_bits(value, dtype, n, device):
    return torch.full((n,), value, dtype=torch.float32, device=device).to(dtype).view(INT[dtype])


def sign_bits(neg, dtype):
    """Bits of -0 where `neg`, +0 elsewhere."""
    return torch.where(neg, {torch.float32: -2 ** 31}.get(dtype, -2 ** 15), 0).to(INT[dtype])


def lower_half(st):
    """The 16-bit normal's draws below the median: 1 <= k < 32768, or the lower tail (k == 0 and bit 31
    of the tail word clear)."""
    neg = (st.k >= 1) & (st.k < 32768)
    neg[st.k == 0] = (st.tail0 >> 31) & 1 == 0
    return neg


def negative_zero(x):
    return math.copysign(1.0, x) < 0


def check_bm_sign(bits, st, flip, what):
    """Box-Muller families: wherever the float64 Box-Muller value r d of the element's two words is clearly
    away from 0 (r > 1e-3, |d| > 1e-5: beyond the kernel's MUFU error), the output's sign bit is the sign
    of r d, xor `flip`."""
    r, d = st.bm
    sure = (r > 1e-3) & (d.abs() > 1e-5)
    assert float(sure.double().mean()) > 0.999
    bad = sure & ((bits < 0) != ((d < 0) ^ flip))
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} signs that are not those of the float64 Box-Muller value"


class Stream:
    """The engine's stream at global elements g (int64 tensor): 16-bit k, the tail words of the elements
    whose k is 0, 32-bit words -- each decoded once, when first asked for."""

    def __init__(self, seed, offset, g):
        self.seed, self.offset, self.g = seed, offset, g

    @functools.cached_property
    def k(self):
        return PT.halfwords(self.seed, self.offset, self.g)

    @functools.cached_property
    def tail0(self):
        return PT.tail_words(self.seed, self.offset, self.g[self.k == 0])

    @functools.cached_property
    def w(self):
        return PT.words32(self.seed, self.offset, self.g)

    @functools.cached_property
    def bm(self):
        """(r, d) of the float64 Box-Muller value r d of each element of the 32-bit stream: x and y are words
        2j and 2j + 1 of the element's block (j = lane / 2), d = cos for even lanes, sin for odd ones."""
        w = torch.stack(PT.blocks(self.seed, self.offset, self.g >> 2))
        lane = self.g & 3
        x = w.gather(0, (2 * (lane >> 1)).unsqueeze(0)).squeeze(0)
        y = w.gather(0, (2 * (lane >> 1) + 1).unsqueeze(0)).squeeze(0)
        u1 = x.float().double() * 2.0 ** -32 + 2.0 ** -33
        r = torch.sqrt((-2.0 * torch.log(u1)).clamp_min(0.0))
        ang = torch.where(y >= 2 ** 31, y - 2 ** 32, y).double() * (math.pi / 2 ** 31)
        return r, torch.where(lane % 2 == 0, torch.cos(ang), torch.sin(ang))


def assert_bits(got, want, what):
    """Raw bits equal; otherwise how many differ, the most frequent wrong patterns and a few examples."""
    got, want = got.reshape(-1), want.reshape(-1)
    bad = got != want
    if bool(bad.any()):
        m = 0xFFFF if got.element_size() == 2 else 0xFFFFFFFF
        pat, cnt = torch.unique(got[bad], return_counts=True)
        top = sorted(zip(cnt.tolist(), pat.tolist()), reverse=True)[:3]
        i = bad.nonzero()[:3].flatten()
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} elements differ; most frequent wrong bits "
                             f"{[(hex(p & m), c) for c, p in top]}; e.g. got {[hex(x & m) for x in got[i].tolist()]} "
                             f"want {[hex(x & m) for x in want[i].tolist()]}")


def check(case, dtype, wide, bits, st, raw, what):
    """bits (integer view of one output) against the case's reference.  st: the Stream of its elements;
    raw(p0, p1): the same family's output for other parameters, without epilogue steps.  Returns the k
    table of a `range` case."""
    native16 = dtype != torch.float32 and not wide
    dev = bits.device
    if case.kind == "const":
        assert_bits(bits, full_bits(const_value(case), dtype, bits.numel(), dev), what)
    elif case.kind == "signed":
        if native16:
            assert_bits(bits, sign_bits(lower_half(st), dtype), what)
        else:
            assert_bits(bits, sign_bits(raw(-0.0, 1.0) < 0, dtype), what)
            check_bm_sign(bits, st, False, what)
    elif case.kind == "times0":
        c = case.steps[0][1]
        assert_bits(bits, raw(case.p0, case.p1).view(dtype).mul(c).view(INT[dtype]), what + " (ATen mul_ on the draw)")
        if native16:
            assert_bits(bits, sign_bits(lower_half(st) ^ negative_zero(c), dtype), what + " (sign of z(k))")
        else:
            check_bm_sign(bits, st, negative_zero(c), what)
    elif case.kind == "zero":
        assert_bits(bits, sign_bits(torch.full(bits.shape, bool(case.sign), device=dev), dtype),
                    what)
    elif case.kind == "uniform":
        want = uniform_expected(dtype, wide, case.p0, case.p1, k=st.k if native16 else None,
                                w=None if native16 else st.w)
        assert_bits(bits, want, what)
        check_uniform_bounds(bits, dtype, case.p0, case.p1, wide)
    else:  # range
        assert native16
        table = G.table_of(bits.to(torch.int64) & 0xFFFF, st.k, skip_zero=True)
        check_range_table(table, case.p0, case.p1)
        check_range_tails(to_np16(bits[st.k == 0]), st.tail0.cpu().numpy(), case.p0, case.p1)
        return table
    return None


def prev_of(to, dtype):
    """OutTraits<dtype>::prev: the largest value of the dtype below `to` (fp32 bits for bf16)."""
    if dtype == torch.bfloat16:
        b = int(np.float32(to).view(np.uint32))
        step = 0x10000
        if to > 0:
            return float(np.uint32(b - step).view(np.float32))
        if to < 0:
            return float(np.uint32(b + step).view(np.float32))
        return float(np.uint32(0x80010000).view(np.float32))
    if dtype == torch.float32:
        b, one, conv = int(np.float32(to).view(np.uint32)), 1, lambda x: float(np.uint32(x).view(np.float32))
        if to > 0:
            return conv(b - one)
        if to < 0:
            return conv(b + one)
        return conv(0x80000001)
    h = int(np.float16(np.float32(to)).view(np.uint16))
    conv = lambda x: float(np.uint16(x).view(np.float16))  # noqa: E731
    if to > 0:
        return conv(h - 1)
    if to < 0:
        return conv(h + 1)
    return conv(0x8001)


def f32_of_sum(a, b):
    """fp32 rounding (nearest even) of the exact sum of float64 tensors a and b: the float64 sum, its
    rounding error (TwoSum), and the error breaks the ties the float64 sum created."""
    s = a + b
    bb = s - a
    err = (a - (s - bb)) + (b - bb)
    r = s.float()
    up = torch.nextafter(r, torch.full_like(r, math.inf))
    dn = torch.nextafter(r, torch.full_like(r, -math.inf))
    r = torch.where((s == (r.double() + up.double()) / 2) & (err > 0), up, r)
    return torch.where((s == (r.double() + dn.double()) / 2) & (err < 0), dn, r)


def uniform_expected(dtype, wide, lo, hi, k=None, w=None):
    """Bits of the `uniform` reference for 16-bit stream k (native 16-bit) or 32-bit words w (fp32 and
    the wide 16-bit forms)."""
    f, t = np.float32(lo), np.float32(hi)
    rng = float(np.float32(t - f))
    if wide or dtype == torch.float32:
        kf, scale, prev = w.float().double(), rng * 2.0 ** -32, prev_of(float(t), torch.float32)
    else:
        kf, scale, prev = k.double(), rng * 2.0 ** -16, prev_of(float(t), dtype)
    v = f32_of_sum(torch.full_like(kf, float(f)), kf * scale)
    v = torch.minimum(v, torch.tensor(prev if t > f else float(t), dtype=torch.float32, device=v.device))
    return v.to(dtype).view(INT[dtype])


def check_uniform_bounds(bits, dtype, lo, hi, wide):
    """Every value lies in [from, to) as real numbers (the dtype's rounding of `from` below)."""
    v = bits.view(dtype).double()
    lo_d = float(torch.tensor(f32(lo)).to(dtype))
    assert bool((v >= lo_d).all()), float(v.min())
    if not wide:  # (a wide form rounds its fp32 value: `to` itself is a possible result)
        assert bool((v < f32(hi)).all()), float(v.max())
        if f32(hi) == 0.0:
            assert not bool((v == 0).any()), "a zero from a range that ends at 0"


OVF16 = 65520.0  # fp16 rounds to +-inf at and beyond this magnitude


def round16(x):
    """fp16 rounding of float64 values (numpy), +-inf beyond the range."""
    r = G.round_to(x, torch.float16)
    return np.where(np.abs(x) >= OVF16, np.copysign(np.inf, x), r)


def check_range_table(table, mean, std):
    """The `range` bar over k = 1 ... 65535 (fp16 bits of each k, numpy)."""
    k = np.arange(1, 65536, dtype=np.float64)
    got = G.as_f64(table[1:], torch.float16)
    ref = G.normal_ref(k, mean, std)
    z = np.abs(ref - mean) / std
    slack = G.ICDF_REL_ERR * std * z + 8 * G.EPS32 * (abs(mean) + std * z) + 1e-300
    lo_e, hi_e = round16(ref - slack), round16(ref + slack)
    ok = (got >= lo_e) & (got <= hi_e)
    assert ok.all(), ("beyond the stated error", ref[~ok][:4], got[~ok][:4])
    assert (got[1:] >= got[:-1]).all(), "not non-decreasing in k"
    neg = (table[1:].astype(np.int64) & 0x8000) != 0
    assert (neg[ref != mean] == (ref[ref != mean] < 0)).all(), "a sign that is not the sign of the value"
    assert table[32768] == int(np.float16(mean).view(np.uint16)), hex(int(table[32768]))


def check_range_tails(bits, words, mean, std):
    """The k == 0 elements of a `range` case: within 1 ulp of float64, +-inf exactly beyond the range."""
    got = G.as_f64(bits, torch.float16)
    w = np.asarray(words, dtype=np.int64)
    p = ((w & 0x7FFFFFFF).astype(np.float64) + 0.5) * 2.0 ** -31 * 2.0 ** -17
    ref = mean + std * np.where(w & 0x80000000, 1.0, -1.0) * -ndtri(p)
    slack = 8 * G.EPS32 * np.abs(ref)
    lo_e, hi_e = round16(ref - slack), round16(ref + slack)
    assert ((got >= lo_e) & (got <= hi_e)).all(), (ref[:4], got[:4])
    neg = (np.asarray(bits).astype(np.int64) & 0x8000) != 0
    assert (neg == (ref < 0)).all()


def to_np16(bits):
    return (bits.to(torch.int64) & 0xFFFF).cpu().numpy()
