/*
 * tdx_oracle.c -- CPU restatement of the fused initialisation kernels (TEST INFRASTRUCTURE).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this file; the
 * product (torchdistx_b200) never does and has no CPU path for CUDA tensors.
 *
 * What is restated, and against what it is pinned:
 *   philox4x32_R     the Philox4x32 generator ATen/curand use on CUDA (tdx_philox.c).  Published
 *                    algorithm: Salmon, Moraes, Dror, Shaw, SC'11 (Random123 1.x).  Dependency of
 *                    the reference path: PyTorch (un-vendored; pinned here: torch 2.11.0+cu128,
 *                    $TORCH/include/ATen/core/PhiloxRNGEngine.h:60-220).  Pinned by
 *                    tests/golden/philox_kat.json = Random123 known-answer vectors + outputs of
 *                    at::Philox4_32 itself (tests/golden/make_philox_kat.py).
 *   transforms       element g of a tensor := f(seed, offset, g) exactly as
 *                    torchdistx_b200/csrc/kernels compute it, for every descriptor of
 *                    include/tdx_init.h (tdx_oracle_generate): constants, the fused uniform and
 *                    normal generators, windows, index programs, sinusoid tables, copies of host
 *                    arrays, band masks and every epilogue step.  libm stands in for the MUFU
 *                    approximations (lg2/sqrt/sin/cos) and for libdevice's exp/log/expm1/erfinv, so
 *                    those floats agree to the tolerances the tests state, and everything else
 *                    (constants, uniform, rounding, epilogue arithmetic, sharding) bit for bit.
 *   ATen's stream    TDX_ALGO_ATEN(_WIDE) draws: the unit uniform / normal of each element
 *                    (tdx_oracle_aten_units, on tdx_philox.c); tdx_oracle_generate rejects them.
 *   semantics        what uniform_/normal_/fill_ MEAN follows ATen, the arithmetic owner of the
 *                    reference's replay (reference src/cc/torchdistx/deferred_init.cc:218-220):
 *                    bounds cast to the tensor dtype, value = u*(to-from)+from, half-open range
 *                    ($TORCH/include/ATen/native/cuda/DistributionTemplates.h:428-470,
 *                     $TORCH/include/ATen/core/TransformationHelper.h:84-99).
 *                    The element-wise random STREAM is this engine's own (shard-invariant Philox
 *                    indexing); agreement with the reference's CPU mt19937 stream is
 *                    distributional and checked against oracle/_ref in tests/.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "tdx_init.h"
#include "tdx_philox.c"

/* the engine's counter layout (include/tdx_init.h "Random stream specification") */
static void block_of(const TdxInitDesc* d, uint64_t blk, uint32_t wflag, uint32_t out[4]) {
  const uint32_t ctr[4] = {(uint32_t)d->philox_offset, (uint32_t)(blk >> 32),
                           (uint32_t)(d->philox_offset >> 32) | 0x80000000u | wflag, (uint32_t)blk};
  const uint32_t key[2] = {(uint32_t)d->philox_seed, (uint32_t)(d->philox_seed >> 32)};
  tdx_oracle_philox4x32(ctr, key, 10, out);
}

/* ---- dtype helpers ------------------------------------------------------------------------- */
static float bits_f(uint32_t b) { float f; memcpy(&f, &b, 4); return f; }
static uint32_t f_bits(float f) { uint32_t b; memcpy(&b, &f, 4); return b; }

static uint16_t f32_to_bf16(float f) { /* round to nearest even */
  uint32_t b = f_bits(f);
  if ((b & 0x7fffffffu) > 0x7f800000u) return 0x7fff;
  b += 0x7fffu + ((b >> 16) & 1u);
  return (uint16_t)(b >> 16);
}
static float bf16_to_f32(uint16_t h) { return bits_f((uint32_t)h << 16); }
static uint16_t f32_to_f16(float f) { _Float16 h = (_Float16)f; uint16_t b; memcpy(&b, &h, 2); return b; }
static float f16_to_f32(uint16_t b) { _Float16 h; memcpy(&h, &b, 2); return (float)h; }

static float round_through(float v, int dtype) {
  if (dtype == TDX_BF16) return bf16_to_f32(f32_to_bf16(v));
  if (dtype == TDX_F16) return f16_to_f32(f32_to_f16(v));
  return v;
}
/* largest representable value of `dtype` strictly below `to` (kernel: OutTraits<>::prev) */
static float prev_of(float to, int dtype) {
  if (dtype == TDX_F32) {
    if (to > 0.f) return bits_f(f_bits(to) - 1);
    if (to < 0.f) return bits_f(f_bits(to) + 1);
    return bits_f(0x80000001u);
  }
  if (dtype == TDX_BF16) {
    if (to > 0.f) return bits_f(f_bits(to) - 0x10000u);
    if (to < 0.f) return bits_f(f_bits(to) + 0x10000u);
    return bits_f(0x80010000u);
  }
  {
    const uint16_t h = f32_to_f16(to);
    if (to > 0.f) return f16_to_f32((uint16_t)(h - 1));
    if (to < 0.f) return f16_to_f32((uint16_t)(h + 1));
    return f16_to_f32(0x8001);
  }
}

/* ---- inverse normal CDF in double (Wichura, AS 241, PPND16): used for the rare tail bin and for
 * erfinv in the epilogue; relative accuracy ~1e-16, far below the fp32 the kernel works in. ------- */
static double ndtri(double p) {
  static const double a[8] = {3.3871328727963666080e0, 1.3314166789178437745e+2, 1.9715909503065514427e+3,
                              1.3731693765509461125e+4, 4.5921953931549871457e+4, 6.7265770927008700853e+4,
                              3.3430575583588128105e+4, 2.5090809287301226727e+3};
  static const double b[8] = {1.0, 4.2313330701600911252e+1, 6.8718700749205790830e+2,
                              5.3941960214247511077e+3, 2.1213794301586595867e+4, 3.9307895800092710610e+4,
                              2.8729085735721942674e+4, 5.2264952788528545610e+3};
  static const double c[8] = {1.42343711074968357734e0, 4.63033784615654529590e0, 5.76949722146069140550e0,
                              3.64784832476320460504e0, 1.27045825245236838258e0, 2.41780725177450611770e-1,
                              2.27238449892691845833e-2, 7.74545014278341407640e-4};
  static const double d[8] = {1.0, 2.05319162663775882187e0, 1.67638483018380384940e0,
                              6.89767334985100004550e-1, 1.48103976427480074590e-1, 1.51986665636164571966e-2,
                              5.47593808499534494600e-4, 1.05075007164441684324e-9};
  static const double e[8] = {6.65790464350110377720e0, 5.46378491116411436990e0, 1.78482653991729133580e0,
                              2.96560571828504891230e-1, 2.65321895265761230930e-2, 1.24266094738807843860e-3,
                              2.71155556874348757815e-5, 2.01033439929228813265e-7};
  static const double f[8] = {1.0, 5.99832206555887937690e-1, 1.36929880922735805310e-1,
                              1.48753612908506148525e-2, 7.86869131145613259100e-4, 1.84631831751005468180e-5,
                              1.42151175831644588870e-7, 2.04426310338993978564e-15};
  const double q = p - 0.5;
  double r, num, den;
  int i;
  if (p <= 0.0 || p >= 1.0) return p == 0.0 ? -INFINITY : p == 1.0 ? INFINITY : NAN; /* erfinv(-1) = -inf */
  if (fabs(q) <= 0.425) {
    r = 0.180625 - q * q;
    num = a[7]; den = b[7];
    for (i = 6; i >= 0; --i) { num = num * r + a[i]; den = den * r + b[i]; }
    return q * num / den;
  }
  r = q < 0 ? p : 1.0 - p;
  r = sqrt(-log(r));
  if (r <= 5.0) {
    r -= 1.6;
    num = c[7]; den = d[7];
    for (i = 6; i >= 0; --i) { num = num * r + c[i]; den = den * r + d[i]; }
  } else {
    r -= 5.0;
    num = e[7]; den = f[7];
    for (i = 6; i >= 0; --i) { num = num * r + e[i]; den = den * r + f[i]; }
  }
  return q < 0 ? -num / den : num / den;
}

/* kernel: apply_epi<Out> (and, for index programs, sinusoid columns and fp32 copies, apply_epi<float>:
 * `dtype` is the type each step rounds to).  expf / logf / expm1f and the double ndtri for erfinv are
 * C libm's, each within a few ulp of the CUDA libdevice functions the kernels call, not their bits. */
static float apply_epi(const TdxInitDesc* d, float v, int dtype) {
  if (!(d->reserved & TDX_FLAG_SRC_NOROUND)) v = round_through(v, dtype);
  for (int i = 0; i < d->n_epi && i < TDX_MAX_EPI; ++i) {
    const uint32_t op = d->epi[i].op;
    const int rnd = !(op & TDX_EPI_NOROUND);
    const float a = d->epi[i].a, b = d->epi[i].b;
    switch (op & 0xffu) {
      case TDX_EPI_MUL: v = v * a; break;
      case TDX_EPI_ADD: v = v + a; break;
      case TDX_EPI_ERFINV: v = (float)(ndtri(((double)v + 1.0) * 0.5) * 0.70710678118654752440); break;
      case TDX_EPI_CLAMP: v = isnan(v) ? v : fminf(fmaxf(v, a), b); break; /* clamp_ keeps a NaN */
      case TDX_EPI_RPOW: v = powf(a, v); break; /* libm vs CUDA powf: both ~1 ulp, not each other's bits */
      case TDX_EPI_RECIP: v = 1.0f / v; break;
      case TDX_EPI_EXP: v = expf(v); break;
      case TDX_EPI_LOG: v = logf(v); break;
      case TDX_EPI_EXPM1: v = expm1f(v); break;
      case TDX_EPI_INV_SOFTPLUS: { /* v + log(-expm1(-v)), rounded after each ATen op */
        float t = expm1f(-v);
        if (rnd) t = round_through(t, dtype);
        t = logf(-t);
        if (rnd) t = round_through(t, dtype);
        v = v + t;
        break;
      }
      case TDX_EPI_MULADD:
        v = v * a;
        if (rnd) v = round_through(v, dtype);
        v = v + b;
        break;
      default: break;
    }
    if (rnd) v = round_through(v, dtype);
  }
  return v;
}

static uint32_t halfword(const uint32_t w[4], int e) { return (w[e >> 1] >> (16 * (e & 1))) & 0xffffu; }

/* kernel: icdf16_tail */
static float icdf16_tail(uint32_t word) {
  const float sgn = (word & 0x80000000u) ? 1.0f : -1.0f;
  const float p = ((float)(word & 0x7fffffffu) + 0.5f) * 4.656612873077393e-10f * 7.62939453125e-06f;
  return sgn * -(float)ndtri((double)p);
}

/* kernel: box_muller32 */
static void box_muller32(uint32_t x, uint32_t y, float* r, float* c, float* s) {
  const float u1 = fmaf((float)x, 2.3283064365386963e-10f, 1.1641532182693481e-10f);
  *r = sqrtf(-1.3862943611198906f * log2f(u1));
  const float ang = (float)(int32_t)y * 1.4629180792671596e-09f; /* y signed, times pi / 2^31 */
  *c = cosf(ang);
  *s = sinf(ang);
}

static int resolve_algo(const TdxInitDesc* d) {
  const int a = d->algo & 0x0f;
  if (d->src == TDX_SRC_NORMAL) return a ? a : (d->dtype == TDX_F32 ? TDX_ALGO_BM32 : TDX_ALGO_ICDF16);
  if (d->src == TDX_SRC_UNIFORM && d->dtype != TDX_F32 && a == TDX_ALGO_WIDE32) return TDX_ALGO_WIDE32;
  return 0;
}

/* The generated value (fp32, before any epilogue step) of GLOBAL element g of a random descriptor. */
static float element(const TdxInitDesc* d, uint64_t g) {
  const int algo = resolve_algo(d);
  uint32_t w[4];
  float v = 0.f;
  if (d->src == TDX_SRC_UNIFORM) {
    const float from = (float)d->p0, to = (float)d->p1;
    /* the wide form of a 16-bit output keeps fp32 bounds (kernel: GenUniform32<Out>) */
    const int wide = d->dtype == TDX_F32 || algo == TDX_ALGO_WIDE32;
    const float to_prev = to > from ? prev_of(to, wide ? TDX_F32 : d->dtype) : to;
    if (wide) {
      block_of(d, g / 4, 0, w);
      const float k = (float)w[g % 4]; /* all 32 bits, round to nearest (kernel: I2FP) */
      v = fminf(fmaf(k, (to - from) * 2.3283064365386963e-10f, from), to_prev);
    } else {
      block_of(d, g / 8, 0, w);
      const float k = (float)halfword(w, (int)(g % 8));
      v = fminf(fmaf(k, (to - from) * 1.52587890625e-05f, from), to_prev);
    }
  } else { /* TDX_SRC_NORMAL */
    const float mean = (float)d->p0, std = (float)d->p1;
    if (algo == TDX_ALGO_BM32) {
      float r[2], dir[4];
      block_of(d, g / 4, 0, w);
      box_muller32(w[0], w[1], &r[0], &dir[0], &dir[1]);
      box_muller32(w[2], w[3], &r[1], &dir[2], &dir[3]);
      v = fmaf(r[(g % 4) >> 1] * std, dir[g % 4], mean);
    } else { /* TDX_ALGO_ICDF16 */
      const int e = (int)(g % 8);
      block_of(d, g / 8, 0, w);
      const uint32_t k = halfword(w, e);
      if (k == 0) {
        uint32_t t[4];
        block_of(d, g / 8, e < 4 ? 0x40000000u : 0x20000000u, t);
        v = fmaf(icdf16_tail(t[e & 3]), std, mean);
      } else {
        const float x = fmaf(8388608.0f + (float)k, 3.0517578125e-05f, -257.0f);
        const float t1 = fmaf(-x, x, 1.0f);
        const float l = log2f(t1);
        float q = fmaf(std * 0x1.152c90p-19f, l, std * 0x1.9c35c0p-14f);
        q = fmaf(q, l, std * 0x1.bfaecap-10f);
        q = fmaf(q, l, std * 0x1.26ef76p-7f);
        q = fmaf(q, l, std * -0x1.d03266p-3f);
        q = fmaf(q, l, std * 0x1.40de66p+0f);
        v = fmaf(q, x, mean);
      }
    }
  }
  return v;
}

static int itemsize(int dtype) {
  switch (dtype) {
    case TDX_RAW8: return 1;
    case TDX_RAW16: case TDX_BF16: case TDX_F16: return 2;
    case TDX_RAW32: case TDX_F32: return 4;
    case TDX_RAW64: case TDX_I64: return 8;
    default: return 0;
  }
}

static int is_float(int dtype) { return dtype == TDX_F32 || dtype == TDX_BF16 || dtype == TDX_F16; }

/* the store of a float output: one rounding */
static void store_float(const TdxInitDesc* d, void* out, uint64_t i, float v) {
  if (d->dtype == TDX_F32) ((float*)out)[i] = v;
  else if (d->dtype == TDX_BF16) ((uint16_t*)out)[i] = f32_to_bf16(v);
  else ((uint16_t*)out)[i] = f32_to_f16(v);
}

/* kernel: tdx_init_sincos.cu sincos_value.  sinf / cosf are C libm's, each within an ulp or two of the
 * CUDA libdevice functions the kernel calls, not their bits. */
static float sincos_element(const TdxInitDesc* d, uint64_t g) {
  const uint64_t half = d->fill_bits[0], width = 2 * half;
  const uint64_t r = g / width, c = g % width;
  const int second = c >= half;
  const uint64_t k = second ? c - half : c;
  float f = (float)((int64_t)d->p0 + (int64_t)k * (int64_t)d->p1);
  if (d->n_epi) f = apply_epi(d, f, TDX_F32); /* the column program runs in fp32 */
  const float x = (float)r * f;
  const int cos_first = (d->fill_bits[1] & TDX_SINCOS_COS_FIRST) != 0;
  return second != cos_first ? cosf(x) : sinf(x);
}

/*
 * Fills `out` (host memory, elem_count elements of the descriptor's dtype) with what the GPU
 * kernels write for this descriptor.  Returns 0, or -1 for a descriptor outside the restatement:
 * ATen's stream included (tdx_oracle_aten_units restates its draws).
 */
int tdx_oracle_generate(const TdxInitDesc* d, void* out) {
  if (d->algo & ~(0x0f | TDX_ALGO_NOLUT)) return -1; /* the library rejects unknown flags too */
  if (d->reserved & TDX_FLAG_WINDOW) {
    /* the plain descriptors of its runs: run o is global elements [elem_begin + o * P, + W), written
     * at local o * W */
    const uint64_t W = d->fill_bits[0], P = d->fill_bits[1];
    const int isz = itemsize(d->dtype);
    if ((d->src != TDX_SRC_UNIFORM && d->src != TDX_SRC_NORMAL) || W == 0 || P < W) return -1;
    for (uint64_t l = 0; l < d->elem_count; l += W) {
      TdxInitDesc run = *d;
      run.reserved &= ~TDX_FLAG_WINDOW;
      run.fill_bits[0] = run.fill_bits[1] = 0;
      run.elem_begin = d->elem_begin + (l / W) * P;
      run.elem_count = d->elem_count - l < W ? d->elem_count - l : W;
      if (tdx_oracle_generate(&run, (unsigned char*)out + l * isz)) return -1;
    }
    return 0;
  }
  switch (d->src) {
    case TDX_SRC_CONST: {
      const int isz = itemsize(d->dtype);
      unsigned char pat[16];
      if (!isz) return -1;
      memcpy(pat, d->fill_bits, 16);
      for (uint64_t i = 0; i < d->elem_count; ++i) memcpy((unsigned char*)out + i * isz, pat, isz);
      return 0;
    }
    case TDX_SRC_IOTA: { /* element g = p0 + g * p1 (integers), then the fp32 epilogue */
      /* broadcast (fill_bits = {P, R}, P > 0): global element g indexes (g / R) % P */
      const int64_t start = (int64_t)d->p0, step = (int64_t)d->p1;
      const uint64_t period = d->fill_bits[0], repeat = d->fill_bits[1] ? d->fill_bits[1] : 1;
      if (!(is_float(d->dtype) || (d->dtype == TDX_I64 && d->n_epi == 0))) return -1;
      for (uint64_t i = 0; i < d->elem_count; ++i) {
        uint64_t g = d->elem_begin + i;
        if (period) g = (g / repeat) % period;
        const int64_t val = start + (int64_t)g * step;
        if (d->dtype == TDX_I64) { ((int64_t*)out)[i] = val; continue; }
        float v = (float)val;
        if (d->n_epi) v = apply_epi(d, v, TDX_F32); /* index programs run in fp32 whatever the output type */
        store_float(d, out, i, v);
      }
      return 0;
    }
    case TDX_SRC_SINCOS:
      if (!is_float(d->dtype)) return -1;
      if (d->fill_bits[0] == 0 || (d->fill_bits[1] & ~(uint64_t)TDX_SINCOS_COS_FIRST)) return -1;
      if (d->elem_count && (d->elem_begin + d->elem_count - 1) / (2 * d->fill_bits[0]) >= (1ull << 24)) return -1;
      for (uint64_t i = 0; i < d->elem_count; ++i) store_float(d, out, i, sincos_element(d, d->elem_begin + i));
      return 0;
    case TDX_SRC_GATHER: { /* kernel: tdx_init_gather.cu gather_tiles; the source is a host address here */
      const void* src = (const void*)(uintptr_t)d->fill_bits[0];
      const uint64_t period = d->fill_bits[1] & 0xffffffffull, rep = d->fill_bits[1] >> 32;
      if (!(is_float(d->dtype) || (d->dtype == TDX_I64 && d->n_epi == 0))) return -1;
      if (src == NULL || d->algo || d->reserved || (period == 0 && rep != 0)) return -1;
      for (uint64_t j = 0; j < d->elem_count; ++j) {
        const uint64_t g = d->elem_begin + j;
        const uint64_t i = period ? (g / (rep ? rep : 1)) % period : g;
        if (d->dtype == TDX_I64) {
          ((uint64_t*)out)[j] = ((const uint64_t*)src)[i];
        } else if (d->dtype == TDX_F32) {
          float v = ((const float*)src)[i];
          if (d->n_epi) v = apply_epi(d, v, TDX_F32);
          memcpy((uint32_t*)out + j, &v, 4); /* (the bits as they are without an epilogue) */
        } else {
          const uint16_t w = ((const uint16_t*)src)[i];
          if (!d->n_epi) {
            ((uint16_t*)out)[j] = w;
            continue;
          }
          const float v = d->dtype == TDX_BF16 ? bf16_to_f32(w) : f16_to_f32(w);
          store_float(d, out, j, apply_epi(d, v, d->dtype));
        }
      }
      return 0;
    }
    case TDX_SRC_BAND: { /* kernel: tdx_init_band.cu band_tiles, element by element with its own division */
      const int isz = itemsize(d->dtype);
      const uint64_t C = d->fill_bits[0] & 0xffffffffull, R = d->fill_bits[0] >> 32;
      const int64_t lo = (int32_t)(uint32_t)d->fill_bits[1], hi = (int32_t)(uint32_t)(d->fill_bits[1] >> 32);
      if (!isz || C == 0 || R == 0 || C >= (1ull << 31) || R >= (1ull << 31) || lo > hi || d->n_epi || d->algo ||
          d->reserved)
        return -1;
      for (uint64_t j = 0; j < d->elem_count; ++j) {
        const uint64_t g = d->elem_begin + j;
        const int64_t c = (int64_t)(g % C), r = (int64_t)((g / C) % R);
        const uint64_t v = (lo <= c - r && c - r <= hi) ? d->philox_seed : d->philox_offset;
        memcpy((unsigned char*)out + j * isz, &v, (size_t)isz); /* (the low bytes: little-endian) */
      }
      return 0;
    }
    case TDX_SRC_UNIFORM:
    case TDX_SRC_NORMAL: {
      const int algo = resolve_algo(d);
      if (!is_float(d->dtype)) return -1;
      if ((d->algo & 0x0f) == TDX_ALGO_ATEN || (d->algo & 0x0f) == TDX_ALGO_ATEN_WIDE) return -1;
      if (d->src == TDX_SRC_NORMAL && algo != TDX_ALGO_BM32 && !(algo == TDX_ALGO_ICDF16 && d->dtype != TDX_F32))
        return -1;
      for (uint64_t i = 0; i < d->elem_count; ++i) {
        float v = element(d, d->elem_begin + i);
        if (d->n_epi) v = apply_epi(d, v, d->dtype);
        store_float(d, out, i, v);
      }
      return 0;
    }
    default:
      return -1;
  }
}

/*
 * ATen's stream (TDX_ALGO_ATEN, TDX_ALGO_ATEN_WIDE): out[l] = the unit draw -- aten_uniform01 or
 * aten_normal01, before ATen's transform and the epilogue -- of local element l's global index, under
 * the descriptor's window (fill_bits[0] = W | P << 32) if it has one; fill_bits[1] = S.  Returns 0, or
 * -1 for another descriptor, S == 0, a bad window or a last global element >= 2^31.
 */
int tdx_oracle_aten_units(const TdxInitDesc* d, float* out) {
  const int window = (d->reserved & TDX_FLAG_WINDOW) != 0;
  const uint64_t W = window ? (d->fill_bits[0] & 0xffffffffull) : 1, P = window ? d->fill_bits[0] >> 32 : 1;
  const uint32_t S = (uint32_t)d->fill_bits[1];
  if ((d->src != TDX_SRC_UNIFORM && d->src != TDX_SRC_NORMAL) ||
      (d->algo != TDX_ALGO_ATEN && d->algo != TDX_ALGO_ATEN_WIDE) || S == 0 || W == 0 || P < W)
    return -1;
  if (d->elem_count && d->elem_begin + ((d->elem_count - 1) / W) * P + (d->elem_count - 1) % W >= (1ull << 31))
    return -1;
  for (uint64_t l = 0; l < d->elem_count; ++l) {
    const uint32_t g = (uint32_t)(d->elem_begin + (l / W) * P + l % W);
    out[l] = d->src == TDX_SRC_NORMAL ? aten_normal01(d->philox_seed, d->philox_offset, S, g)
                                      : aten_uniform01(d->philox_seed, d->philox_offset, S, g);
  }
  return 0;
}

/* Philox blocks one RNG op consumes from the generator (planner.cc assign_rng). */
uint64_t tdx_oracle_offset_increment(uint64_t numel) {
  const uint64_t blocks = (numel + 3) / 4;
  return ((blocks + 3) / 4) * 4 + 4;
}
