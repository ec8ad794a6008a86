/*
 * tdx_philox.c -- Philox4x32 and ATen's CUDA random stream on it (TEST INFRASTRUCTURE: part of
 * libtdx_oracle, which includes this file whole).  Self-contained, so that
 * tests/test_aten_stream_cpu.py can build it alone beside curand's host code and pin it there.
 *
 *   tdx_oracle_philox4x32   Philox4x32-R (Salmon, Moraes, Dror, Shaw, SC'11): the generator of both
 *                           the engine's stream and ATen's (curand's curand_Philox4x32_10, R = 10).
 *   aten_*                  ATen's CUDA stream (include/tdx_init.h, "ATen stream"): the map of
 *                           element g to (t, k, j), the uniform lanes, and the Box-Muller normal
 *                           through libm (the device uses __sincosf: a few ulp apart).
 */
#include <math.h>
#include <stdint.h>

#define PHILOX_M0 0xD2511F53u
#define PHILOX_M1 0xCD9E8D57u
#define PHILOX_W0 0x9E3779B9u
#define PHILOX_W1 0xBB67AE85u

/* out[4] = Philox4x32-`rounds`(counter ctr[4], key[2]) */
void tdx_oracle_philox4x32(const uint32_t ctr[4], const uint32_t key[2], int rounds, uint32_t out[4]) {
  uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3], k0 = key[0], k1 = key[1];
  for (int r = 0; r < rounds; ++r) {
    const uint64_t p0 = (uint64_t)c0 * PHILOX_M0, p1 = (uint64_t)c2 * PHILOX_M1;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += PHILOX_W0; k1 += PHILOX_W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

/* the block element g takes its lane from: counter (o/4 + k, t), key = seed; returns lane j */
static int aten_block(uint64_t seed, uint64_t offset, uint32_t S, uint32_t g, uint32_t x[4]) {
  const uint32_t t = g % S, q = g / S, k = q / 4;
  const uint64_t ctr = offset / 4 + k;
  const uint32_t c[4] = {(uint32_t)ctr, (uint32_t)(ctr >> 32), t, 0};
  const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  tdx_oracle_philox4x32(c, key, 10, x);
  return (int)(q % 4);
}

uint32_t aten_word(uint64_t seed, uint64_t offset, uint32_t S, uint32_t g) {
  uint32_t x[4];
  return x[aten_block(seed, offset, S, g, x)];
}

/* curand_uniform4's lane: x * 2^-32 + 2^-33, one FMA (as nvcc contracts it) */
float aten_uniform01(uint64_t seed, uint64_t offset, uint32_t S, uint32_t g) {
  return fmaf((float)aten_word(seed, offset, S, g), 2.3283064e-10f, 2.3283064e-10f / 2.0f);
}

/* curand_normal4's lane: Box-Muller on (x0, x1) and (x2, x3), libm sinf / cosf */
float aten_normal01(uint64_t seed, uint64_t offset, uint32_t S, uint32_t g) {
  uint32_t x[4];
  const int j = aten_block(seed, offset, S, g, x);
  const int h = j / 2;
  const float u = fmaf((float)x[2 * h], 2.3283064e-10f, 2.3283064e-10f / 2.0f);
  const float w = fmaf((float)x[2 * h + 1], 2.3283064e-10f * 6.2831855f, (2.3283064e-10f * 6.2831855f) / 2.0f);
  const float s = sqrtf(-2.0f * logf(u));
  return (j % 2 ? cosf(w) : sinf(w)) * s;
}
