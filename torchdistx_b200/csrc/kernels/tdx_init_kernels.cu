// libtdx_init.so -- fused parameter-initialisation kernels for H100 (sm_90a).
//
// What this replaces: the reference materialises a deferred tensor by replaying
// every recorded aten op through the dispatcher, one stock ATen kernel per op,
// dead (overwritten) ops included
// (reference src/cc/torchdistx/deferred_init.cc:506-528 OpNode::materialize,
//  :256-272 Op::materialize, :218-220 handle.callBoxed).
// Here one TdxInitDesc carries the folded expression of a whole tensor and a
// persistent kernel streams it to HBM exactly once: Philox counter-based RNG in
// registers, 128-bit coalesced stores, zero reads, no intermediates.
//
// Roofline: pure HBM write.  Algorithmic bytes = elem_count * itemsize per descriptor.  Besides HBM,
// what bounds the RNG kernels is instruction issue (benchmarks/instr_rate.cu,
// benchmarks/philox_rate.cu measure it on the device at hand): Philox4x32-10 is 20 IMAD.WIDE + 20
// LOP3 per 128 random bits, against 16 bytes of output per block.  So 16-bit outputs draw 16 random bits
// per element (8 elements per Philox block), large 16-bit descriptors turn half-words into outputs
// through a shared-memory table (tdx_lut16_kernel), counter.y is hoisted per tile, and the fp32
// generators spend one I2FP per element.  See DESIGN.md section 4.
//
// Scheduling: one kernel launch per kernel family (<= a handful per module, not one per tensor).
// 256-thread kernels: grid = #SM x resident CTAs, CTAs grab runs of tiles of the family's global
// tile space from an atomic counter (grab size chosen per launch).  Table kernel: one 512-thread
// CTA per SM, grabs from a host-built, descriptor-pure work list.  Small and large tensors, shards
// and ragged tails balance across all SMs either way; every kernel zeroes its work counter
// when its last CTA leaves.
//
// The shared device code is tdx_device.cuh; the host side (validation, routing, plan, launch) is
// tdx_init_host.cu.
#define TDX_DEVICE_BASE_UNIT  // (tdx_device.cuh icdf16_tail)
#include "tdx_device.cuh"

namespace tdx {

// half-word `e` of a Philox block as the float k (one I2F.U16 with a half-word operand select: no
// byte-permute constant to keep in a register, which the table kernel re-materialised for every
// vector)
__device__ __forceinline__ float halfword_as_float(const uint4& w, int e) {
  const uint32_t word = (e >> 1) == 0 ? w.x : (e >> 1) == 1 ? w.y : (e >> 1) == 2 ? w.z : w.w;
  unsigned short lo, hi;
  asm("mov.b32 {%0, %1}, %2;" : "=h"(lo), "=h"(hi) : "r"(word));
  float f;
  asm("cvt.rn.f32.u16 %0, %1;" : "=f"(f) : "h"((e & 1) ? hi : lo));
  return f;
}

// Scheduler of the table kernel: a host-built work list instead of (chunk index -> binary search).
// Every grab costs microseconds -- the warps drain into the barrier, then three dependent trips
// through a memory system that is saturated with stores (work counter, list entry, descriptor) before
// the first new store; larger grabs cost fewer of them.  So
//  * the host cuts every descriptor into grabs of its own (guided sizes: up to 4 MiB while there is
//    plenty of work left, down to one tile at the end, for balance);
//  * all but the last four tiles per CTA of the work are PRE-ASSIGNED: the host cuts it into one
//    contiguous share per CTA and CTA b walks its own segment of the list -- no counter, and the
//    index of the next grab is known when the current one starts.  Only the tail is handed out
//    dynamically, which is what keeps the CTAs finishing together;
//  * the NEXT grab is brought into shared memory while the current one is being written: thread 0
//    starts an asynchronous copy (cp.async: no destination register, nothing to stall on) of the
//    16-byte list entry when a grab starts and, one tile later, prefetches the 128-byte descriptor
//    it names into the SM's L1.  After the barrier at the end of the grab everything the next one
//    needs is a shared-memory read or an L1 hit away.  All of thread 0's scheduling state lives in shared memory: the hot
//    loop has no register to spare.
struct LutSched {
  unsigned int next[2];  // list index of the grab in each slot (>= n_chunks: no more work)
  unsigned int pos, end; // CTA's segment of the pre-assigned part: next entry, one past the last
  volatile unsigned int stage;  // of the prefetch of the next grab: 2 = entry under way, 3 = descriptor under way / nothing to do
  unsigned int pad_[3];
  uint4 item[2];         // {descriptor, tiles, first tile in descriptor (lo, hi)}
  TdxInitDesc tab;       // the descriptor the table in shared memory was built for
};
static_assert(sizeof(TdxInitDesc) == 128, "a descriptor is one 128-byte line");
static_assert(sizeof(LutSched) % 16 == 0 && offsetof(LutSched, item) % 16 == 0, "LutSched follows the table in dynamic shared memory");

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// Thread 0's side job during a grab (every function is called by thread 0 only).
__device__ __forceinline__ void lut_prefetch_start(const GroupArgs& g, LutSched* s, unsigned int slot) {
  unsigned int c = s->pos;
  if (c < s->end) {
    s->pos = c + 1u;
  } else {
    // dynamic tail: this thread waits for the counter here (~1 us, once per tail grab)
    c = g.n_static + atomicAdd(g.counter, 1u);
  }
  s->next[slot] = c;
  if (c < g.n_chunks) {
    cp_async16(&s->item[slot], g.chunks + c);
    cp_async_commit();
    s->stage = 2u;
  } else {
    s->stage = 3u;
  }
}
__device__ __forceinline__ void lut_prefetch_desc(const GroupArgs& g, LutSched* s, unsigned int slot) {
  cp_async_wait_all();
  const uint32_t di = *reinterpret_cast<volatile uint32_t*>(&s->item[slot]);
  // (into this SM's L1, where the loads after the barrier find it; the descriptor table is 128-byte
  // aligned, so a descriptor is one line.  A copy into shared memory was tried: with the descriptor
  // behind a shared-memory reference ptxas no longer keeps the generator's constants in uniform
  // registers across the hot loop and reloads them from local memory for every group of vectors.)
  asm volatile("prefetch.global.L1 [%0];" ::"l"(g.descs + di));
  s->stage = 3u;
}
// hook of the tile loop (after the grab's first tile)
__device__ __forceinline__ void lut_prefetch_hook(const GroupArgs& g, LutSched* s, unsigned int slot) {
  if (s->stage == 2u) lut_prefetch_desc(g, s, slot);
}
__device__ __forceinline__ void lut_prefetch_finish(const GroupArgs& g, LutSched* s, unsigned int slot) {
  if (s->stage == 2u) lut_prefetch_desc(g, s, slot);  // (the grab was too short, or too odd, to overlap it)
  cp_async_wait_all();
}

// f(desc_index, descriptor, first tile, tiles, slot of the next grab)
//
// The SHAPE of this loop is load-bearing.  ptxas keeps the generator's constants (warp-reduction
// results) in registers across the hot loop inside f only if it can prove the warps converged
// there, and it proves that from control flow whose conditions are shared-memory loads at
// thread-independent addresses, kernel parameters and counters derived from them.  A barrier-free
// walk of the pre-assigned share (list entries read by every thread from global memory, or per-warp
// positions, or `continue` past the barrier -- all tried) made it guard every REDUX with BRA.DIV and
// keep the constants in local memory, reloaded for every group of vectors: a slower kernel, every
// test green.  A convergence-friendly barrier-free form (the share copied to a shared-memory window,
// inner counted loop) compiles well but was no faster than this one barrier per grab: with the next
// grab prefetched, the barrier costs less than warps that drift apart.  tests/test_lut_codegen.py guards the codegen.
template <class F>
__device__ __forceinline__ void for_each_listed_chunk(const GroupArgs& g, LutSched* s, F&& f) {
  if (threadIdx.x == 0) {
    unsigned int lo = 0u, hi = 0u;
    if (g.n_static) {
      lo = __ldg(g.seg_off + blockIdx.x);
      hi = __ldg(g.seg_off + blockIdx.x + 1u);
    }
    s->pos = lo;
    s->end = hi;
    unsigned int c;
    if (lo < hi) {
      c = lo;
      s->pos = lo + 1u;
    } else {
      c = g.n_static + atomicAdd(g.counter, 1u);
    }
    s->next[0] = c;
    if (c < g.n_chunks) s->item[0] = __ldg(g.chunks + c);
  }
  __syncthreads();
  for (unsigned int it = 0;; ++it) {
    const unsigned int slot = it & 1u;
    if (s->next[slot] >= g.n_chunks) {
      leave_grid(g);
      return;
    }
    const uint4 e = s->item[slot];
    if (threadIdx.x == 0) lut_prefetch_start(g, s, slot ^ 1u);
    f(e.x, g.descs[e.x], static_cast<unsigned long long>(e.z) | (static_cast<unsigned long long>(e.w) << 32),
      static_cast<unsigned long long>(e.y), slot ^ 1u);
    if (threadIdx.x == 0) lut_prefetch_finish(g, s, slot ^ 1u);
    __syncthreads();
  }
}

// constant fill: 16-byte pattern, frame = absolute 16-byte lines of the destination
template <int THREADS, int VECS>
__device__ __forceinline__ void fill_tiles(const TdxInitDesc& d, unsigned long long tile0, unsigned long long ntiles) {
  const uint4 pat = make_uint4(static_cast<uint32_t>(d.fill_bits[0]),
                               static_cast<uint32_t>(d.fill_bits[0] >> 32),
                               static_cast<uint32_t>(d.fill_bits[1]),
                               static_cast<uint32_t>(d.fill_bits[1] >> 32));
  const int isz = d.dtype == TDX_F32 || d.dtype == TDX_RAW32 ? 4 : d.dtype == TDX_RAW64 ? 8 : d.dtype == TDX_RAW8 ? 1 : 2;
  const uintptr_t a = reinterpret_cast<uintptr_t>(d.dst);
  const uintptr_t end = a + d.elem_count * isz;
  const uintptr_t a0 = a & ~static_cast<uintptr_t>(15);
  const uint64_t nvec = (end - a0 + 15) / 16;
  for (unsigned long long tile = tile0; tile < tile0 + ntiles; ++tile) {
    for (int i = 0; i < VECS; ++i) {
      const uint64_t j = tile * (THREADS * VECS) + static_cast<uint64_t>(i) * THREADS + threadIdx.x;
      if (j >= nvec) break;
      const uintptr_t p = a0 + j * 16;
      if (p >= a && p + 16 <= end) {
        store_vec(reinterpret_cast<void*>(p), pat);
      } else {  // head / tail line: byte-granular, the pattern phase follows the address
        const unsigned char* pb = reinterpret_cast<const unsigned char*>(&pat);
        for (int b = 0; b < 16; ++b) {
          const uintptr_t q = p + b;
          if (q >= a && q < end) *reinterpret_cast<unsigned char*>(q) = pb[(q - a) % isz];
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads) tdx_fill_kernel(const __grid_constant__ GroupArgs g) {
  for_each_tile_run(g, [&](uint32_t di, unsigned long long tile0, unsigned long long ntiles) {
    fill_tiles<kThreads, kVecsPerThread>(*desc_of(g, di), tile0, ntiles);
  });
}

// One element of an index program: the integer, then (floating outputs) the epilogue in fp32, then
// -- TDX_BF16 / TDX_F16: `inv_freq.to(torch.bfloat16)`, what Module.to(dtype) does to a rotary
// buffer -- one rounding to nearest even at the store.
__device__ __forceinline__ void iota_store(const TdxInitDesc& d, const EpiParams& epi, uint64_t j, long long val) {
  if (d.dtype == TDX_I64) {
    static_cast<long long*>(d.dst)[j] = val;
    return;
  }
  float v = static_cast<float>(val);
  if (epi.n) v = apply_epi<float>(epi, v);
  if (d.dtype == TDX_F32) static_cast<float*>(d.dst)[j] = v;
  else if (d.dtype == TDX_BF16) static_cast<__nv_bfloat16*>(d.dst)[j] = __float2bfloat16_rn(v);
  else static_cast<__half*>(d.dst)[j] = __float2half_rn(v);
}

// index programs: element g = start + g * step (integers), then the epilogue (in fp32).  Tiny
// buffers (rotary inv_freq: 64 elements, position ids: a few K): nothing to optimise but the launch
// they no longer need -- they ride in the module's plan like any other descriptor.
template <int THREADS, int VECS>
__device__ __forceinline__ void iota_tiles(const TdxInitDesc& d, unsigned long long tile0, unsigned long long ntiles) {
  const long long start = static_cast<long long>(d.p0), step = static_cast<long long>(d.p1);
  const EpiParams epi = load_epi(d);
  const uint64_t per_vec = 16 / iota_itemsize(d.dtype);
  // (frame: element i of the descriptor is global element elem_begin + i; one "vector" = 16 bytes)
  for (unsigned long long tile = tile0; tile < tile0 + ntiles; ++tile) {
    for (int i = 0; i < VECS; ++i) {
      const uint64_t vec = tile * (THREADS * VECS) + static_cast<uint64_t>(i) * THREADS + threadIdx.x;
      for (uint64_t e = 0; e < per_vec; ++e) {
        const uint64_t j = vec * per_vec + e;
        if (j >= d.elem_count) break;
        iota_store(d, epi, j, start + static_cast<long long>(d.elem_begin + j) * step);
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads) tdx_iota_kernel(const __grid_constant__ GroupArgs g) {
  for_each_tile_run(g, [&](uint32_t di, unsigned long long tile0, unsigned long long ntiles) {
    iota_tiles<kThreads, kVecsPerThread>(*desc_of(g, di), tile0, ntiles);
  });
}

// ---------------------------------------------------------------------------------------------
// 16-bit outputs through a shared-memory table
// ---------------------------------------------------------------------------------------------
// A 16-bit normal or uniform is a pure function of the Philox half-word k in [0, 65535] once the
// descriptor's parameters are fixed, so a CTA evaluates it once per k into a 128 KiB shared-memory
// table and then turns most half-words into outputs with one LDS.U16 each.  The table is built by
// the SAME device function as the direct kernel, so the two are bit-identical
// (tests/test_kernels_gpu.py checks it); the host picks this kernel for large descriptors only,
// because the table costs 65536 evaluations per CTA.
// 512 threads (one CTA per SM, 128 registers per thread): at 1024 threads and 64 registers ptxas
// for sm_90a keeps the generator's constants in local memory and reloads them inside the hot loop;
// on an H100 (80 GB HBM3, 700 W) the 512-thread kernel writes a 4 GiB bf16 normal in 1.37 ms instead
// of 1.70 ms, same bits (benchmarks/variant_bench.cu).
constexpr int kLutThreads = 512;
constexpr int kLutVecsPerThread = 16;
constexpr int kLutTileVecs = kLutThreads * kLutVecsPerThread;  // bytes per tile = 16 x this
constexpr int kLutTilesPerChunk = (1 << 20) / (kLutTileVecs * 16);                     // 1 MiB
constexpr uint32_t kLutBytes = 65536u * 2u;
constexpr unsigned short kLutSentinel = 0xffffu;  // a NaN pattern in bf16 and fp16: never a value

// cold path of the table kernel (a vector that contains k == 0): out of line, to keep the hot loop
// small enough for the instruction cache
template <class Gen>
__device__ __noinline__ uint4 lut_slow_vector(const TdxInitDesc* d, uint64_t gv) {
  using Out = typename Gen::OutT;
  const typename Gen::Params P = Gen::setup(*d);
  float v[8];
  Gen::gen(P, gv, v);
  return OutTraits<Out>::pack(v);
}

// ---------------------------------------------------------------------------------------------
// the table kernel
// ---------------------------------------------------------------------------------------------
// What shaped it (instruction counts of its first version and benchmarks/instr_rate.cu):
//  * byte address of a table entry = 2*k in ONE instruction: IDP.2A (dp2a.lo with the byte pair
//    (2,0) or (0,2) selects a half-word and doubles it) instead of PRMT + IADD3; the table's base
//    is the LDS immediate;
//  * counter.y (blk >> 32) is uniform inside a tile, so Philox round 1's second product and round
//    2's first product are loop-invariant: 18 IMAD.WIDE + 19 LOP3 per block instead of 20 + 20;
//    the round keys are kernel parameters (constant bank operands of the LOP3s);
//  * the normal's k == 0 sentinel (NaN) is accumulated with 2 HFMA2 per vector (NaN survives
//    a*b+c) and tested once per kLutGroup vectors; a hit re-derives the group's Philox blocks and
//    repairs only the vectors that really contain a zero half-word;
//  * LUT_ELEMS of the 8 elements of a vector go through the table, the others are computed (same
//    device function as the table builder => same bits): random indices cost 3.56 shared-memory
//    wavefronts per LDS and an SM delivers one wavefront per cycle, so a pure table kernel is
//    bound by the shared-memory pipe;
//  * work comes from a host-built list of descriptor-pure grabs (for_each_listed_chunk).
constexpr int kLutGroup = 4;

// byte offset 2*k of the table entry of the low / high half-word of a Philox word, in one IDP.2A
__device__ __forceinline__ uint32_t lut_off_lo(uint32_t w) {
  uint32_t a;
  asm("dp2a.lo.u32.u32 %0, %1, %2, %3;" : "=r"(a) : "r"(w), "r"(0x00000002u), "r"(0u));
  return a;
}
__device__ __forceinline__ uint32_t lut_off_hi(uint32_t w) {
  uint32_t a;
  asm("dp2a.lo.u32.u32 %0, %1, %2, %3;" : "=r"(a) : "r"(w), "r"(0x00000200u), "r"(0u));
  return a;
}
// Dynamic shared memory of a kernel without static shared memory starts at this offset of the
// shared window on sm_90 (the first KiB is reserved by the system).  The table kernel folds it
// into the immediate field of its LDS instructions; it checks the assumption at run time and
// takes the generic path if it ever does not hold.
constexpr uint32_t kDynSmemBase = 1024;
__device__ __forceinline__ uint32_t lds_u16_tab(uint32_t off) {
  unsigned short v;
  asm volatile("ld.shared.u16 %0, [%1+1024];" : "=h"(v) : "r"(off));
  return v;
}
__device__ __forceinline__ uint32_t pack_u16(uint32_t lo, uint32_t hi) {
  uint32_t r;
  asm("mad.lo.u32 %0, %1, 65536, %2;" : "=r"(r) : "r"(hi), "r"(lo));
  return r;
}
// exact test for "some 16-bit half of w is zero"
__device__ __forceinline__ bool has_zero_half(uint32_t w) {
  return ((w - 0x00010001u) & ~w & 0x80008000u) != 0u;
}

// Philox4x32-10 with precomputed round keys
__device__ __forceinline__ uint4 philox4x32_rk(uint4 c, const uint32_t (&rk)[20]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    unsigned long long p0, p1;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(p0) : "r"(c.x), "r"(kPhiloxM0));
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(p1) : "r"(c.z), "r"(kPhiloxM1));
    const uint32_t hi0 = static_cast<uint32_t>(p0 >> 32), lo0 = static_cast<uint32_t>(p0);
    const uint32_t hi1 = static_cast<uint32_t>(p1 >> 32), lo1 = static_cast<uint32_t>(p1);
    c = make_uint4(hi1 ^ c.y ^ rk[2 * r], lo1, hi0 ^ c.w ^ rk[2 * r + 1], lo0);
  }
  return c;
}

template <class Out>
struct NanAcc;
template <>
struct NanAcc<__nv_bfloat16> {
  uint32_t acc = 0;
  __device__ __forceinline__ void add(uint32_t a, uint32_t b) {
    asm("fma.rn.bf16x2 %0, %1, %2, %0;" : "+r"(acc) : "r"(a), "r"(b));
  }
};
template <>
struct NanAcc<__half> {
  uint32_t acc = 0;
  __device__ __forceinline__ void add(uint32_t a, uint32_t b) {
    asm("fma.rn.f16x2 %0, %1, %2, %0;" : "+r"(acc) : "r"(a), "r"(b));
  }
};

// What the table kernel needs to know about a 16-bit generator: the value of half-word k (the table
// entry and, for the elements that are not looked up, the directly computed value -- one device
// function, hence the same bits), the parameters that identify a table, and whether some k needs the
// exact out-of-line path (the normal's k == 0 tail).
// Two descriptors of one table-kernel family share a table iff their generator parameters and
// epilogues are equal (dtype, source and "has an epilogue" are the family's).  Equal as bit patterns:
// +0 and -0 compare equal as numbers but give tables of opposite signed zeros (normal_(+0, 0) against
// normal_(-0, 0), uniform_(-0, -0) against uniform_(-0, +0), mul_(0) against mul_(-0)).
__device__ __forceinline__ bool same_table(const TdxInitDesc& a, const TdxInitDesc& b) {
  bool same = __double_as_longlong(a.p0) == __double_as_longlong(b.p0) &&
              __double_as_longlong(a.p1) == __double_as_longlong(b.p1) && a.n_epi == b.n_epi && a.reserved == b.reserved;
  for (int i = 0; i < TDX_MAX_EPI; ++i)
    if (i < a.n_epi)
      same = same && a.epi[i].op == b.epi[i].op && __float_as_uint(a.epi[i].a) == __float_as_uint(b.epi[i].a) &&
             __float_as_uint(a.epi[i].b) == __float_as_uint(b.epi[i].b);
  return same;
}

// EPI: the descriptor carries epilogue steps (trunc_normal_, randn * s + m, ...).  The table then
// holds the FINAL value for every half-word -- the epilogue is as elementwise as the source
// transform -- so an erfinv costs the same as nothing once the table is built.
template <class Out, bool EPI = false>
struct TabNormal {
  using Gen = GenNormalICDF16<Out, EPI>;
  using Params = typename Gen::Params;
  static constexpr bool kHasTail = true;
  // The grid x = k/32768 - 1 is symmetric about k = 32768 and, with mean == +0, std != 0 and no
  // epilogue, so is the value (fma(q, -x, +0) == -fma(q, x, +0), rounding included): the upper half of
  // the table is the lower half with the sign bit flipped -- half the evaluations per table build.
  // With std == +-0 every q x is an exact zero and +-0 + +0 is +0 for both signs of x: no mirror.
  __device__ static __forceinline__ bool mirrored(const Params& p) {
    return !EPI && __float_as_uint(p.mean) == 0u && p.std != 0.f;
  }
  __device__ static __forceinline__ float value(const Params& p, float magic) {
    float t;
    const float v = Gen::element(p, magic, t);  // k == 0: +-inf or NaN (lg2(0) = -inf)
    return EPI ? apply_epi<Out>(p.epi, v) : v;
  }
  // the same value from k as a float (hot loop: halfword_as_float)
  __device__ static __forceinline__ float value_kf(const Params& p, float kf) {
    const float v = Gen::element_kf(p, kf);
    return EPI ? apply_epi<Out>(p.epi, v) : v;
  }
  __device__ static __forceinline__ void uniformize(Params& p) {
    p.mean = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.mean)));
    p.c0 = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.c0)));
    p.c1 = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.c1)));
    p.c2 = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.c2)));
    p.c3 = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.c3)));
    p.c4 = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.c4)));
    p.c5 = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.c5)));
  }
};
template <class Out, bool EPI = false>
struct TabUniform {
  using Gen = GenUniform16<Out, EPI>;
  using Params = typename Gen::Params;
  static constexpr bool kHasTail = false;
  __device__ static __forceinline__ bool mirrored(const Params&) { return false; }
  __device__ static __forceinline__ float value(const Params& p, float magic) {
    const float x = fminf(fmaf(magic - 8388608.0f, p.scale, p.from), p.to_prev);  // == Gen::gen, element by element
    return EPI ? apply_epi<Out>(p.epi, x) : x;
  }
  __device__ static __forceinline__ float value_kf(const Params& p, float kf) {
    const float x = fminf(fmaf(kf, p.scale, p.from), p.to_prev);  // magic - 2^23 == k exactly
    return EPI ? apply_epi<Out>(p.epi, x) : x;
  }
  __device__ static __forceinline__ void uniformize(Params& p) {
    p.from = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.from)));
    p.scale = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.scale)));
    p.to_prev = __uint_as_float(__reduce_or_sync(0xffffffffu, __float_as_uint(p.to_prev)));
  }
};

// Out-of-line work of the table kernel, each self-contained (everything is re-derived from the
// descriptor) so that none of its state is live across the hot loop:
//  * tiles that are not made of full, aligned vectors only (unaligned shards, ragged ends) or that
//    straddle a 2^32-block boundary;
template <class Gen>
__device__ __noinline__ void lut_ragged_tile(const TdxInitDesc* dp, unsigned long long tile) {
  const TdxInitDesc& d = *dp;
  const uint64_t begin = d.elem_begin, count = d.elem_count;
  const uint64_t gv0 = begin / 8;
  const uint64_t nvec = (begin + count - 1) / 8 - gv0 + 1;
  char* const dst = static_cast<char*>(d.dst);
  const bool aligned = (begin % 8 == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0);
  const uint64_t nfull = aligned ? count / 8 : 0;
  ragged_tile<Gen, kLutThreads, kLutVecsPerThread>(Gen::setup(d), dst, begin, count, gv0, nvec, nfull, tile);
}

//  * constant fills, which ride along in the table kernel's work list (the host folds a module's
//    few small fills -- norm weights, biases -- into it instead of paying a kernel launch for them);
__device__ __noinline__ void lut_fill_tiles(const TdxInitDesc* dp, unsigned long long tile0,
                                            unsigned long long ntiles) {
  fill_tiles<kLutThreads, kLutVecsPerThread>(*dp, tile0, ntiles);
}

//  * and index programs (rotary inv_freq, position ids: a few hundred bytes).
__device__ __noinline__ void lut_iota_tiles(const TdxInitDesc* dp, unsigned long long tile0, unsigned long long ntiles) {
  iota_tiles<kLutThreads, kLutVecsPerThread>(*dp, tile0, ntiles);
}

// Exponent-all-ones test of either half of a packed pair (inf or NaN).
template <class Out>
__device__ __forceinline__ bool any_nonfinite2(uint32_t v) {
  constexpr uint32_t m = sizeof(Out) == 2 && OutTraits<Out>::kDtype == TDX_BF16 ? 0x7f80u : 0x7c00u;
  return ((v & m) == m) || ((v & (m << 16)) == (m << 16));
}

// LUT_A / LUT_B: number of the 8 elements of an even / odd vector that go through the table (the
// others are computed).  PKEYS: Philox round keys are kernel parameters (the group's descriptors
// share one seed).  Per vector the cost is Philox (34 integer instructions after hoisting), a few
// instructions per looked-up element (IDP + LDS + half a pack) and several times that per computed
// normal -- against 3.56 shared-memory wavefronts per looked-up element, of which an SM delivers one
// per cycle (benchmarks/instr_rate.cu measures the issue costs on the device at hand).
template <class Tab, class Out, bool PKEYS, int LUT_A, int LUT_B>
__global__ void __launch_bounds__(kLutThreads, 1) tdx_lut16_kernel(const GroupArgs g) {
  using Gen = typename Tab::Gen;
  using T = OutTraits<Out>;
  static_assert(kLutVecsPerThread % kLutGroup == 0, "kLutGroup must divide the vectors per thread");
  // The table is the first thing in shared memory (this kernel has no static shared memory; the
  // scheduler's two slots follow the table), so the byte address of entry k is 2*k plus a constant
  // that fits the LDS immediate, and the IDP that forms 2*k reads one vector register.
  extern __shared__ __align__(16) unsigned short lut[];
  LutSched* const sched = reinterpret_cast<LutSched*>(lut + 65536);
  const bool base_ok = static_cast<uint32_t>(__cvta_generic_to_shared(lut)) == kDynSmemBase;
  uint32_t have_di = 0xffffffffu;  // descriptor the table in shared memory was built for (its copy: sched->tab)
  const bool t0 = threadIdx.x == 0;
  for_each_listed_chunk(g, sched, [&](uint32_t di, const TdxInitDesc& d, unsigned long long tile0,
                                      unsigned long long ntiles, unsigned int next_slot) {
    if (d.src == TDX_SRC_CONST) {  // a fill folded into this launch (build_plan): the table stays as it is
      lut_fill_tiles(&d, tile0, ntiles);
      return;
    }
    if (d.src == TDX_SRC_IOTA) {
      lut_iota_tiles(&d, tile0, ntiles);
      return;
    }
    typename Gen::Params P = Gen::setup(d);
    // Loop-invariant scalars that come out of a global load: a warp reduction's result lives in a
    // uniform register by construction, so the FFMAs / LOP3s that use them read two vector
    // registers instead of three.
    Tab::uniformize(P);
    P.ph.cz = __reduce_or_sync(0xffffffffu, P.ph.cz);
    P.ph.cw = __reduce_or_sync(0xffffffffu, P.ph.cw);
    if (have_di == 0xffffffffu || (di != have_di && !same_table(d, sched->tab))) {
      __syncthreads();  // everyone is done reading the old table (and comparing with its descriptor)
      if (threadIdx.x < 8)
        reinterpret_cast<uint4*>(&sched->tab)[threadIdx.x] = reinterpret_cast<const uint4*>(&d)[threadIdx.x];
      if (Tab::mirrored(P)) {
        for (uint32_t k = threadIdx.x; k <= 32768u; k += kLutThreads) {
          const Out o = static_cast<Out>(Tab::value(P, __uint_as_float(0x4b000000u | k)));
          const unsigned short bits = *reinterpret_cast<const unsigned short*>(&o);
          lut[k] = (Tab::kHasTail && k == 0) ? kLutSentinel : bits;
          if (k != 0u && k != 32768u) lut[65536u - k] = bits ^ 0x8000u;
        }
      } else {
        for (uint32_t k = threadIdx.x; k < 65536u; k += kLutThreads) {
          const Out o = static_cast<Out>(Tab::value(P, __uint_as_float(0x4b000000u | k)));
          lut[k] = (Tab::kHasTail && k == 0) ? kLutSentinel : *reinterpret_cast<const unsigned short*>(&o);
        }
      }
      __syncthreads();
    }
    have_di = di;
    const uint64_t begin = d.elem_begin;
    const uint64_t gv0 = begin / 8;
    char* const dst = static_cast<char*>(d.dst);
    const bool aligned = (begin % 8 == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0);
    const uint64_t nfull = aligned ? d.elem_count / 8 : 0;
    for (unsigned long long tile = tile0; tile < tile0 + ntiles; ++tile) {
      const uint64_t tbase = tile * kLutTileVecs;  // first vector of the tile (descriptor-relative)
      const uint64_t gfirst = gv0 + tbase;         // its global block index
      const uint32_t blk_hi = static_cast<uint32_t>(gfirst >> 32);
      const bool one_hi = static_cast<uint32_t>((gfirst + (kLutTileVecs - 1)) >> 32) == blk_hi;
      if (tbase + kLutTileVecs <= nfull && one_hi && base_ok) {
        const uint32_t lo0 = static_cast<uint32_t>(gfirst) + threadIdx.x;  // no carry: one_hi
        char* const p0 = dst + (tbase + threadIdx.x) * 16;
#pragma unroll
        for (int i0 = 0; i0 < kLutVecsPerThread; i0 += kLutGroup) {
          NanAcc<Out> nan;
#pragma unroll
          for (int i = i0; i < i0 + kLutGroup; ++i) {
            const int LUT_ELEMS = (i & 1) ? LUT_B : LUT_A;
            const uint4 c = make_uint4(P.ph.cz, blk_hi, P.ph.cw, lo0 + static_cast<uint32_t>(i) * kLutThreads);
            const uint4 w = PKEYS ? philox4x32_rk(c, g.rk) : philox4x32<10>(c, P.ph.k0, P.ph.k1);
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
            uint32_t r[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const bool lo_lut = 2 * q < LUT_ELEMS, hi_lut = 2 * q + 1 < LUT_ELEMS;
              if (lo_lut && hi_lut) {
                r[q] = pack_u16(lds_u16_tab(lut_off_lo(ws[q])), lds_u16_tab(lut_off_hi(ws[q])));
              } else if (!lo_lut && !hi_lut) {
                r[q] = T::pack2(Tab::value_kf(P, halfword_as_float(w, 2 * q)),
                                Tab::value_kf(P, halfword_as_float(w, 2 * q + 1)));
              } else {  // low half from the table, high half computed
                const uint32_t hi16 = T::pack2(0.0f, Tab::value_kf(P, halfword_as_float(w, 2 * q + 1)));
                r[q] = (hi16 & 0xffff0000u) | lds_u16_tab(lut_off_lo(ws[q]));
              }
            }
            if (Tab::kHasTail) {
              nan.add(r[0], r[1]);
              nan.add(r[2], r[3]);
            }
            store_vec(p0 + static_cast<size_t>(i) * (kLutThreads * 16), make_uint4(r[0], r[1], r[2], r[3]));
          }
          // k == 0 reads the NaN sentinel from the table and makes a computed element +-inf or NaN;
          // either survives the a*b+c accumulation.  Rare (2^-16 per element; also after an
          // overflow of the accumulator, which only costs time): find the vector(s) that contain
          // a zero half-word and redo them exactly.
          if (Tab::kHasTail && any_nonfinite2<Out>(nan.acc)) {
#pragma unroll 1
            for (int i = i0; i < i0 + kLutGroup; ++i) {
              const uint64_t gv = gfirst + threadIdx.x + static_cast<uint64_t>(i) * kLutThreads;
              const uint4 w = philox_block(P.ph, gv);
              if (has_zero_half(w.x) || has_zero_half(w.y) || has_zero_half(w.z) || has_zero_half(w.w))
                store_vec(p0 + static_cast<size_t>(i) * (kLutThreads * 16), lut_slow_vector<Gen>(&d, gv));
            }
          }
        }
      } else {
        lut_ragged_tile<Gen>(&d, tile);
      }
      // (thread 0, after the grab's first tile: the next list entry has arrived -- start on its descriptor)
      if (t0 && tile == tile0) lut_prefetch_hook(g, sched, next_slot);
    }
  });
}


// ---------------------------------------------------------------------------------------------
// the rows of this unit's kernels (tdx_device.cuh Family)
// ---------------------------------------------------------------------------------------------
using bf16 = __nv_bfloat16;
using f16 = __half;

#define TDX_FAM(src, dt, algo, epi, ...) \
  { src, dt, algo, epi, kPlain, false, static_cast<KernelFn>(tdx_rng_kernel<__VA_ARGS__>), #__VA_ARGS__ }
// fp32 generators: 16 vectors per thread (tile = 64 KiB, 4 tiles per 256 KiB grab)
#define TDX_FAM_V16(src, dt, algo, epi, ...)                                                               \
  { src, dt, algo, epi, kPlain, false, static_cast<KernelFn>(tdx_rng_kernel<__VA_ARGS__, 16>), #__VA_ARGS__, \
    kThreads, kThreads * 16, 0, (kVecsPerThread * kTilesPerChunk) / 16 }
// table-driven twins of the 16-bit generators: `fn` takes the Philox round keys from the kernel
// parameters (groups that share one seed: the normal case), `fn_any_seed` from each descriptor
#define TDX_FAM_LUT(src, dt, algo, epi, name, out, la, lb, ...)                                                  \
  { src, dt, algo, epi, kPlain, true, static_cast<KernelFn>(tdx_lut16_kernel<__VA_ARGS__, out, true, la, lb>), name, \
    kLutThreads, kLutTileVecs, static_cast<int>(kLutBytes + sizeof(LutSched)), kLutTilesPerChunk,                \
    static_cast<KernelFn>(tdx_lut16_kernel<__VA_ARGS__, out, false, la, lb>) }

static const Family kRows[] = {
    // (fills and index programs with a basic epilogue also ride in the table kernel's work list: build_plan)
    {TDX_SRC_CONST, kAnyDtype, 0, kEpiAny, kPlain, false, tdx_fill_kernel, "fill"},
    {TDX_SRC_IOTA, kAnyDtype, 0, kEpiNone | kEpiBasic, kPlain, false, tdx_iota_kernel, "iota"},
    TDX_FAM_V16(TDX_SRC_UNIFORM, TDX_F32, 0, kEpiNone, GenUniform32<float, false>),
    TDX_FAM(TDX_SRC_UNIFORM, TDX_F32, 0, kEpiBasic, GenUniform32<float, true>),
    TDX_FAM(TDX_SRC_UNIFORM, TDX_BF16, 0, kEpiNone, GenUniform16<bf16, false>),
    TDX_FAM(TDX_SRC_UNIFORM, TDX_BF16, 0, kEpiBasic, GenUniform16<bf16, true>),
    TDX_FAM(TDX_SRC_UNIFORM, TDX_F16, 0, kEpiNone, GenUniform16<f16, false>),
    TDX_FAM(TDX_SRC_UNIFORM, TDX_F16, 0, kEpiBasic, GenUniform16<f16, true>),
    TDX_FAM_V16(TDX_SRC_NORMAL, TDX_F32, TDX_ALGO_BM32, kEpiNone, GenNormalBM32<float, false>),
    TDX_FAM(TDX_SRC_NORMAL, TDX_F32, TDX_ALGO_BM32, kEpiBasic, GenNormalBM32<float, true>),
    TDX_FAM(TDX_SRC_NORMAL, TDX_BF16, TDX_ALGO_ICDF16, kEpiNone, GenNormalICDF16<bf16, false>),
    TDX_FAM(TDX_SRC_NORMAL, TDX_BF16, TDX_ALGO_ICDF16, kEpiBasic, GenNormalICDF16<bf16, true>),
    TDX_FAM(TDX_SRC_NORMAL, TDX_F16, TDX_ALGO_ICDF16, kEpiNone, GenNormalICDF16<f16, false>),
    TDX_FAM(TDX_SRC_NORMAL, TDX_F16, TDX_ALGO_ICDF16, kEpiBasic, GenNormalICDF16<f16, true>),
    // "wide" 16-bit outputs (TDX_ALGO_WIDE32): the fp32 stream and arithmetic, rounded once at the
    // store -- what `t_fp32.uniform_()/normal_()` followed by `.to(bf16/fp16)` means
    TDX_FAM(TDX_SRC_UNIFORM, TDX_BF16, TDX_ALGO_WIDE32, kEpiNone, GenUniform32<bf16, false>),
    TDX_FAM(TDX_SRC_UNIFORM, TDX_BF16, TDX_ALGO_WIDE32, kEpiBasic, GenUniform32<bf16, true>),
    TDX_FAM(TDX_SRC_UNIFORM, TDX_F16, TDX_ALGO_WIDE32, kEpiNone, GenUniform32<f16, false>),
    TDX_FAM(TDX_SRC_UNIFORM, TDX_F16, TDX_ALGO_WIDE32, kEpiBasic, GenUniform32<f16, true>),
    TDX_FAM(TDX_SRC_NORMAL, TDX_BF16, TDX_ALGO_BM32, kEpiNone, GenNormalBM32<bf16, false>),
    TDX_FAM(TDX_SRC_NORMAL, TDX_BF16, TDX_ALGO_BM32, kEpiBasic, GenNormalBM32<bf16, true>),
    TDX_FAM(TDX_SRC_NORMAL, TDX_F16, TDX_ALGO_BM32, kEpiNone, GenNormalBM32<f16, false>),
    TDX_FAM(TDX_SRC_NORMAL, TDX_F16, TDX_ALGO_BM32, kEpiBasic, GenNormalBM32<f16, true>),
    // table-driven twins of the 16-bit normal and uniform for large descriptors (bit-identical
    // output).  The normal looks up 7 of the 8 elements of a vector and computes one; a computed
    // uniform is cheap, so two of its eight elements relieve the shared-memory pipe.
    TDX_FAM_LUT(TDX_SRC_NORMAL, TDX_BF16, TDX_ALGO_ICDF16, kEpiNone, "lut<normal, bf16>", bf16, 7, 7, TabNormal<bf16>),
    TDX_FAM_LUT(TDX_SRC_NORMAL, TDX_F16, TDX_ALGO_ICDF16, kEpiNone, "lut<normal, f16>", f16, 7, 7, TabNormal<f16>),
    TDX_FAM_LUT(TDX_SRC_UNIFORM, TDX_BF16, 0, kEpiNone, "lut<uniform, bf16>", bf16, 6, 6, TabUniform<bf16>),
    TDX_FAM_LUT(TDX_SRC_UNIFORM, TDX_F16, 0, kEpiNone, "lut<uniform, f16>", f16, 6, 6, TabUniform<f16>),
    // with an epilogue every element is looked up: the computed alternative may contain an erfinv
    TDX_FAM_LUT(TDX_SRC_NORMAL, TDX_BF16, TDX_ALGO_ICDF16, kEpiBasic, "lut<normal+epilogue, bf16>", bf16, 8, 8, TabNormal<bf16, true>),
    TDX_FAM_LUT(TDX_SRC_NORMAL, TDX_F16, TDX_ALGO_ICDF16, kEpiBasic, "lut<normal+epilogue, f16>", f16, 8, 8, TabNormal<f16, true>),
    TDX_FAM_LUT(TDX_SRC_UNIFORM, TDX_BF16, 0, kEpiBasic, "lut<uniform+epilogue, bf16>", bf16, 8, 8, TabUniform<bf16, true>),
    TDX_FAM_LUT(TDX_SRC_UNIFORM, TDX_F16, 0, kEpiBasic, "lut<uniform+epilogue, f16>", f16, 8, 8, TabUniform<f16, true>),
};
const FamilyRows kBaseFamilies{kRows, sizeof(kRows) / sizeof(kRows[0])};

}  // namespace tdx
