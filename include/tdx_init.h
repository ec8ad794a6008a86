/*
 * tdx_init.h -- C ABI of the H100 (sm_90a) fused-initialisation kernel library
 * (libtdx_init.so).
 *
 * This is the drop-in boundary BELOW the Python/pybind surface of
 * torchdistx.deferred_init.  The reference replays every recorded aten op
 * through the PyTorch dispatcher, one ATen kernel per op
 * (reference: src/cc/torchdistx/deferred_init.cc:218-220 `handle.callBoxed`,
 * :256-272 `Op::materialize`, :506-528 `OpNode::materialize`).  Here the whole
 * recorded expression of one tensor (empty -> uniform_/normal_/fill_/zero_ ->
 * mul/add/erfinv/clamp ...) is folded by the host-side planner into ONE
 * `TdxInitDesc`, and a table of descriptors is executed by one persistent
 * kernel launch per kernel family.
 *
 * Rules of the ABI: plain C, no torch types, no exceptions, no allocation.
 * Every buffer (destination tensors, device workspace) is owned by the caller.
 * All functions return 0 on success or a (positive) cudaError_t value /
 * negative TDX_E* code on failure; tdx_last_error() gives a message.
 *
 * Random stream specification (normative; restated on the CPU in
 * oracle/tdx_oracle.c and pinned by tests/golden):
 *
 *   Philox4x32-10, key = (seed_lo, seed_hi),
 *   counter = (off_lo, blk_hi, off_hi | 0x80000000, blk_lo)
 *   where off = TdxInitDesc.philox_offset (the torch generator offset at the
 *   time the op was issued == unique id of this RNG op under that seed) and
 *   blk = floor(g / EPB) for GLOBAL linear element index g of the unsharded
 *   tensor.  EPB = 8 for 16-bit outputs (16 random bits per element), 4 for
 *   32-bit outputs and for 16-bit outputs generated "wide" (TDX_ALGO_WIDE32).  Bit 31 of counter.z
 *   keeps the stream disjoint from ATen's own (offset, thread-id) use of the same generator
 *   (ATen/native/cuda/DistributionTemplates.h:72-88: ATen's third counter word is the high half of a
 *   thread index, far below 2^31); bits 30/29 of counter.z select the two tail-refinement blocks of
 *   the 16-bit normal.  The per-element word blk_lo is the LAST counter word: a Philox round only
 *   XORs and moves it, so the first multiplications of a block are per-tile constants (see
 *   tdx_device.cuh philox_block); every bit of it still passes nine multiplying rounds.
 *   Because the value of element g depends only on (seed, off, g), any
 *   partition of [0, numel) over ranks reproduces the unsharded tensor
 *   bit-for-bit.
 */
#ifndef TDX_INIT_H_
#define TDX_INIT_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define TDX_C_API __attribute__((visibility("default")))
#else
#define TDX_C_API
#endif

#define TDX_ABI_VERSION 2 /* 2: TdxPlan is 4 KiB; TDX_SRC_IOTA, TDX_I64, TDX_EPI_RPOW/RECIP; counter layout of the stream */

/* element type of the destination */
enum {
  TDX_F32 = 0,
  TDX_BF16 = 1,
  TDX_F16 = 2,
  TDX_I64 = 3, /* only valid with TDX_SRC_IOTA (arange buffers: position ids) */
  /* raw widths: only valid with TDX_SRC_CONST (bit-pattern fill) */
  TDX_RAW8 = 8,
  TDX_RAW16 = 9,
  TDX_RAW32 = 10,
  TDX_RAW64 = 11,
};

/* source of the expression (what the LAST full-tensor writer produces) */
enum {
  TDX_SRC_CONST = 0,   /* fill_/zero_/zeros/ones/full, constant-folded chains */
  TDX_SRC_UNIFORM = 1, /* uniform_(from,to), rand, kaiming_uniform_, xavier_uniform_ */
  TDX_SRC_NORMAL = 2,  /* normal_(mean,std), randn, kaiming_normal_, xavier_normal_ */
  /* element g = p0 + g * p1 (both integers, exactly representable in the destination), then the
   * epilogue: `arange` buffers and the index programs built on them -- rotary inv_freq is
   * arange -> float -> / dim -> base ** x -> reciprocal -> * scale.  dtype TDX_F32, or TDX_BF16 /
   * TDX_F16 (the fp32 value rounded once, to nearest even, at the store: `inv_freq.to(bf16)`)
   * -- epilogue allowed -- or TDX_I64 (none).  The reference replays these op by op through ATen
   * (deferred_init.cc:256-272); here they are one descriptor in the module's launch. */
  TDX_SRC_IOTA = 3,
  /* Sinusoidal position table [R, 2H] (Whisper, M2M100 / NLLB, GPT-J, CodeGen, MusicGen): the sin and
   * cos of an outer product of two index programs, P[r, k] = float(r) * f(k).  For GLOBAL element g:
   *   r = g / 2H, c = g % 2H, k = c mod H;
   *   f = the column program: float(p0 + k * p1) (integers, as TDX_SRC_IOTA) through the epilogue, in
   *       fp32 (an fp32 intermediate: TDX_EPI_NOROUND / TDX_FLAG_SRC_NOROUND change nothing);
   *   x = float(r) * f, one fp32 rounding (rows are arange(R) only, R < 2^24: float(r) is exact);
   *   v = sinf(x) for c < H and cosf(x) for c >= H, swapped by the order bit -- the accurate libdevice
   *       functions ATen's CUDA float kernels call;
   * and one rounding to the destination dtype at the store: TDX_F32, or TDX_BF16 / TDX_F16 (the table
   * cast at the end).  fill_bits = {H, flags}: H > 0; flags bit 0 = the order [cos | sin] (MusicGen).
   * Every other flag bit, and R >= 2^24, is rejected (TDX_E_BADARG). */
  TDX_SRC_SINCOS = 4,
  /* Copy of a host-built tensor (RWKV's time_* parameters, the numpy sinusoid tables of Pegasus and
   * Marian): the caller has staged the source on the device, already in the destination dtype.  For
   * GLOBAL element g:
   *   i = P ? (g / max(R, 1)) % P : g   (the broadcast geometry of TDX_SRC_IOTA; {0, 0}: a plain copy)
   *   v = src[i]
   * then the epilogue (TDX_F32 / TDX_BF16 / TDX_F16; every step rounds to the dtype, as for the RNG
   * sources); without one the element's bits are copied unchanged.  TDX_I64 copies, no epilogue.
   * fill_bits = {src, P | R << 32}: fill_bits[0] is the device address of the source array (element
   * aligned, at least P -- or, for P = 0, elem_begin + elem_count -- elements); P and R are below
   * 2^32, and R must be 0 when P is.  `algo` and `reserved` carry no flag for this source: a null
   * source, another dtype or any flag bit is rejected (TDX_E_BADARG). */
  TDX_SRC_GATHER = 5,
  /* Band mask of an [..., R, C] tensor (the causal-mask buffers of GPT-BigCode, GPT-Neo, ImageGPT,
   * OpenAI GPT, Bark and CLVP: `tril` / `triu` of a constant).  For GLOBAL element g:
   *   c = g % C;  r = (g / C) % R;  d = c - r   (signed)
   *   v = (lo <= d && d <= hi) ? IN : OUT
   * fill_bits = {C | R << 32, (uint32)lo | (uint64)(uint32)hi << 32}: 0 < C, R < 2^31; lo and hi are
   * int32 with lo <= hi (the planner clamps them to [-R, C]: an unbounded side needs no sentinel).
   * IN and OUT are element bit patterns, in the low itemsize bytes of philox_seed (IN) and
   * philox_offset (OUT): the source draws no random numbers.  dtype gives the width only: TDX_RAW8 ...
   * TDX_RAW64 or TDX_F32 / TDX_BF16 / TDX_F16 / TDX_I64 (bool is TDX_RAW8).  Nothing is read.
   * Rejected (TDX_E_BADARG): C or R equal to 0 or at least 2^31, lo > hi, any epilogue step, any
   * `algo` bit or `reserved` flag (TDX_FLAG_WINDOW included), an unknown dtype. */
  TDX_SRC_BAND = 6,
};
#define TDX_SINCOS_COS_FIRST 0x1u /* fill_bits[1] of TDX_SRC_SINCOS: the table is [cos | sin] */

/* sampling algorithm.  0 = the shipped default for (src, dtype). */
enum {
  TDX_ALGO_DEFAULT = 0,
  TDX_ALGO_ICDF16 = 1, /* 16-bit dtypes: inverse-CDF on 16 random bits/element + tail refinement */
  TDX_ALGO_BM32 = 2,   /* Box-Muller on 32 random bits/element (f32 default) */
  TDX_ALGO_WIDE32 = 2, /* same value: for 16-bit outputs of EITHER source, use the fp32 stream and
                        * arithmetic (EPB = 4) and round once at the store -- the meaning of
                        * `fp32_tensor.uniform_()/normal_()` followed by `.to(bf16/fp16)` */
  /* ATen's own CUDA stream: the bits torch's `normal_` / `uniform_` give the tensor the draw ran on (see
   * "ATen stream" below).  TDX_SRC_UNIFORM / TDX_SRC_NORMAL in TDX_F32 / TDX_BF16 / TDX_F16 only. */
  TDX_ALGO_ATEN = 3,      /* the draw ran on a tensor of the descriptor's dtype */
  TDX_ALGO_ATEN_WIDE = 4, /* the draw ran on an fp32 tensor; its value is rounded to the dtype at the store */
  TDX_ALGO_NOLUT = 0x20, /* OR-able flag: never use the shared-memory-table twin of ICDF16
                          * (same bits either way; for A/B measurements) */
};  /* any other bit of TdxInitDesc.algo is rejected (TDX_E_BADARG) */

/* epilogue steps, applied in order after the source transform; every step
 * rounds its result to the destination dtype, exactly like a chain of in-place
 * ATen ops on a tensor of that dtype does. */
enum {
  TDX_EPI_MUL = 1,    /* x = x * a            (mul_, mul.Tensor/Scalar)  */
  TDX_EPI_ADD = 2,    /* x = x + a            (add_, add.Tensor/Scalar with alpha folded) */
  TDX_EPI_ERFINV = 3, /* x = erfinv(x)        (trunc_normal_)            */
  TDX_EPI_CLAMP = 4,  /* x = min(max(x,a),b)  (clamp_; a NaN x stays NaN, as ATen's clamp keeps it) */
  TDX_EPI_RPOW = 5,   /* x = powf(a, x)       (pow.Scalar: scalar ** tensor) */
  TDX_EPI_RECIP = 6,  /* x = 1 / x            (reciprocal; `1.0 / t`)    */
  /* (`t / c` with a scalar c is TDX_EPI_MUL by float(1.0 / c), the reciprocal of the double c rounded
   * once to fp32: what ATen's CUDA kernel computes, $TORCH/.../cuda/BinaryDivTrueKernel.cu) */
  /* The state-space / linear-attention steps (Mamba A_log and dt bias).  expf / logf / expm1f are
   * the accurate libdevice functions ATen's CUDA float unary kernels call.  Like every step, each
   * rounds to the destination dtype after every ATen op it stands for. */
  TDX_EPI_EXP = 7,          /* x = expf(x)          (exp, exp_)                */
  TDX_EPI_LOG = 8,          /* x = logf(x)          (log, log_)                */
  TDX_EPI_EXPM1 = 9,        /* x = expm1f(x)        (expm1, expm1_)            */
  TDX_EPI_INV_SOFTPLUS = 10, /* x = x + log(-expm1(-x)): t = R(expm1f(-x)); t = R(logf(-t));
                              * x = R(x + t) (the inverse of softplus; negation is exact) */
  TDX_EPI_MULADD = 11,      /* x = R(R(x * a) + b)  (mul then add: two ATen ops in one step) */
};
/* OR-able into TdxEpiStep.op: do not round to the destination dtype after this step (the step
 * was recorded on an fp32 intermediate that is cast to the destination dtype later). */
#define TDX_EPI_NOROUND 0x100u
/* TdxInitDesc.reserved bit 0: the source op itself produced an fp32 intermediate (do not round
 * the generated value to the destination dtype before the first epilogue step). */
#define TDX_FLAG_SRC_NOROUND 0x1u
/* TdxInitDesc.reserved bit 1: a windowed descriptor -- one rank's Shard(d) block, d >= 1, of a
 * row-major parameter [s0 ... sn] (RowwiseParallel's Linear weight, ColwiseParallel's Embedding
 * weight).  Valid with TDX_SRC_UNIFORM and TDX_SRC_NORMAL only (any dtype, TDX_ALGO_WIDE32, any
 * epilogue step).  fill_bits = {W, P}: the block is runs of W consecutive global elements, P apart,
 * so LOCAL element l (0 <= l < elem_count, written at dst + l) is GLOBAL element
 *   g = elem_begin + (l / W) * P + l % W
 * and takes exactly the value element g of the unsharded tensor has.  For Shard(d) with torch.chunk
 * row counts, rank r's block is O = s0 * ... * s(d-1) runs, W = rows_r * inner, P = s_d * inner,
 * elem_begin = start_r * inner (inner = s(d+1) * ... * sn), elem_count = O * W.  Rejected
 * (TDX_E_BADARG): another source, W == 0, P < W, and a last element g beyond 2^64 - 1. */
#define TDX_FLAG_WINDOW 0x2u
/*
 * ATen stream (TDX_ALGO_ATEN, TDX_ALGO_ATEN_WIDE; normative).  One `normal_` / `uniform_` of ATen's CUDA
 * backend on a contiguous tensor of N < 2^31 elements (a 32-bit, trivially 1-D TensorIterator:
 * $TORCH/include/ATen/native/cuda/DistributionTemplates.h distribution_nullary_kernel) launches
 * grid = min(#SM * (max threads per SM / 256), ceil(N / 256)) blocks of 256 threads, grid stride
 * S = 256 * grid, and advances the generator's offset o by ((N - 1) / (4S) + 1) * 4.  Element g:
 *   t = g % S, q = g / S, k = q / 4, j = q % 4;
 *   x = curand Philox4x32-10, key = (seed_lo, seed_hi), counter = (o/4 + k) in words x, y and t in z, w
 *       (curand_init(seed, t, o), then k + 1 calls of curand4); element g takes lane j;
 *   uniform: r_j = x_j * 2^-32 + 2^-33 (one FMA); from, to cast to the dtype D; range = float(to - from)
 *       in D's arithmetic; v = D(fma(r, range, from)); v == to ? from : v;
 *   normal: Box-Muller on (x0, x1) and (x2, x3): u = x * 2^-32 + 2^-33, w = y * 2^-32 * 2pi + 2^-33 * 2pi
 *       (FMAs), s = sqrtf(-2 * logf(u)), __sincosf(w); lanes (s sin, s cos, s sin, s cos); v = fma(r, std, mean),
 *       rounded to D at the store;
 * then the epilogue (every step, as for the other algos).  TDX_ALGO_ATEN_WIDE: the same draw with D = fp32,
 * rounded to the dtype at the store (`fp32_tensor.uniform_().to(dtype)`).  philox_offset = o (a multiple of
 * 4), fill_bits[1] = S; with TDX_FLAG_WINDOW, fill_bits[0] = W | P << 32 (the window of TDX_FLAG_WINDOW).
 * Rejected (TDX_E_BADARG): S == 0 or not a multiple of 256, o % 4 != 0, a last global element >= 2^31,
 * TDX_ALGO_NOLUT, any other source or dtype.
 */
#define TDX_MAX_EPI 4

typedef struct TdxEpiStep {
  uint32_t op;
  float a;
  float b;
} TdxEpiStep;

/* One fused per-tensor (or per-shard) initialisation program.  128 bytes. */
typedef struct TdxInitDesc {
  void* dst;              /* device address where element `elem_begin` is written */
  uint64_t elem_begin;    /* global linear index (unsharded tensor) of the first element written */
  uint64_t elem_count;    /* number of consecutive elements written */
  uint64_t philox_seed;   /* generator seed           (RNG sources; BAND: the IN bits) */
  uint64_t philox_offset; /* generator offset at issue (RNG sources; BAND: the OUT bits) */
  double p0;              /* UNIFORM: from   NORMAL: mean */
  double p1;              /* UNIFORM: to     NORMAL: std  */
  uint64_t fill_bits[2];  /* CONST: 16-byte store pattern (element bits replicated)
                           * IOTA: broadcast geometry {P, R}: the index of GLOBAL element g is
                           * i = P ? (g / max(R, 1)) % P : g, and its value p0 + i * p1.
                           * `arange(n)[None, :].expand(D, -1)` is P = n; `arange(n)[:, None]
                           * .expand(-1, m)` is P = n, R = m; {0, 0} is the plain arange.
                           * SINCOS: {H, flags} (see TDX_SRC_SINCOS)
                           * GATHER: {source address, P | R << 32} (see TDX_SRC_GATHER)
                           * BAND: {C | R << 32, lo | hi << 32} (see TDX_SRC_BAND)
                           * UNIFORM / NORMAL with TDX_FLAG_WINDOW: {W, P} (see there)
                           * UNIFORM / NORMAL, TDX_ALGO_ATEN(_WIDE): {W | P << 32 (windows only), S} */
  uint8_t dtype;          /* TDX_F32 ... */
  uint8_t src;            /* TDX_SRC_* */
  uint8_t algo;           /* TDX_ALGO_* */
  uint8_t n_epi;          /* number of valid epilogue steps */
  uint32_t reserved;
  TdxEpiStep epi[TDX_MAX_EPI];
} TdxInitDesc;

/*
 * A table may mix any descriptors: the library routes each to a kernel family (80 of them: the
 * generators by dtype, algo, epilogue class, window and stream; the table kernels; the deterministic
 * sources) and issues one launch per family the table uses.  One plan header holds 47 families;
 * tdx_init_launch / tdx_init_prepare + tdx_init_submit lay a table that spans more out as consecutive
 * plans in one workspace (each with its own header and work counters) and launch them in order on the
 * stream, so any table is taken whole.  tdx_plan_upload keeps to one plan: a table of more than 47
 * families is refused there (TDX_E_BADARG).  Which kernel a descriptor runs in is decided over the whole
 * table, not per plan, so the split changes no bit.
 */

/* Bytes of device workspace tdx_init_launch() needs for `n` descriptors. */
TDX_C_API size_t tdx_init_workspace_bytes(int n);

/*
 * Validates and executes `n` descriptors on `stream` (a cudaStream_t passed as
 * void*; NULL = legacy default stream) of the CURRENT device.
 * `descs` is host memory; `workspace` is device memory of at least
 * tdx_init_workspace_bytes(n) bytes that must stay untouched until the
 * launches complete.  Asynchronous w.r.t. the host.
 * Replaces: the per-op replay loop of OpNode::materialize
 * (reference deferred_init.cc:506-528).
 */
TDX_C_API int tdx_init_launch(const TdxInitDesc* descs, int n, void* workspace,
                              size_t workspace_bytes, void* stream);

/*
 * The same in two steps, for callers that want to allocate exactly what a table
 * needs instead of the upper bound of tdx_init_workspace_bytes(n) (which has to
 * allow for the table kernels' work lists: ~1.6 MB): tdx_init_prepare validates
 * and lays the plan out on the host and returns its size (0: nothing to launch);
 * tdx_init_submit copies it into `workspace` and launches.  The prepared plan
 * belongs to the calling thread and is consumed by the next tdx_init_submit.
 */
TDX_C_API int tdx_init_prepare(const TdxInitDesc* descs, int n, size_t* workspace_bytes);
TDX_C_API int tdx_init_submit(void* workspace, size_t workspace_bytes, void* stream);

/*
 * Two-phase variant for callers that re-launch one plan (benchmarks, CUDA
 * graphs): upload once, launch many times.  `tdx_plan_upload` copies the
 * grouped descriptor table into `workspace`; `tdx_plan_launch` only issues the
 * kernels (the work counters in the workspace are uploaded as zero and every
 * kernel puts its own back to zero when its last CTA leaves, so there is no
 * memset between launches; one plan must not run on two streams at once).
 * One plan: at most 47 kernel families (see above), else TDX_E_BADARG.
 */
typedef struct TdxPlan {
  uint64_t opaque[512]; /* host-side copy of the plan header; owned by the caller */
} TdxPlan;
TDX_C_API int tdx_plan_upload(const TdxInitDesc* descs, int n, void* workspace,
                              size_t workspace_bytes, void* stream, TdxPlan* plan);
TDX_C_API int tdx_plan_launch(const TdxPlan* plan, void* workspace, void* stream);

/*
 * Host destinations (CPU-offloaded shards: FSDP2's CPUOffloadPolicy, FSDP1's offload_params).
 * tdx_init_submit_host runs a table whose `dst` addresses are all host memory, pinned or pageable, in
 * passes through a device staging buffer the caller owns (`staging`: device memory, 16-byte aligned,
 * untouched until the stream has run the call's work).  Each pass:
 *   1. places pieces of descriptors in the staging buffer -- a piece is the local elements [l0, l1) of
 *      one descriptor, kept at its destination's address mod 16, so the kernels take the vector/element
 *      split they take at the real address;
 *   2. lays the pass's table out as tdx_init_prepare would, carves its plan workspace from the head of
 *      `staging` and launches it on `stream`;
 *   3. enqueues one cudaMemcpyAsync device-to-host per piece on `stream` (local element l of a descriptor
 *      is at dst + l * itemsize: a piece is one contiguous copy).
 * Stream order is the only synchronisation: the next pass's launch runs after the previous pass's copies
 * have read the buffer.  The host does not block for pinned destinations; a pageable one makes its copy
 * synchronous (CUDA's rule for pageable memory).  The values depend only on (seed, offset, global index),
 * so the host gets the bits a device destination gets.
 * A piece of a plain descriptor is the descriptor with elem_begin += l0 and elem_count = l1 - l0.  A piece
 * of a windowed one (TDX_FLAG_WINDOW) keeps the window over its whole runs (elem_begin += (l0 / W) * P);
 * a partial first or last run is a plain descriptor of that run's elements.
 * Everything is validated before anything is enqueued: the descriptors as tdx_init_prepare checks them;
 * a `dst` that CUDA reports as device (or managed) memory, a null, unaligned or too small staging buffer
 * (smaller than one 16-byte vector plus the workspace of a one-descriptor pass) are TDX_E_BADARG.
 * tdx_last_launch_count() then counts every pass's launches, tdx_last_host_copies() the copies.
 */
TDX_C_API int tdx_init_submit_host(const TdxInitDesc* descs, int n, void* staging, size_t staging_bytes,
                                   void* stream);

/* One piece of the cut of tdx_init_submit_host. */
typedef struct TdxHostPiece {
  int32_t desc;         /* index of its descriptor in the table */
  int32_t pass;         /* the pass that writes it (0, 1, ...) */
  uint64_t elem_first;  /* first local element of the descriptor it holds */
  uint64_t elem_count;  /* its elements */
  uint64_t staging_off; /* byte offset in the staging buffer (== dst + elem_first * itemsize, mod 16) */
} TdxHostPiece;

/*
 * The cut tdx_init_submit_host makes of a table for a staging buffer of `staging_bytes`, without a device:
 * the pieces in submission order (pass by pass).  Writes at most `max_pieces` of them into `pieces` (may
 * be NULL) and the count and the number of passes into `*n_pieces` and `*n_passes`.  Validates the
 * table as tdx_init_submit_host does, but for the memory type of `dst`.
 */
TDX_C_API int tdx_init_host_cut(const TdxInitDesc* descs, int n, size_t staging_bytes, TdxHostPiece* pieces,
                                int max_pieces, int* n_pieces, int* n_passes);

/*
 * The descriptors (one to three) that write `piece` (of the descriptor `d`) into a staging buffer whose
 * first byte is at `staging`, in local order; returns their number (negative: an error code).
 */
TDX_C_API int tdx_init_host_piece_descs(const TdxInitDesc* d, const TdxHostPiece* piece, void* staging,
                                        TdxInitDesc out[3]);

/* Device-to-host copies the last tdx_init_submit_host on this thread enqueued (one per piece). */
TDX_C_API int tdx_last_host_copies(void);

/* Number of kernel launches the last tdx_plan_launch/tdx_init_launch on this
 * thread issued (one per non-empty kernel family). */
TDX_C_API int tdx_last_launch_count(void);

/* Bytes of the plan image (descriptor table, prefix sums, work lists) the last
 * tdx_plan_upload/tdx_init_launch on this thread copied host -> device. */
TDX_C_API size_t tdx_last_upload_bytes(void);

/* Elements of the global tensor covered by one Philox block for this dtype/algo
 * (the planner rounds RNG consumption with it). */
TDX_C_API int tdx_elems_per_block(int dtype, int src, int algo);

TDX_C_API int tdx_abi_version(void);
TDX_C_API const char* tdx_last_error(void);

#define TDX_E_BADARG (-1)
#define TDX_E_WORKSPACE (-2)
#define TDX_E_NODEVICE (-3)

#ifdef __cplusplus
}
#endif
#endif /* TDX_INIT_H_ */
