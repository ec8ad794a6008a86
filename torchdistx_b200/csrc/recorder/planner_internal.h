// What the planner's three units share.  planner_eval.cc evaluates a storage's recorded program
// symbolically (a State) and lowers it to descriptors (a StorageTemplate); it needs no GPU.
// planner_engine.cc emits those descriptors and replays what does not lower (Engine,
// MaterializeSession); planner_pipeline.cc runs a session on a helper thread.
#pragma once

#include <ATen/Tensor.h>
#include <c10/core/Scalar.h>
#include <c10/core/impl/LocalDispatchKeySet.h>
#include <c10/util/SmallVector.h>

#include <cstdint>
#include <string>
#include <vector>

#include "planner.h"
#include "tape.h"
#include "tdx_init.h"

namespace tdx {

// Never record / fake anything we do while materialising.
struct NoInterception {
  c10::impl::ExcludeDispatchKeyGuard a{c10::DispatchKey::DeferredInit};
  c10::impl::ExcludeDispatchKeyGuard b{c10::DispatchKey::Fake};
};

// Where constant chains are folded.  ATen's CPU and CUDA kernels differ in the last bit for 16-bit
// dtypes (the CPU kernels round a Python scalar to the tensor dtype first, the CUDA kernels keep it
// in fp32), and a tensor recorded for CUDA must hold what the program computes on CUDA: so while
// materialising onto a CUDA device the 1-element stand-in lives there.  (plan_info, which may run
// on a machine without a GPU, folds on the CPU.)  Folds constants on `d` for the guard's lifetime.
struct FoldOn {
  c10::Device prev;
  explicit FoldOn(c10::Device d);
  ~FoldOn();
};

// ---------------------------------------------------------------------------------------------
// symbolic state of a storage: what its elements are, as a function of the element index
// ---------------------------------------------------------------------------------------------
// A storage is a list of disjoint SEGMENTS [begin, end) (element indices of the storage, in the
// dtype it currently holds), each with one simple content description.  A tensor initialised as a
// whole is one segment; `weight.normal_(); weight[padding_idx].zero_()` (nn.Embedding, BERT, Gemma,
// OPT, Phi-3) is three; an in-place op through a contiguous view splits the segments it crosses.
struct Sym {
  // Iota: element i = p0 + (i - origin) * p1 (integers): `arange`, and -- with epilogue steps -- the
  // index programs built on it (rotary inv_freq: arange -> float -> / dim -> base ** x -> 1/x -> * s)
  // Outer: the outer product of a sinusoidal position table, element i = float(r) * f(k) with
  // r = (i - origin) / half, k = (i - origin) % half and f the column index program (p0, p1, epi);
  // `trig` 1 / 2: its sin / cos.  An intermediate only: never emitted, and every op but sin / cos of
  // the product and the cat of the two leaves it opaque.
  // Sincos: the table cat([sin(P), cos(P)], -1) (or [cos | sin]: cos_first) of such a product:
  // TDX_SRC_SINCOS over [R, 2 * half], indexed like an arange.
  // Gather: a copy of a host-built (real) tensor: element i = gsrc[((i - origin) / max(repeat, 1)) %
  // period] (period 0: gsrc[i - origin]), then the epilogue -- TDX_SRC_GATHER.
  // Band: a band mask of an [..., R, C] storage (`tril` / `triu` of a constant, the bitwise_xor of two
  // nested bands): with g = i - origin, c = g % C and r = (g / C) % R, element i holds band_in when
  // band_lo <= c - r <= band_hi and band_out otherwise -- TDX_SRC_BAND.
  enum Src { Uninit, Const, Uniform, Normal, Iota, Outer, Sincos, Gather, Band } src = Uninit;
  at::Tensor cval;                           // Const: a 1-element tensor of the state's dtype (built lazily)
  // Gather: the source, read when the storage is evaluated for materialisation (never when the
  // recording is analysed): 1-D, contiguous, on the CPU, in the state's dtype
  at::Tensor gsrc;
  c10::Scalar cscalar;                       // Const: the value, while no folding has needed a tensor
  bool has_scalar = false;
  double p0 = 0, p1 = 1;                     // Uniform: from,to   Normal: mean,std   Iota: start,step
  uint32_t rng_op = kNoValue;                // the live RNG op
  // Iota broadcast (`arange(n)[None, :].expand(D, -1).contiguous()`, `arange(n).repeat(D, 1)`):
  // element i takes index ((i - origin) / max(repeat, 1)) % period; period 0 = the plain arange
  int64_t period = 0, repeat = 0;  // (Gather: the same broadcast geometry)
  int64_t half = 0;                      // Outer, Sincos: H, the column count of the product
  uint8_t trig = 0;                      // Outer: 0 the product, 1 its sin, 2 its cos
  bool cos_first = false;                // Sincos: the table is [cos | sin]
  uint32_t outer_storage = kNoValue;     // Outer: the storage the product was written to
  int64_t band_rows = 0, band_cols = 0;  // Band: R, C
  int64_t band_lo = 0, band_hi = 0;      // Band: the diagonals c - r it covers, within [-R, C]
  c10::Scalar band_in, band_out;         // Band: the values, as stored in the state's dtype
  // Up to TDX_MAX_EPI steps, or kMaxPlanEpi for programs with a state-space step (their
  // intermediates, e.g. `-expm1(-dt)`, are longer than any descriptor: emit_epi compacts them)
  c10::SmallVector<TdxEpiStep, TDX_MAX_EPI> epi;
  // The RNG source ran on an fp32 tensor that was later cast to a 16-bit dtype: keep the fp32
  // stream and arithmetic (TDX_ALGO_WIDE32) so that the result IS `fp32_tensor.to(dtype)`.
  bool wide = false;
  bool src_noround = false;  // the generated value feeds fp32 epilogue steps before the cast
  // `wide` exists to keep the 16-bit tensor equal to `fp32_source.to(dtype)` when BOTH get
  // materialised.  If nothing can ever ask for the fp32 source (`module.to(torch.bfloat16)` rebinds
  // every parameter to its cast and drops the fp32 tensor), the equality is unobservable and the
  // tensor takes the native 16-bit stream -- same distribution, the fast kernel (wide_observable()).
  uint32_t wide_src_storage = kNoValue;  // the storage the RNG op wrote (and the cast read), if that simple
  uint32_t wide_cast_op = kNoValue;
  bool rng() const { return src == Uniform || src == Normal; }
};

struct Seg {
  int64_t begin = 0, end = 0;
  // Storage index of element 0 of the tensor the segment's source op ran on: an RNG op on a view
  // numbers its elements from the view's first element (global Philox index = index - origin).
  int64_t origin = 0;
  Sym st;
};

struct RngPass {
  uint32_t op;     // tape op
  int64_t numel;   // of the tensor it ran on: what it consumes of the generator's offset
  uint32_t slot;   // Tape::rng entry of the op
};

// (inline storage: a recording holds one State per storage, and every heap block of a recording is
// one somebody has to free when it dies)
using SegList = c10::SmallVector<Seg, 1>;
using RngChain = c10::SmallVector<RngPass, 2>;

struct State {
  bool opaque = true;
  c10::ScalarType dtype = c10::ScalarType::Undefined;  // dtype of the tensor currently holding the state
  SegList segs;        // sorted, disjoint, covering [0, numel)
  RngChain rng_chain;  // every RNG pass met, live or dead, chronological
};

// What analyze_tape leaves on a storage: the symbolic state, and -- for the states the kernels can
// run -- the same thing laid out for the materialise call, which then touches this block, the
// value's geometry and two RNG slots per tensor and nothing else of the recording (the recording is
// cold in the caches by the time a model is materialised: every line touched is ~100 ns).
struct FastSeg {
  int64_t begin = 0, end = 0, origin = 0;
  uint32_t rng_slot = kNoValue;  // kNoValue: no RNG pass (a constant or an index program)
  bool indexed = false;          // the descriptor's elem_begin matters (RNG and iota sources)
  bool wide = false;
  const Sym* sym = nullptr;      // (into StorageTemplate::st) for the rare questions: wide_observable
  at::Tensor gather;             // TDX_SRC_GATHER: the host source, staged by the submission (Batch::flush)
  TdxInitDesc proto;             // everything but dst / elem_begin / elem_count / seed / offset
};
struct StorageTemplate {
  State st;
  bool fast = false;
  uint8_t isz = 0;
  int64_t numel = 0;
  c10::SmallVector<FastSeg, 1> segs;  // Uninit segments are left out
};

// State of storage S after every recorded op with index < upto.
State eval_storage(Tape& tape, uint32_t S, uint32_t upto);
// Lays a state out for emission (StorageTemplate's fast form).  false: some segment is not
// expressible as a descriptor.  `may_sync`: a constant that only exists as a (device) tensor may be
// read back (the materialise path; never the analysis at the end of the recording).
bool build_fast(const StorageInfo& si, StorageTemplate& t, bool may_sync);
// Can anything still observe the fp32 tensor a `wide` segment was cast from?  Not if no fake tensor
// names its storage any more, nothing of it has been materialised, and the only ops that ever
// touched it are its own writers and the cast.
bool wide_observable(const Tape& tape, const Sym& sy);
// RngStream::Aten's rule (planner_engine.cc aten_fusible).  Why ATen does not launch every draw of
// `chain`, live or dead, as one 32-bit, trivially 1-D iterator ("": it does), and whether the kernels
// compute epilogue step `op` on a draw bit for bit as ATen's CUDA op does.
std::string aten_draw_refusal(const Tape& tape, const RngChain& chain);
bool aten_exact_step(uint32_t op);
// The position of argument `name` in the op's schema (size_t(-1): none).
size_t find_arg(const TapeOp& op, const char* name);

// The TDX_RAW* dtype of a constant fill of `isz`-byte elements (1, 2, 4 or 8).
inline uint8_t raw_dtype(size_t isz) {
  return isz == 1 ? TDX_RAW8 : isz == 2 ? TDX_RAW16 : isz == 4 ? TDX_RAW32 : TDX_RAW64;
}

// The materialise call's counters and descriptor table on this thread (planner_engine.cc), which the
// pipelined session hands from its helper thread to the caller.
extern thread_local MaterializeStats g_stats;
extern thread_local std::vector<TdxInitDesc> g_last_descs;
extern thread_local double g_pending_traverse_us;  // see add_traverse_time
double now_us();
at::Tensor finish_tensor(const at::Tensor& fake, at::Tensor out);
bool prebuild_output(const at::Tensor& fake, const MaterializeOptions& opts, bool apply_shard, Prebuilt& pre);

}  // namespace tdx
