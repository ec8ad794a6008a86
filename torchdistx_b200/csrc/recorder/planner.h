// Materialisation: turning recorded tapes into real tensors.
//
// Replaces the reference's materialise path
//   materializeTensor / detail::materialize      reference deferred_init.cc:1163-1173, :713-729
//   OpNode::materialize / buildCallStack / ...   reference deferred_init.cc:506-667
//   Op::materialize -> handle.callBoxed          reference deferred_init.cc:256-272, :218-220
// with a two-tier executor:
//   1. FUSED (CUDA tensors): the ops that determine a storage are evaluated symbolically
//      (last-writer analysis; overwritten RNG passes only advance the Philox offset) into ONE
//      TdxInitDesc; all descriptors of a materialize call are executed by O(#kernel families)
//      launches of libtdx_init (include/tdx_init.h).  Under sharding each rank's descriptor covers
//      only its slice [elem_begin, elem_begin+elem_count) and writes into a shard-sized buffer:
//      the unsharded tensor never exists.
//   2. GENERIC replay through the dispatcher, in recorded order, for CPU-device tensors (bit-exact
//      with eager initialisation, same mt19937 stream) and for programs the planner does not
//      understand (executed by ATen on the recorded device).  Same semantics as the reference.
#pragma once

#include <ATen/Tensor.h>
#include <c10/core/StorageImpl.h>

#include <cstdint>
#include <functional>
#include <memory>
#include <optional>
#include <string>
#include <tuple>
#include <vector>

namespace tdx {

struct ShardSpec {
  int64_t rank = 0;
  int64_t world = 1;
  // dim-0 chunking as torch.chunk / FSDP2 Shard(0): rank r owns rows [r*ceil(d0/W), ...)
  // (reference callers: $TORCH/distributed/fsdp/_fully_shard/_fsdp_param.py:381-402)
  // dim > 0: the same rows of dimension `dim` (DTensor's Shard(dim): RowwiseParallel's Linear weight,
  // ColwiseParallel's Embedding weight), written by windowed descriptors (TDX_FLAG_WINDOW)
  int64_t dim = 0;
};

// Which Philox stream random tensors on CUDA are drawn from.  Fused: the engine's own layout (include/
// tdx_init.h; the reference's distribution, other bits).  Aten: ATen's own CUDA stream (TDX_ALGO_ATEN) --
// the bits eager `normal_` / `uniform_` and the reference's replay give, same generator offsets; draws
// the kernels cannot reproduce bit for bit are replayed through ATen at their place in the RNG order.
enum class RngStream { Fused, Aten };

struct MaterializeOptions {
  std::optional<c10::Device> device;  // override of the recorded device (e.g. record on cpu, build on cuda)
  std::optional<ShardSpec> shard;     // materialise only this rank's dim-0 chunk
  bool fused = true;                  // false: force generic replay (tests: elision must not change results)
  RngStream rng = RngStream::Fused;
};

struct MaterializeStats {
  int64_t tensors = 0;          // tensors requested
  int64_t fused_tensors = 0;    // served by the fused CUDA path
  int64_t generic_ops = 0;      // ops replayed through the dispatcher
  int64_t elided_rng_ops = 0;   // dead RNG passes that only advanced the Philox offset
  int64_t kernel_launches = 0;  // libtdx_init launches
  int64_t bytes_written = 0;    // algorithmic bytes of the fused descriptors
  int64_t descriptors = 0;
  double plan_us = 0;    // host time: slicing, symbolic evaluation, allocation, descriptor build
  double launch_us = 0;  // host time inside tdx_init_launch (plan image + H2D copy + launches)
  double wrap_us = 0;    // host time giving results their Python class / identity
  double traverse_us = 0;  // host time walking the module tree and unpacking its tensors (before planning)
  double assign_us = 0;    // host time putting the results back into the modules' dicts
  double eval_us = 0;            // part of plan_us: symbolic evaluation of the recorded programs
  double alloc_us = 0;           // part of plan_us: output allocations (caching allocator)
  int64_t upload_bytes = 0;      // plan images copied host -> device
  int64_t submissions = 0;       // tdx_init_launch calls (early submissions + the final one)
  double first_submit_us = 0;    // host time from the start of the call to the first submission
  double last_submit_us = 0;     // ... and to the last one
  int64_t template_hits = 0;     // storages whose analysis was done when the recording ended
  double helper_start_us = 0, helper_done_us = 0;  // when the planner thread started / finished, since the call began
  double deferred_us = 0;        // host time replaying the RNG-free unfusable programs after the last submission
  int64_t prebuilt_outputs = 0;  // outputs the calling thread had built before the helper planned them
  int64_t narrowed_tensors = 0;  // Shard(d >= 1) tensors built whole and narrowed (index, table, copy programs)
  int64_t aten_stream_tensors = 0;  // fused tensors with a draw in ATen's stream (RngStream::Aten)
  int64_t host_bytes = 0;   // bytes built into host memory (a CPU `out`: tdx_init_submit_host)
  int64_t host_copies = 0;  // ... and the device-to-host copies that moved them
};

// Materialises `fake` (a no-op returning `fake` itself for real tensors).
at::Tensor materialize_one(const at::Tensor& fake, const MaterializeOptions& opts);

// Materialises many tensors with one batched kernel submission; order defines RNG consumption.
// `shard_mask` (optional, one flag per tensor): apply opts.shard only where the flag is set
// (parameters are chunked, buffers replicated -- one ordered batch either way); a flag k > 0 cuts
// the tensor along dimension k - 1.
std::vector<at::Tensor> materialize_many(const std::vector<at::Tensor>& fakes,
                                         const MaterializeOptions& opts,
                                         const std::vector<uint8_t>* shard_mask = nullptr);

// FSDP1's layout (SURVEY 8e): this rank's chunk of the FlatParameter the given parameters form --
// flattened, concatenated in order (each start aligned to `align_numel` elements if > 1), chunked
// `world` ways like torch.chunk, right-padded with zeros ($TORCH/distributed/fsdp/_flat_param.py
// `_get_shard`) -- written directly into one 1-D tensor (`out`, if given: e.g. the handle's
// `_local_shard`).  Nothing unsharded is ever allocated.  `offsets` (optional) receives every
// parameter's start in the flat parameter, then the total.  opts.shard is ignored.
at::Tensor materialize_flat_shard(const std::vector<at::Tensor>& fakes, const MaterializeOptions& opts, int64_t rank,
                                  int64_t world, int64_t align_numel, const std::optional<at::Tensor>& out,
                                  std::vector<int64_t>* offsets = nullptr);

// The same, one tensor at a time: `materialize_module` walks the module tree and feeds tensors as it
// finds them, so the first kernels are on the GPU while the walk is still going on (the walk of a
// Llama-3-8B costs as much host time as planning a third of it).  add() order defines RNG
// consumption; finish() submits what is left and writes the generators back (the destructor does
// the latter on error paths too).
// An output tensor built ahead of its planning (PipelinedMaterialize::add): no memory yet -- the
// submission that carries its descriptors assigns it.
struct Prebuilt {
  at::Tensor out;
  c10::intrusive_ptr<c10::StorageImpl> storage;
  size_t nbytes = 0;
};

class MaterializeSession {
 public:
  explicit MaterializeSession(const MaterializeOptions& opts);
  ~MaterializeSession();
  MaterializeSession(const MaterializeSession&) = delete;
  MaterializeSession& operator=(const MaterializeSession&) = delete;
  // Returns the tensor -- or an undefined tensor if its program was deferred (see below); the
  // result then arrives through the sink, tagged with `ticket`, during finish().
  // `shard_dim`: the dimension opts.shard cuts this tensor along (ShardSpec::dim).
  at::Tensor add(const at::Tensor& fake, bool apply_shard = true, size_t ticket = 0, Prebuilt* pre = nullptr,
                 int64_t shard_dim = 0);
  // Programs the kernels cannot express and that draw no random numbers (rotary inv_freq, position
  // ids, masks) are replayed through ATen after the call's last fused submission instead of where the
  // walk meets them: their dispatches then overlap the GPU's work on the whole model.
  void defer_generic_programs(std::function<void(size_t ticket, at::Tensor result)> sink);
  void finish();

 private:
  struct Impl;
  std::unique_ptr<Impl> impl_;
};

// The session, run on a helper thread: the calling thread keeps walking its modules (and, once it
// has handed everything over, starts giving finished tensors their Python identity) while the
// helper plans, allocates and submits.  Host time of a 300-tensor module drops from walk + plan +
// wrap to roughly max(walk + wrap, plan) -- what a sharded materialise is bound by from 4 GPUs on.
// add() returns a ticket; result(ticket) blocks until that tensor has been planned (and rethrows
// the helper's exception, if any); join() waits for the final submission and moves the call's
// statistics to the calling thread.  The helper runs under the caller's ThreadLocalState (grad
// mode, dispatch keys, ...) and on the caller's current CUDA streams.
class PipelinedMaterialize {
 public:
  explicit PipelinedMaterialize(const MaterializeOptions& opts);
  ~PipelinedMaterialize();
  PipelinedMaterialize(const PipelinedMaterialize&) = delete;
  PipelinedMaterialize& operator=(const PipelinedMaterialize&) = delete;
  // `speculative` (optional): receives, if the recording's analysis says the tensor takes the fused
  // path, the very tensor object result(ticket) is going to return -- built on the calling thread,
  // before the helper has planned it.  The caller may wrap it at once but must compare with
  // result(ticket) in the end (the helper falls back to a tensor of its own when anything differs).
  size_t add(const at::Tensor& fake, bool apply_shard = true, at::Tensor* speculative = nullptr);
  void finish();
  at::Tensor result(size_t ticket);
  bool ready(size_t ticket);  // result(ticket) would not block
  // After result()/join() threw: the ticket of the tensor whose materialisation failed (or -1 if the
  // failure was not a tensor's: session set-up, the final submission).
  size_t failed_ticket();
  void join();

 private:
  struct State;
  std::shared_ptr<State> st_;
};

// A recording dies with the last fake tensor that names it -- typically at the end of the
// materialize_module call that replaces the module's fake tensors: ~3000 recorded call frames for
// Llama-3-8B, half a millisecond of destructors.  The caller hands its references to the helper
// thread, which lets go of them after the call has returned.
struct Tape;
void release_in_background(std::vector<std::shared_ptr<Tape>> tapes);
// Returns once the helper thread has finished everything queued so far (recordings handed to
// release_in_background included).  Call without the GIL.
void drain_background();

// The sizes (bytes) a materialize_module call cuts its submissions at, for a call that will write
// `total_bytes` in `tensors` tensors of `tensor_bytes` each (the rule of Batch::note; for tests and
// documentation -- nothing is allocated or launched).
std::vector<int64_t> submission_sizes(int64_t total_bytes, int64_t tensors, bool with_estimate);

// ATen's launch of one CUDA normal_ / uniform_ of `numel` elements on a device with `sm` SMs and `tps`
// threads per SM ($TORCH/include/ATen/native/cuda/DistributionTemplates.h calc_execution_policy):
// the grid stride S = 256 * min(sm * (tps / 256), ceil(numel / 256)) and the generator offset increment
// ((numel - 1) / (4 S) + 1) * 4 (0 for an empty tensor, which draws nothing).
std::pair<uint32_t, uint64_t> aten_stream_policy(int64_t numel, int sm, int tps);
inline uint64_t aten_offset_increment(int64_t numel, uint64_t S) {
  return ((static_cast<uint64_t>(numel) - 1) / (4 * S) + 1) * 4;
}

MaterializeStats last_stats();
void add_wrap_time(double us);
void add_traverse_time(double us);
// The TdxInitDesc table (raw bytes) the last materialize call on this thread submitted; lets
// benchmarks and tests re-launch / inspect exactly what the engine ran.
std::string last_descriptors();

// Planner verdict for one tensor, without allocating or launching anything (works without a GPU:
// used by CPU tests and by `torchdistx_b200.deferred_init.plan_report`).
struct PlanSegment {
  int64_t begin = 0, end = 0;  // elements of the tensor
  int64_t origin = 0;          // element of the tensor that is element 0 of the source op's tensor
  std::string source;          // "uninit" | "const" | "uniform" | "normal" | "iota" | "sincos" | "gather" | "band"
  double p0 = 0, p1 = 0;
  bool wide = false, src_noround = false;
  std::vector<std::tuple<int, double, double>> epilogue;
  std::string const_bytes;
  int rng_pass = -1;           // index into PlanInfo::rng_numels of the live RNG pass
  int64_t iota_period = 0, iota_repeat = 0;  // "iota": broadcast geometry (TdxInitDesc.fill_bits)
  // "sincos": H (the table is [R, 2H]) and the [cos | sin] order (TdxInitDesc.fill_bits); p0, p1 and
  // the epilogue are the column index program
  int64_t sincos_half = 0;
  bool sincos_cos_first = false;
  // "gather": a copy of a host-built tensor -- its broadcast geometry {P, R} (TdxInitDesc.fill_bits[1])
  // and the source's bytes in the tensor's dtype (P elements; for P = 0, those of the copied range)
  int64_t gather_period = 0, gather_repeat = 0;
  std::string gather_bytes;
  // "band": a band mask of an [..., R, C] tensor (TdxInitDesc.fill_bits): element (r, c) holds the bits
  // band_in when band_lo <= c - r <= band_hi and band_out otherwise (little-endian element bits)
  int64_t band_rows = 0, band_cols = 0, band_lo = 0, band_hi = 0;
  uint64_t band_in = 0, band_out = 0;
  // RngStream::Aten, a drawn segment: the draw ran on fp32 and is rounded at the store
  // (TDX_ALGO_ATEN_WIDE), whether or not anything can observe the fp32 tensor -- unlike `wide`
  bool aten_wide = false;
};

struct PlanInfo {
  bool deferred = false;   // the tensor awaits materialisation
  bool fusible = false;    // its program folds into one descriptor
  std::string source;      // "uninit" | "const" | "uniform" | "normal" | "opaque" | "real"
  std::string dtype;
  int64_t numel = 0;
  double p0 = 0, p1 = 0;
  int n_epilogue = 0;
  int rng_ops = 0;         // RNG passes on the chain, live + dead
  bool wide = false;       // fp32 source cast to a 16-bit dtype: TDX_ALGO_WIDE32
  bool src_noround = false;  // TDX_FLAG_SRC_NOROUND
  std::string first_unfusable_op;  // for "opaque": the op that stopped the fold (best effort)
  // everything needed to rebuild the descriptor later without the recording (InitPlan)
  std::vector<int64_t> sizes;
  std::string device;
  bool requires_grad = false;
  std::vector<std::tuple<int, double, double>> epilogue;  // (TDX_EPI_*, a, b)
  std::string const_bytes;                                 // "const": one element's bytes
  std::vector<int64_t> rng_numels;  // global numel of every RNG pass on the chain, in order
  // identity of every RNG pass (stable inside one recording): a clone shares its source's passes,
  // so a pass met again under another tensor consumes nothing and yields the same stream
  std::vector<int64_t> rng_op_ids;
  // the tensor as a list of disjoint segments (one for a tensor initialised as a whole; three for
  // `w.normal_(); w[padding_idx].zero_()`); the scalar fields above describe the largest one
  std::vector<PlanSegment> segments;
  // RngStream::Aten: why ATen's stream cannot take the storage's random program ("": it can; then
  // `fusible` is the default stream's verdict, else false).  Computed without a device: the grid
  // stride a draw takes depends on the device that materialises it.
  std::string aten_refusal;
};
PlanInfo plan_info(const at::Tensor& fake, RngStream rng = RngStream::Fused);
// Every recorded op touching the tensor's storage, in order (debug aid for unfusable programs).
std::vector<std::string> storage_history(const at::Tensor& fake);

// The tensor that a previous materialisation handed to Python for this fake tensor (keeps the
// Python object identity stable), and the hook to store it.
at::Tensor cached_python_tensor(const at::Tensor& fake);
void cache_python_tensor(const at::Tensor& fake, const at::Tensor& wrapped);

}  // namespace tdx
