// The engine: emits the descriptors of the storages that lower (Batch, Engine::emit_from), replays
// the others through ATen, and the materialise calls built on it (MaterializeSession, flat shards).
#include "planner_internal.h"

#include <ATen/Context.h>
#include <ATen/Functions.h>
#include <ATen/ThreadLocalState.h>
#include <ATen/core/Generator.h>
#include <ATen/cuda/EmptyTensor.h>
#include <c10/core/DeviceGuard.h>
#include <c10/cuda/CUDACachingAllocator.h>
#include <c10/cuda/CUDAFunctions.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime_api.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <functional>
#include <mutex>

#include "fake_tensor.h"
#include "stack_walk.h"

namespace tdx {

using c10::IValue;
using c10::ScalarType;
using torch::jit::Stack;

thread_local MaterializeStats g_stats;
thread_local double g_pending_traverse_us = 0;
thread_local std::vector<TdxInitDesc> g_last_descs;  // what the last materialize call launched

double now_us() {
  return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

namespace {

// ---------------------------------------------------------------------------------------------
// batched fused execution
// ---------------------------------------------------------------------------------------------
thread_local double g_call_begin_us = 0;

// Memory of the fused outputs.  A call's tensors are carved out of ONE allocation per submission
// (a "slab"): one trip to the caching allocator -- and, on a cold allocator, one cudaMalloc instead
// of one per tensor (226 of them for Llama-3-8B: ~0.6 s) -- while every tensor still gets a
// StorageImpl of its own (no aliasing is visible through storage identity, `torch.save` writes
// them separately, `untyped_storage().resize_()` works).  The slab goes back to the allocator
// when the last tensor carved from it dies.
struct Slab {
  c10::DataPtr block;
};
void slab_ref_delete(void* ctx) { delete static_cast<std::shared_ptr<Slab>*>(ctx); }

// Bytes of one element of a descriptor's destination (include/tdx_init.h dtypes).
size_t itemsize_of(uint8_t dtype) {
  switch (dtype) {
    case TDX_F32: case TDX_RAW32: return 4;
    case TDX_BF16: case TDX_F16: case TDX_RAW16: return 2;
    case TDX_RAW8: return 1;
    default: return 8;  // TDX_I64, TDX_RAW64
  }
}

std::atomic<uint64_t> g_epoch{1};  // process-wide: storages remember the epoch across sessions

struct Batch {
  c10::Device device = c10::Device(c10::kCPU);
  std::vector<TdxInitDesc> descs;
  // The descriptors' destinations are host memory (a CPU `out` of a flat shard: FSDP1's offload_params):
  // flush() runs them through tdx_init_submit_host.  A batch never mixes the two: flush before switching.
  bool host = false;
  // Outputs whose memory is assigned at the next submission: the tensor object exists as soon as
  // its program has been planned (the caller can give it its Python identity meanwhile), its
  // storage gets its address when the slab is allocated.
  struct Pending {
    c10::intrusive_ptr<c10::StorageImpl> storage;
    size_t nbytes = 0;
    uint32_t first_desc = 0, n_desc = 0;  // descriptors whose dst is relative to this tensor's base
  };
  std::vector<Pending> pending;
  // TDX_SRC_GATHER descriptors (index into descs) and their host sources: flush() stages the sources
  // on the device and fills in their addresses
  std::vector<std::pair<uint32_t, at::Tensor>> gathers;
  // Early submission: the first descriptors are launched as soon as a modest amount of work has
  // accumulated, so the GPU starts writing while the host is still planning the rest of the
  // module; the threshold grows after every submission so that the launch count (each launch
  // has a ~10-20 us tail) stays logarithmic.
  int64_t pending_bytes = 0;
  uint64_t epoch = g_epoch.fetch_add(1);  // bumped by every submission: a storage whose fused_epoch == epoch is not on the GPU yet
  // 256 MiB keeps the first launch early when a rank only owns 1/8 of the model
  int64_t flush_threshold = int64_t{256} << 20;
  // (Submission points depend on bytes only, never on timing: a call then cuts the same slabs every
  // time, which is what lets the caching allocator serve them from its free lists.  A gate on the
  // estimated GPU backlog -- submit only when the GPU is about to run dry -- saved one launch per
  // call at N = 1 and cost a cudaMalloc, i.e. a device synchronisation, whenever the cut moved.)
  // When the call materialises a whole recording the total is known in advance (Tape::fused_bytes,
  // divided by the world size of a sharded call), and so is how fast the host plans relative to the
  // GPU: planning costs ~1.5 us per tensor whatever its size, the kernels write ~4.8 GB/ms.  After
  // the first (256 MiB) submission the rest is cut into at most three more whose sizes grow by the
  // ratio q of the two rates, clamped to [1, 4]: with big tensors (one GPU, q = 4) the GPU is the
  // bottleneck and every chunk hides the planning of the next, larger one -- three launches for
  // 16 GB; when a rank owns an eighth of the model the host is as slow as the GPU (q = 1), the call
  // ends one chunk's GPU time after the last tensor has been planned, and equal chunks make that
  // the smallest.  A function of byte counts only, like the fallback rule (x4 per submission) that
  // applies when there is no estimate or the call outgrows it.
  int64_t expected_total = 0, expected_tensors = 0, submitted_bytes = 0;
  c10::SmallVector<int64_t, 4> schedule;  // thresholds of the submissions after the first
  size_t schedule_pos = 0;
  int64_t last_threshold = 0;
  void expect(int64_t total_bytes, int64_t tensors) {
    if (expected_total == 0 && submitted_bytes == 0) {
      expected_total = total_bytes;
      expected_tensors = tensors;
    }
  }
  int64_t next_threshold() {
    constexpr int64_t kNever = int64_t{1} << 62;
    const int64_t fallback = std::min<int64_t>(last_threshold * 4, int64_t{64} << 30);
    if (expected_total <= 0) return fallback;
    if (submitted_bytes >= expected_total) {  // more than the recording promised (several recordings in one call)
      expected_total = 0;
      return fallback;
    }
    if (schedule.empty()) {
      const double rest = static_cast<double>(expected_total - submitted_bytes);
      const double per_tensor = static_cast<double>(expected_total) / static_cast<double>(std::max<int64_t>(expected_tensors, 1));
      const double q = std::min(4.0, std::max(1.0, per_tensor / 7.2e6));
      int m = 1;
      double sum = q, term = q;
      while (m < 3 && static_cast<double>(submitted_bytes) * sum < rest) {
        ++m;
        term *= q;
        sum += term;
      }
      term = q;
      for (int i = 0; i + 1 < m; ++i) {  // the last chunk is whatever is left when the call ends
        schedule.push_back(std::max<int64_t>(static_cast<int64_t>(rest * term / sum), int64_t{64} << 20));
        term *= q;
      }
      schedule.push_back(kNever);
    }
    const int64_t t = schedule[std::min(schedule_pos, schedule.size() - 1)];
    ++schedule_pos;
    return t;
  }
  // A submission of `bytes` is cut: counts it and moves the threshold to the next cut.
  void cut(int64_t bytes) {
    submitted_bytes += bytes;
    if (flush_threshold < (int64_t{1} << 60)) last_threshold = flush_threshold;
    flush_threshold = next_threshold();
  }
  void note(int64_t bytes) {
    pending_bytes += bytes;
    if (pending_bytes >= flush_threshold) {
      cut(pending_bytes);
      flush();
    }
  }
  void assign_memory();
  void flush();
};

// An output tensor without memory yet (see Batch::Pending).  Built like at::detail::empty_generic
// does, minus the allocation.
at::Tensor make_output(c10::IntArrayRef sizes, ScalarType dtype, c10::Device dev, size_t nbytes,
                       c10::intrusive_ptr<c10::StorageImpl>& storage_out) {
  c10::Allocator* alloc = c10::cuda::CUDACachingAllocator::get();
  storage_out = c10::make_intrusive<c10::StorageImpl>(c10::StorageImpl::use_byte_size_t(),
                                                      static_cast<int64_t>(nbytes),
                                                      c10::DataPtr(nullptr, dev), alloc, /*resizable=*/true);
  at::Tensor t = at::detail::make_tensor<c10::TensorImpl>(
      c10::Storage(storage_out), c10::DispatchKeySet(c10::DispatchKey::CUDA), c10::scalarTypeToTypeMeta(dtype));
  t.unsafeGetTensorImpl()->generic_set_sizes_contiguous(sizes);
  return t;
}

void Batch::assign_memory() {
  if (pending.empty()) return;
  const double t0 = now_us();
  c10::Allocator* alloc = c10::cuda::CUDACachingAllocator::get();
  constexpr size_t kAlign = 256;  // vector stores need 16; 256 keeps every tensor on its own L2 lines
  if (pending.size() > 1) {
    // Slabs hold at most kSlabBytes (a tensor larger than that gets one of its own) and their sizes
    // are rounded to 1/32 of a power of two (<= 3 % over): where a call cuts its submissions depends on
    // timing, and slabs of arbitrary sizes would miss the caching allocator's free lists from one
    // call to the next (a miss is a cudaMalloc -- milliseconds, and a device synchronisation).
    constexpr size_t kSlabBytes = size_t{1} << 30;
    auto rounded = [](size_t n) {
      if (n <= (size_t{2} << 20)) return (n + 511) & ~size_t{511};
      size_t p2 = size_t{1} << 21;
      while (p2 < n) p2 <<= 1;
      const size_t step = p2 >> 5;
      return (n + step - 1) / step * step;
    };
    size_t i = 0;
    while (i < pending.size()) {
      size_t j = i, total = 0;
      while (j < pending.size()) {
        const size_t sz = (pending[j].nbytes + kAlign - 1) & ~(kAlign - 1);
        if (j > i && total + sz > kSlabBytes) break;
        total += sz;
        ++j;
      }
      if (total) {
        auto slab = std::make_shared<Slab>();
        slab->block = alloc->allocate(rounded(total));
        char* base = static_cast<char*>(slab->block.get());
        size_t off = 0;
        for (size_t k = i; k < j; ++k) {
          Pending& p = pending[k];
          if (p.nbytes == 0) continue;
          char* ptr = base + off;
          off += (p.nbytes + kAlign - 1) & ~(kAlign - 1);
          p.storage->set_data_ptr_noswap(
              c10::DataPtr(ptr, new std::shared_ptr<Slab>(slab), &slab_ref_delete, device));
          for (uint32_t q = p.first_desc; q < p.first_desc + p.n_desc; ++q)
            descs[q].dst = ptr + reinterpret_cast<uintptr_t>(descs[q].dst);
        }
      }
      i = j;
    }
  } else {
    for (Pending& p : pending) {
      if (p.nbytes == 0) continue;
      c10::DataPtr d = alloc->allocate(p.nbytes);
      char* ptr = static_cast<char*>(d.get());
      p.storage->set_data_ptr_noswap(std::move(d));
      for (uint32_t k = p.first_desc; k < p.first_desc + p.n_desc; ++k)
        descs[k].dst = ptr + reinterpret_cast<uintptr_t>(descs[k].dst);
    }
  }
  pending.clear();
  g_stats.alloc_us += now_us() - t0;
}

void Batch::flush() {
  NoInterception guard;
  c10::DeviceGuard dg(device.is_cuda() ? device : c10::Device(c10::kCPU));
  assign_memory();
  if (descs.empty()) {
    epoch = g_epoch.fetch_add(1);
    pending_bytes = 0;
    return;
  }
  const double t0 = now_us();
  const int n = static_cast<int>(descs.size());
  // the sources of copies of host-built tensors: one pinned buffer, one copy on the submission's
  // stream ahead of the kernels (the pinned block is not reused before the copy has left it, the
  // device block -- like the workspace -- is freed into the stream's own reuse order at the end)
  at::Tensor gather_dev;
  if (!gathers.empty()) {
    std::vector<std::pair<const c10::TensorImpl*, size_t>> placed;  // (a source shared by several descriptors goes once)
    std::vector<size_t> at_of(gathers.size());
    size_t total = 0;
    for (size_t k = 0; k < gathers.size(); ++k) {
      const at::Tensor& src = gathers[k].second;
      size_t off = static_cast<size_t>(-1);
      for (const auto& p : placed)
        if (p.first == src.unsafeGetTensorImpl()) off = p.second;
      if (off == static_cast<size_t>(-1)) {
        off = total;
        placed.emplace_back(src.unsafeGetTensorImpl(), off);
        total += (src.nbytes() + 15) & ~size_t{15};
      }
      at_of[k] = off;
    }
    at::Tensor host = at::empty({static_cast<int64_t>(total)}, at::TensorOptions().dtype(at::kByte).pinned_memory(true));
    gather_dev = at::empty({static_cast<int64_t>(total)}, at::TensorOptions().dtype(at::kByte).device(device));
    auto* hp = static_cast<unsigned char*>(host.data_ptr());
    const uintptr_t dp = reinterpret_cast<uintptr_t>(gather_dev.data_ptr());
    for (size_t k = 0; k < gathers.size(); ++k) {
      const at::Tensor& src = gathers[k].second;
      std::memcpy(hp + at_of[k], src.data_ptr(), src.nbytes());
      descs[gathers[k].first].fill_bits[0] = static_cast<uint64_t>(dp + at_of[k]);
    }
    gather_dev.copy_(host, /*non_blocking=*/true);
    gathers.clear();
  }
  auto stream = c10::cuda::getCurrentCUDAStream(device.index());
  if (host) {
    // host destinations: built in passes through one staging buffer of at most the first submission's
    // size (flush_threshold's start), and never more than the whole table needs
    size_t need = tdx_init_workspace_bytes(3 * n);
    for (const TdxInitDesc& d : descs) need += d.elem_count * itemsize_of(d.dtype) + 16;
    const size_t staging_bytes = std::min<size_t>(need, size_t{256} << 20);
    at::Tensor staging = at::detail::empty_cuda({static_cast<int64_t>(staging_bytes)}, at::kByte, device, std::nullopt);
    const int rc = tdx_init_submit_host(descs.data(), n, staging.data_ptr(), staging_bytes, stream.stream());
    TORCH_CHECK(rc == 0, "libtdx_init: host submission failed (", rc, "): ", tdx_last_error());
    g_stats.host_copies += tdx_last_host_copies();
    for (const TdxInitDesc& d : descs) g_stats.host_bytes += static_cast<int64_t>(d.elem_count * itemsize_of(d.dtype));
  } else {
    // prepare: the plan is laid out on the host and says how much workspace it needs (descriptor table
    // + prefix sums + work lists: tens of KB, not the upper bound of tdx_init_workspace_bytes)
    size_t ws_bytes = 0;
    int rc = tdx_init_prepare(descs.data(), n, &ws_bytes);
    TORCH_CHECK(rc == 0, "libtdx_init: plan failed (", rc, "): ", tdx_last_error());
    // (straight from the caching allocator: freed at the end of this scope, reused in stream order)
    at::Tensor ws = at::detail::empty_cuda({static_cast<int64_t>(std::max<size_t>(ws_bytes, 16))}, at::kByte,
                                           device, std::nullopt);
    rc = tdx_init_submit(ws.data_ptr(), ws_bytes, stream.stream());
    TORCH_CHECK(rc == 0, "libtdx_init: launch failed (", rc, "): ", tdx_last_error());
  }
  g_stats.kernel_launches += tdx_last_launch_count();
  g_stats.descriptors += n;
  g_stats.submissions++;
  g_stats.upload_bytes += static_cast<int64_t>(tdx_last_upload_bytes());
  if (g_stats.first_submit_us == 0) g_stats.first_submit_us = now_us() - g_call_begin_us;
  g_stats.last_submit_us = now_us() - g_call_begin_us;
  g_last_descs.insert(g_last_descs.end(), descs.begin(), descs.end());
  descs.clear();
  pending_bytes = 0;
  epoch = g_epoch.fetch_add(1);
  g_stats.launch_us += now_us() - t0;
}

// Generator state is read once per materialize call and written back once (a CUDA generator's
// set_offset() asks the driver whether the stream is capturing: ~1 us, twice per tensor).
struct GenCache {
  struct Entry {
    at::Generator gen;
    uint64_t seed = 0, offset = 0;
    bool dirty = false;
  };
  std::vector<Entry> entries;
  // the default generator of a device, looked up once per materialize call (the global context's
  // accessor takes a lock and re-validates the device on every call)
  std::vector<std::pair<c10::Device, at::Generator>> defaults;
  const at::Generator& default_generator(c10::Device device) {
    for (const auto& d : defaults)
      if (d.first == device) return d.second;
    defaults.emplace_back(device, at::globalContext().defaultGenerator(device));
    return defaults.back().second;
  }
  Entry& get(const at::Generator& g) {
    for (auto& e : entries)
      if (e.gen.unsafeGetGeneratorImpl() == g.unsafeGetGeneratorImpl()) return e;
    Entry e;
    e.gen = g;
    std::lock_guard<std::mutex> lock(e.gen.mutex());
    e.seed = g.current_seed();
    e.offset = g.get_offset();
    entries.push_back(std::move(e));
    return entries.back();
  }
  // must run before anything else (ATen replay, the user) looks at the generators
  void write_back() {
    for (auto& e : entries) {
      if (!e.dirty) continue;
      std::lock_guard<std::mutex> lock(e.gen.mutex());
      e.gen.set_offset(e.offset);
      e.dirty = false;
    }
    entries.clear();
  }
};

// The grid stride S of ATen's launch of a draw of `numel` elements on `device` (aten_stream_policy).
uint32_t aten_grid_stride(int64_t numel, c10::Device device) {
  static std::mutex mu;
  static std::vector<std::pair<int, int>> props;  // per device: (#SM, max threads per SM)
  const int idx = device.has_index() ? device.index() : c10::cuda::current_device();
  std::pair<int, int> p;
  {
    std::lock_guard<std::mutex> lock(mu);
    if (props.size() <= static_cast<size_t>(idx)) props.resize(idx + 1, {0, 0});
    if (props[idx].first == 0) {
      int sm = 0, tps = 0;
      TORCH_CHECK(cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, idx) == cudaSuccess &&
                      cudaDeviceGetAttribute(&tps, cudaDevAttrMaxThreadsPerMultiProcessor, idx) == cudaSuccess,
                  "cannot read the properties of CUDA device ", idx);
      props[idx] = {sm, tps};
    }
    p = props[idx];
  }
  return aten_stream_policy(numel, p.first, p.second).first;
}

// Gives an RNG op its Philox stream id (once) and advances the generator, so that replaying in
// the same order with the same seed reproduces the same tensors, dead passes included.  `aten`:
// the op takes ATen's own stream and advances the generator as ATen's launch of it does.
void assign_rng(Tape& tape, RngSlot& slot, int64_t numel, c10::Device device, GenCache& cache, bool aten) {
  if (slot.assigned) return;
  at::Generator gen;
  if (slot.explicit_generator) {
    const TapeOp& op = tape.ops[slot.op];
    const size_t pos = find_arg(op, "generator");
    if (pos != static_cast<size_t>(-1) && op.args[pos].isGenerator()) gen = op.args[pos].toGenerator();
  }
  if (!gen.defined()) gen = cache.default_generator(device);
  TORCH_CHECK(gen.device().type() == device.type(), "Expected a '", device.type(),
              "' device type for generator but found '", gen.device().type(), "'");
  GenCache::Entry& e = cache.get(gen);
  slot.seed = e.seed;
  slot.offset = e.offset;
  // consumption is a function of the GLOBAL element count only: shard-invariant by construction
  if (aten) {
    if (numel > 0) {  // (ATen draws nothing for an empty tensor)
      slot.stride = aten_grid_stride(numel, device);
      e.offset += aten_offset_increment(numel, slot.stride);
    }
  } else {
    const uint64_t blocks = (static_cast<uint64_t>(numel) + 3) / 4;
    e.offset += ((blocks + 3) / 4) * 4 + 4;
  }
  e.dirty = true;
  slot.assigned = true;
}

struct ShardGeom {
  int64_t begin = 0, count = 0;
  c10::SmallVector<int64_t, 4> sizes;
  // Shard(dim >= 1): the block is `runs` runs of `width` consecutive elements, `pitch` apart, the
  // first at `begin` (include/tdx_init.h TDX_FLAG_WINDOW); dim 0: one run
  int64_t runs = 1, width = 0, pitch = 0;
};

ShardGeom shard_of(const ValueInfo& v, const std::optional<ShardSpec>& shard) {
  ShardGeom g;
  g.sizes = v.sizes;
  g.begin = 0;
  g.count = v.numel;
  g.width = g.count;
  if (!shard || shard->world <= 1 || v.sizes.empty()) return g;  // 0-dim tensors are replicated
  const int64_t dim = shard->dim;
  TORCH_CHECK_VALUE(dim >= 0 && dim < static_cast<int64_t>(v.sizes.size()), "shard dim ", dim, " of a ",
                    v.sizes.size(), "-dim tensor");
  const int64_t d0 = v.sizes[dim];
  int64_t outer = 1, inner = 1;
  for (int64_t k = 0; k < dim; ++k) outer *= v.sizes[k];
  for (size_t k = dim + 1; k < v.sizes.size(); ++k) inner *= v.sizes[k];
  const int64_t per = (d0 + shard->world - 1) / shard->world;  // torch.chunk row count
  const int64_t start = std::min(d0, shard->rank * per);
  const int64_t len = std::min(per, d0 - start);
  g.begin = start * inner;
  g.count = outer * len * inner;
  g.sizes[dim] = len;
  g.runs = outer;
  g.width = len * inner;
  g.pitch = d0 * inner;
  return g;
}

at::Tensor alias_of(const at::Tensor& base, const ValueInfo& v, bool first) {
  const bool same = base.sizes() == c10::IntArrayRef(v.sizes) &&
                    base.strides() == c10::IntArrayRef(v.strides) &&
                    base.storage_offset() == v.storage_offset;
  if (same && first) return base;  // the common case: the parameter IS the backing tensor
  NoInterception guard;
  at::Tensor t = base.detach();
  if (!same) t.as_strided_(v.sizes, v.strides, v.storage_offset);
  return t;
}

// Under RngStream::Aten a storage takes the kernels only if ATen launches every draw on it, live or
// dead, as one 32-bit, trivially 1-D iterator, and if every epilogue step of a drawn segment is one
// the kernels compute bit for bit as ATen's CUDA op does (planner_eval.cc aten_draw_refusal,
// aten_exact_step; plan_info(rng="aten") reports the same verdict).  Everything else is replayed
// through ATen.
bool aten_fusible(const Tape& tape, const StorageTemplate& t) {
  if (!aten_draw_refusal(tape, t.st.rng_chain).empty()) return false;
  for (const FastSeg& sg : t.segs) {
    if (sg.rng_slot == kNoValue) continue;
    for (int i = 0; i < sg.proto.n_epi; ++i)
      if (!aten_exact_step(sg.proto.epi[i].op)) return false;
  }
  return true;
}

// ---------------------------------------------------------------------------------------------
// generic replay
// ---------------------------------------------------------------------------------------------
struct Engine {
  MaterializeOptions opts;
  Batch& batch;
  GenCache gens;

  bool sharding(const ValueInfo& vi) const { return opts.shard && opts.shard->world > 1 && !vi.sizes.empty(); }

  at::Tensor real_of(Tape& tape, uint32_t v) {
    ValueInfo& vi = tape.values[v];
    StorageInfo& si = tape.storages[vi.storage];
    if (vi.real.defined() && !(si.fused_done && si.base_is_shard && !sharding(vi))) return vi.real;
    TORCH_INTERNAL_ASSERT(si.fused_done, "value of `", tape.ops[vi.op].name(),
                          "` requested before it was materialised");
    if (si.base_is_shard) {
      if (sharding(vi)) {
        // the backing tensor is this rank's dim-0 chunk; only whole-storage tensors can name it
        TORCH_CHECK(vi.covers_storage,
                    "sharded materialisation only supports tensors that cover their whole storage");
        vi.real = si.base_taken ? [&] { NoInterception guard; return si.base.detach(); }() : si.base;
        si.base_taken = true;
        return vi.real;
      }
      // A reader (a buffer computed from a parameter, say) needs the unsharded tensor of a storage
      // whose backing tensor is one rank's chunk: every element is a function of (seed, offset,
      // index), so the full tensor is generated beside the chunk -- same bits, no communication.
      if (!si.full_base.defined()) {
        int64_t bytes = 0;
        TORCH_INTERNAL_ASSERT(emit_fused(tape, vi.storage, vi, std::nullopt, si.full_base, bytes),
                              "a fused storage stopped being fusible");
        si.fused_epoch = batch.epoch;
      }
      return alias_of(si.full_base, vi, false);  // (not cached in vi.real: that names this rank's view)
    }
    vi.real = alias_of(si.base, vi, !si.base_taken);
    si.base_taken = true;
    return vi.real;
  }

  c10::Device target_device(c10::Device recorded) {
    c10::Device d = opts.device ? *opts.device : recorded;
    if (d.is_cuda() && !d.has_index()) {  // "cuda" = the current device, asked for once per call
      if (current_cuda < 0) current_cuda = c10::cuda::current_device();
      d = c10::Device(c10::kCUDA, current_cuda);
    }
    return d;
  }
  c10::DeviceIndex current_cuda = -1;

  void collect_storage(Tape& tape, uint32_t S, uint32_t upto, std::vector<uint8_t>& mark,
                       std::vector<uint32_t>& visited_upto) {
    if (visited_upto[S] >= upto) return;
    visited_upto[S] = upto;
    if (tape.storages[S].fused_done) return;  // its content comes from the kernels (real_of): nothing to replay
    const auto& touching = tape.storages[S].touching_ops;
    uint32_t last_writer = kNoValue;
    for (uint32_t oi : touching) {
      if (oi >= upto) break;
      for (uint32_t v : tape.ops[oi].outputs)
        if (v != kNoValue && tape.values[v].storage == S) last_writer = oi;
    }
    if (last_writer == kNoValue) return;
    for (size_t k = 0; k < touching.size(); ++k) {
      const uint32_t oi = tape.storages[S].touching_ops[k];
      if (oi > last_writer) break;
      collect_op(tape, oi, mark, visited_upto);
    }
  }

  void collect_op(Tape& tape, uint32_t oi, std::vector<uint8_t>& mark,
                  std::vector<uint32_t>& visited_upto) {
    if (mark[oi] || tape.ops[oi].done) return;
    mark[oi] = 1;
    for (size_t k = 0; k < tape.ops[oi].inputs.size(); ++k) {
      const uint32_t v = tape.ops[oi].inputs[k].value;
      if (v == kNoValue) continue;
      if (tape.values[v].real.defined()) {
        // Built already -- by the op that produced it.  In-place writers recorded on its storage after
        // that op and before this reader may still be waiting: `b = a.clone(); b[2:5].normal_();
        // c = b * 2` with `a` materialised first replays the clone as part of a's history (it reads
        // a), and `b * 2` then found b "real" and never ran the normal_.  Collect what is left of
        // the storage's history up to this op (ops that ran are skipped: TapeOp::done).
        collect_storage(tape, tape.values[v].storage, oi, mark, visited_upto);
        continue;
      }
      // A dependency whose whole program folds is built by the kernels (unsharded: the op reads all
      // of it), not replayed op by op: faster, and its values do not depend on whether it or its
      // reader was asked for first.  (A storage the reader saw in an intermediate state is opaque
      // to the planner -- eval_storage's reader rule -- and is replayed up to `oi` as before.)
      if (!tape.storages[tape.values[v].storage].fused_done) {
        const std::optional<ShardSpec> saved = opts.shard;
        opts.shard = std::nullopt;
        const bool fused = try_fused(tape, v);
        opts.shard = saved;
        if (fused) continue;
      }
      collect_storage(tape, tape.values[v].storage, oi, mark, visited_upto);
    }
  }

  void replay(Tape& tape, uint32_t oi) {
    TapeOp& op = tape.ops[oi];
    if (op.done) return;
    const size_t nargs = op.args.size();
    Stack stack;
    stack.reserve(nargs);
    for (const IValue& a : op.args) {
      if (a.isList()) {  // fresh list: we are about to put tensors into it
        const auto& src = a.toList();
        c10::impl::GenericList l(src.elementType());
        for (const IValue& e : a.toListRef()) l.push_back(e);
        stack.emplace_back(std::move(l));
      } else {
        stack.push_back(a);
      }
    }
    size_t slot = 0;
    for_each_tensor_mut(stack, nargs, [&](at::Tensor& t) {
      InputRef& in = op.inputs[slot++];
      if (in.value != kNoValue) {
        t = real_of(tape, in.value);
        // a fused result that is still sitting in the batch must reach the stream before ATen reads it
        const StorageInfo& isi = tape.storages[tape.values[in.value].storage];
        if (isi.fused_done && isi.fused_epoch == batch.epoch) batch.flush();
      } else if (in.foreign) {
        // (recorded by an earlier deferred_init: same rule -- its descriptor may still be in the batch)
        // It is needed NOW, as an argument: the session's "replay RNG-free programs after the last
        // submission" rule is for tensors the caller asked for, and would hand back nothing here
        // (`b = deferred_init(lambda: a * 2 + 1)` with `a = deferred_init(torch.ones, ...)` raised
        // "Expected a proper Tensor but got None" unless `a` had been materialised first).
        struct NoDeferral {
          bool& flag;
          const bool saved;
          explicit NoDeferral(bool& f) : flag(f), saved(f) { flag = false; }
          ~NoDeferral() { flag = saved; }
        } now(defer_generic);
        t = materialize_value(in.foreign, in.foreign_value);
        const StorageInfo& fsi = in.foreign->storages[in.foreign->values[in.foreign_value].storage];
        if (fsi.fused_done && fsi.fused_epoch == batch.epoch) batch.flush();
      } else if (in.real.defined()) {
        TORCH_CHECK(!in.real.is_inference(), "A `Tensor` argument required for the materialization of `",
                    op.name(), "` was created in inference mode. Materialization cannot be performed "
                    "because in-place updates to inference tensors cannot be tracked.");
        TORCH_CHECK(static_cast<int64_t>(in.real._version()) == in.real_version,
                    "A `Tensor` argument required for the materialization of `", op.name(),
                    "` was updated in-place. Materialization cannot be performed.");
        t = in.real;
        if (opts.device && t.dim() != 0 && t.device() != *opts.device) t = t.to(*opts.device);
      }
    });
    if (opts.device && op.handle) {
      const int di = device_argument_index(*op.handle);
      if (di >= 0 && (stack[di].isDevice() || stack[di].isNone())) stack[di] = *opts.device;
    }
    {
      at::ThreadLocalStateGuard tls(*op.tls);  // (a shared snapshot: see tape.cc)
      NoInterception guard;
      if (op.handle) {
        op.handle->callBoxed(stack);
      } else if (op.kind == OpKind::HookVariableData) {
        at::Tensor self = stack[0].toTensor();
        stack.clear();
        stack.emplace_back(at::Tensor(self.variable_data()));
      } else {  // HookSetData
        at::Tensor self = stack[0].toTensor(), data = stack[1].toTensor();
        self.set_data(data);
        stack.clear();
        stack.emplace_back(self);
      }
    }
    size_t k = 0;
    for_each_tensor(stack, op.num_returns, [&](const at::Tensor& t) {
      if (k < op.outputs.size() && op.outputs[k] != kNoValue) {
        ValueInfo& ov = tape.values[op.outputs[k]];
        ov.real = t;
        tape.storages[ov.storage].replayed = true;  // its content now comes from ATen: never fuse it later
      }
      ++k;
    });
    op.results = std::move(stack);
    op.done = true;
    op.tls.reset();  // (args stay: a later analysis of the tape still reads their scalars)
    g_stats.generic_ops++;
  }

  // Builds the descriptors of storage S (or of one rank's dim-0 chunk of it) and the tensor they
  // write; `vi` is the value whose geometry the tensor takes (the parameter itself, normally).
  // Returns false if the program is not fusible.  `bytes_out`: algorithmic bytes of the descriptors.
  bool emit_fused(Tape& tape, uint32_t S, const ValueInfo& vi, const std::optional<ShardSpec>& shard,
                  at::Tensor& base_out, int64_t& bytes_out, Prebuilt* pre = nullptr) {
    const c10::Device dev = target_device(vi.device);
    StorageTemplate tmp;
    const StorageTemplate* t = template_of(tape, S, dev, tmp);
    return t && (opts.rng != RngStream::Aten || aten_fusible(tape, *t)) &&
           emit_from(tape, *t, vi, shard, dev, base_out, bytes_out, pre);
  }

  // The template storage S is emitted from on `dev`: the one the recording's analysis built, or one
  // evaluated now into `tmp`.  nullptr: some segment is not expressible as a descriptor.
  const StorageTemplate* template_of(Tape& tape, uint32_t S, c10::Device dev, StorageTemplate& tmp) {
    const StorageInfo& si = tape.storages[S];
    if (si.tmpl && si.tmpl->fast) {  // analysed when the recording ended: nothing to evaluate
      g_stats.template_hits++;
      return si.tmpl.get();
    }
    if (si.tmpl && si.tmpl->st.opaque) return nullptr;
    if (si.tmpl) {
      tmp.st = si.tmpl->st;  // (a constant whose bits need a tensor: rare)
    } else {
      FoldOn fold_on(dev);  // constants fold with the target device's arithmetic
      c10::DeviceGuard fold_guard(dev);
      const double t_eval = now_us();
      tmp.st = eval_storage(tape, S, static_cast<uint32_t>(tape.ops.size()));
      g_stats.eval_us += now_us() - t_eval;
    }
    return build_fast(si, tmp, /*may_sync=*/true) ? &tmp : nullptr;
  }

  // Appends the descriptor of `count` elements of segment `sg`, from storage element `lo` on, written
  // to `dst` (a byte offset inside a pending output, or an address), and adds its bytes to `bytes`.
  TdxInitDesc& stamp(Tape& tape, const FastSeg& sg, int64_t lo, void* dst, int64_t count, size_t isz,
                     int64_t& bytes) {
    if (sg.gather.defined()) batch.gathers.emplace_back(static_cast<uint32_t>(batch.descs.size()), sg.gather);
    batch.descs.push_back(sg.proto);
    TdxInitDesc& d = batch.descs.back();
    d.dst = dst;
    d.elem_count = static_cast<uint64_t>(count);
    if (sg.indexed) d.elem_begin = static_cast<uint64_t>(lo - sg.origin);  // index in the tensor the source op ran on
    if (sg.rng_slot != kNoValue) {
      const RngSlot& r = tape.rng[sg.rng_slot];
      d.philox_seed = r.seed;
      d.philox_offset = r.offset;
      if (opts.rng == RngStream::Aten) {  // (`wide` is kept whether or not the fp32 tensor is observable: it changes bits)
        d.algo = sg.wide ? TDX_ALGO_ATEN_WIDE : TDX_ALGO_ATEN;
        d.fill_bits[1] = r.stride;
      } else if (sg.wide && wide_observable(tape, *sg.sym)) {
        d.algo = TDX_ALGO_WIDE32;
      }
    }
    bytes += count * static_cast<int64_t>(isz);
    return d;
  }

  bool emit_from(Tape& tape, const StorageTemplate& t, const ValueInfo& vi, const std::optional<ShardSpec>& shard,
                 c10::Device dev, at::Tensor& base_out, int64_t& bytes_out, Prebuilt* pre = nullptr) {
    const State& st = t.st;
    const size_t isz = t.isz;
    // geometry of what this rank writes
    ShardGeom g;
    if (vi.covers_storage && vi.dtype == st.dtype) {
      g = shard_of(vi, shard);
    } else {
      g.begin = 0;
      g.count = t.numel;
      g.sizes.assign(1, t.numel);
    }
    // Shard(d >= 1) of a program with an index, table or copy segment: built whole (the caller narrows it)
    emitted_whole = false;
    if (g.runs > 1) {
      for (const FastSeg& sg : t.segs)
        emitted_whole |= sg.proto.src != TDX_SRC_CONST && sg.rng_slot == kNoValue;
      if (emitted_whole) g = shard_of(vi, std::nullopt);
    }
    if (batch.device != dev) {
      batch.flush();
      batch.device = dev;
    }
    Batch::Pending pend;
    pend.nbytes = static_cast<size_t>(g.count) * isz;
    at::Tensor base;
    if (pre && pre->out.defined() && pre->nbytes == pend.nbytes && pre->out.scalar_type() == st.dtype &&
        pre->out.device() == dev && pre->out.sizes() == c10::IntArrayRef(g.sizes)) {
      base = std::move(pre->out);  // the calling thread built the (memory-less) output while it walked the module
      pend.storage = std::move(pre->storage);
      g_stats.prebuilt_outputs++;
    } else {
      base = make_output(g.sizes, st.dtype, dev, pend.nbytes, pend.storage);
    }

    // every RNG pass on the chain consumes its slice of the stream, live or dead
    for (const RngPass& r : st.rng_chain) {
      RngSlot& slot = tape.rng[r.slot];
      if (slot.assigned) continue;
      assign_rng(tape, slot, r.numel, dev, gens, opts.rng == RngStream::Aten);
      bool live = false;
      for (const FastSeg& sg : t.segs) live |= sg.rng_slot == r.slot;
      if (!live) g_stats.elided_rng_ops++;
    }

    pend.first_desc = static_cast<uint32_t>(batch.descs.size());
    emitted_draw = false;
    for (const FastSeg& sg : t.segs) emitted_draw |= sg.rng_slot != kNoValue;
    int64_t bytes = 0;
    if (g.runs > 1) {
      bytes = emit_window(t, g, tape);
    } else for (const FastSeg& sg : t.segs) {
      const int64_t lo = std::max(sg.begin, g.begin), hi = std::min(sg.end, g.begin + g.count);
      // (dst: a byte offset inside the output until the submission gives the output its address)
      if (lo < hi) stamp(tape, sg, lo, reinterpret_cast<void*>(static_cast<uintptr_t>(lo - g.begin) * isz), hi - lo, isz, bytes);
    }
    pend.n_desc = static_cast<uint32_t>(batch.descs.size()) - pend.first_desc;
    batch.pending.push_back(std::move(pend));
    g_stats.bytes_written += bytes;
    bytes_out = bytes;
    base_out = std::move(base);
    return true;
  }
  bool emitted_whole = false;  // the last emit_from built the whole tensor in place of a Shard(d >= 1) block
  bool emitted_draw = false;   // the last emit_from wrote a random segment

  // The descriptors of a Shard(d >= 1) block (g.runs runs of g.width elements, g.pitch apart): per
  // segment, the partial runs at its ends are plain descriptors; its whole runs are one windowed
  // descriptor (RNG) or one constant fill (whole runs are contiguous in the block).  Returns the bytes.
  int64_t emit_window(const StorageTemplate& t, const ShardGeom& g, Tape& tape) {
    const int64_t W = g.width, P = g.pitch;
    if (W == 0) return 0;
    int64_t bytes = 0;
    for (const FastSeg& sg : t.segs) {
      auto push = [&](int64_t lo, int64_t local, int64_t count, int64_t runs) {
        TdxInitDesc& d = stamp(tape, sg, lo, reinterpret_cast<void*>(static_cast<uintptr_t>(local) * t.isz), count,
                               t.isz, bytes);
        if (runs > 1 && sg.rng_slot != kNoValue) {
          d.reserved |= TDX_FLAG_WINDOW;
          if (opts.rng == RngStream::Aten) {  // (fill_bits[1] is ATen's grid stride)
            d.fill_bits[0] = static_cast<uint64_t>(W) | (static_cast<uint64_t>(P) << 32);
          } else {
            d.fill_bits[0] = static_cast<uint64_t>(W);
            d.fill_bits[1] = static_cast<uint64_t>(P);
          }
        }
      };
      int64_t o = sg.begin <= g.begin ? 0 : (sg.begin - g.begin) / P;  // the first run that can meet the segment
      while (o < g.runs) {
        const int64_t rb = g.begin + o * P, re = rb + W;
        if (rb >= sg.end) break;
        const int64_t lo = std::max(rb, sg.begin), hi = std::min(re, sg.end);
        if (lo >= hi) {
          ++o;
          continue;
        }
        if (lo == rb && hi == re) {  // runs [o, last) lie inside the segment
          const int64_t last = std::min(g.runs, (sg.end - g.begin - W) / P + 1);
          push(rb, o * W, (last - o) * W, last - o);
          o = last;
        } else {
          push(lo, o * W + (lo - rb), hi - lo, 1);
          ++o;
        }
      }
    }
    return bytes;
  }

  // ---- FSDP1 layout ----------------------------------------------------------------------------
  // The parameters of one FlatParameter, flattened and concatenated in order (each start optionally
  // aligned to `align` elements), chunked `world` ways by torch.chunk's rule, the last chunk
  // right-padded with zeros ($TORCH/distributed/fsdp/_flat_param.py:1089-1140 `_get_shard`,
  // :560-640 alignment padding): rank r's chunk is written straight into one 1-D tensor.  Neither a
  // parameter nor the flat parameter ever exists unsharded.  Every parameter's RNG passes are
  // assigned whether or not its elements fall into this rank's chunk, so all ranks agree.
  at::Tensor flat_shard(const std::vector<at::Tensor>& fakes, int64_t rank, int64_t world, int64_t align,
                        const std::optional<at::Tensor>& out_opt, std::vector<int64_t>* offsets_out) {
    TORCH_CHECK_VALUE(world >= 1 && rank >= 0 && rank < world, "flat shard: 0 <= rank < world_size required");
    struct Item {
      std::shared_ptr<Tape> tape;
      uint32_t value = kNoValue;
      int64_t offset = 0, numel = 0;
    };
    std::vector<Item> items;
    items.reserve(fakes.size());
    ScalarType dtype = ScalarType::Undefined;
    std::optional<c10::Device> dev;
    int64_t total = 0;
    for (const at::Tensor& f : fakes) {
      TORCH_CHECK_VALUE(can_materialize(f), "flat shard: every parameter must be a deferred (fake) tensor");
      const auto rec = fake_impl(f)->record();
      const ValueInfo& vi = rec->tape->values[rec->value];
      if (dtype == ScalarType::Undefined) dtype = vi.dtype;
      TORCH_CHECK_VALUE(vi.dtype == dtype, "flat shard: parameters of one flat parameter share one dtype");
      const c10::Device d = target_device(vi.device);
      TORCH_CHECK_VALUE(d.is_cuda(), "flat shard: the target device must be a CUDA device");
      if (!dev) dev = d;
      TORCH_CHECK_VALUE(*dev == d, "flat shard: parameters live on different devices");
      if (align > 1 && total % align) total += align - total % align;
      Item it;
      it.tape = rec->tape;
      it.value = rec->value;
      it.offset = total;
      it.numel = vi.numel;
      total += vi.numel;
      if (offsets_out) offsets_out->push_back(it.offset);
      items.push_back(std::move(it));
    }
    TORCH_CHECK_VALUE(dev.has_value(), "flat shard: no parameters");
    const size_t isz = c10::elementSize(dtype);
    const int64_t chunk = (total + world - 1) / world;
    const int64_t lo = std::min(total, rank * chunk), hi = std::min(total, lo + chunk);
    if (offsets_out) offsets_out->push_back(total);

    if (batch.device != *dev) {
      batch.flush();
      batch.device = *dev;
    }
    at::Tensor out;
    Batch::Pending pend;
    char* abs_base = nullptr;
    const bool host_out = out_opt && out_opt->defined() && out_opt->device().is_cpu();
    if (host_out) {  // FSDP1's flat_param._local_shard under offload_params: built on *dev, copied to the host
      out = *out_opt;
      TORCH_CHECK_VALUE(out.scalar_type() == dtype && out.dim() == 1 && out.is_contiguous() && out.numel() >= chunk,
                        "flat shard: a CPU `out` must be a contiguous 1-D tensor of the parameters' dtype with at "
                        "least ceil(total / world) elements");
      abs_base = static_cast<char*>(out.data_ptr());
    } else if (out_opt && out_opt->defined()) {
      out = *out_opt;
      TORCH_CHECK_VALUE(out.is_cuda() && out.device() == *dev && out.scalar_type() == dtype && out.dim() == 1 &&
                            out.is_contiguous() && out.numel() >= chunk,
                        "flat shard: `out` must be a contiguous 1-D CUDA tensor of the parameters' dtype with at "
                        "least ceil(total / world) elements");
      abs_base = static_cast<char*>(out.data_ptr());
    } else {
      pend.nbytes = static_cast<size_t>(chunk) * isz;
      const int64_t sizes[1] = {chunk};
      out = make_output(sizes, dtype, *dev, pend.nbytes, pend.storage);
    }
    auto place = [&](int64_t flat_index) {  // dst of a flat element of this rank's chunk
      return reinterpret_cast<void*>(abs_base + static_cast<uintptr_t>(flat_index - lo) * isz);
    };
    auto zero_fill = [&](int64_t b, int64_t e) {  // alignment gaps and the right pad
      if (b >= e) return;
      TdxInitDesc d;
      std::memset(&d, 0, sizeof(d));
      d.src = TDX_SRC_CONST;
      d.dtype = raw_dtype(isz);
      d.dst = place(b);
      d.elem_count = static_cast<uint64_t>(e - b);
      batch.descs.push_back(d);
    };
    struct Deferred {  // parameters the kernels cannot express: replayed whole, then copied (after the flush)
      at::Tensor full;
      int64_t src_begin, dst_begin, count;
    };
    std::vector<Deferred> deferred;
    // Pass 1, in order (it is the order RNG offsets are handed out in): decide per parameter, assign
    // the RNG passes of the fusible ones, replay the others now -- a replay may submit the batch, so
    // none of this chunk's descriptors may be in it yet.
    std::vector<std::unique_ptr<StorageTemplate>> owned;
    std::vector<const StorageTemplate*> plan(items.size(), nullptr);
    for (size_t k = 0; k < items.size(); ++k) {
      const Item& it = items[k];
      Tape& tape = *it.tape;
      const ValueInfo& vi = tape.values[it.value];
      const uint32_t S = vi.storage;
      StorageInfo& si = tape.storages[S];
      const int64_t b = std::max(it.offset, lo), e = std::min(it.offset + it.numel, hi);
      const StorageTemplate* t = nullptr;
      bool fusible = opts.fused && !si.replayed && !si.fused_done && !vi.real.defined() && vi.covers_storage;
      if (fusible) {
        auto tmp = std::make_unique<StorageTemplate>();
        t = template_of(tape, S, *dev, *tmp);
        if (t == tmp.get()) owned.push_back(std::move(tmp));
        fusible = t != nullptr && t->st.dtype == dtype && (opts.rng != RngStream::Aten || aten_fusible(tape, *t));
      }
      if (!fusible) {
        // generic replay of the whole parameter on the GPU; its slice is copied into the chunk below
        at::Tensor full = materialize_value(it.tape, it.value);
        if (b < e) deferred.push_back(Deferred{full, b - it.offset, b, e - b});
        continue;
      }
      plan[k] = t;
      for (const RngPass& r : t->st.rng_chain) {  // every rank assigns every pass, owner or not
        RngSlot& slot = tape.rng[r.slot];
        if (!slot.assigned) assign_rng(tape, slot, r.numel, *dev, gens, opts.rng == RngStream::Aten);
      }
      if (opts.rng == RngStream::Aten)
        for (const FastSeg& sg : t->segs)
          if (sg.rng_slot != kNoValue) {
            g_stats.aten_stream_tensors++;
            break;
          }
    }
    if (batch.device != *dev || batch.host != host_out) {
      batch.flush();
      batch.device = *dev;
      batch.host = host_out;
    }
    pend.first_desc = static_cast<uint32_t>(batch.descs.size());
    // Pass 2: this chunk's descriptors (nothing else touches the batch from here to the flush)
    int64_t bytes = 0, covered = lo;  // [lo, covered) has been written or queued
    for (size_t k = 0; k < items.size(); ++k) {
      const Item& it = items[k];
      Tape& tape = *it.tape;
      const int64_t b = std::max(it.offset, lo), e = std::min(it.offset + it.numel, hi);
      zero_fill(covered, std::min(it.offset, hi));  // the alignment gap in front of this parameter
      covered = std::max(covered, std::min(it.offset + it.numel, hi));
      const StorageTemplate* t = plan[k];
      if (!t || b >= e) continue;
      const int64_t pb = b - it.offset, pe = e - it.offset;  // the parameter's own elements this rank holds
      for (const FastSeg& sg : t->segs) {
        const int64_t slo = std::max(sg.begin, pb), shi = std::min(sg.end, pe);
        if (slo < shi) stamp(tape, sg, slo, place(it.offset + slo), shi - slo, isz, bytes);
      }
    }
    zero_fill(covered, lo + chunk);  // the right zero-pad of the last rank(s): [hi, lo + chunk)
    if (!abs_base) {
      pend.n_desc = static_cast<uint32_t>(batch.descs.size()) - pend.first_desc;
      batch.pending.push_back(std::move(pend));
    }
    g_stats.bytes_written += bytes;
    g_stats.fused_tensors += static_cast<int64_t>(items.size() - deferred.size());
    batch.flush();
    batch.host = false;
    if (!deferred.empty()) {
      NoInterception guard;
      for (const Deferred& d : deferred)
        out.narrow(0, d.dst_begin - lo, d.count).copy_(d.full.reshape({-1}).narrow(0, d.src_begin, d.count));
    }
    if (host_out) {  // (copies into pinned memory are asynchronous: the caller reads `out` on the host next)
      const cudaError_t e = cudaStreamSynchronize(c10::cuda::getCurrentCUDAStream(dev->index()).stream());
      TORCH_CHECK(e == cudaSuccess, "flat shard: ", cudaGetErrorString(e));
    }
    return out;
  }

  // Fused path for the storage of value `v`.  Returns false if the program is not fusible.
  bool try_fused(Tape& tape, uint32_t v, Prebuilt* pre = nullptr) {
    ValueInfo& vi = tape.values[v];
    const uint32_t S = vi.storage;
    StorageInfo& si = tape.storages[S];
    if (!opts.fused || si.replayed) return false;
    if (!target_device(vi.device).is_cuda()) return false;
    const bool sharded = sharding(vi);
    if (sharded && !vi.covers_storage) return false;
    at::Tensor base;
    int64_t bytes = 0;
    if (!emit_fused(tape, S, vi, sharded ? opts.shard : std::nullopt, base, bytes, pre)) return false;
    si.base = std::move(base);
    si.base_is_shard = sharded && !emitted_whole;
    si.fused_done = true;
    si.fused_epoch = batch.epoch;
    if (opts.rng == RngStream::Aten && emitted_draw) g_stats.aten_stream_tensors++;
    // (the storage's writer ops are not marked done one by one: `fused_done` stops every walk over
    // them -- collect_storage, eval_storage's callers -- and costs no cache line per op)
    g_stats.fused_tensors++;
    if (batch.expected_total == 0 && tape.fused_bytes)
      batch.expect(static_cast<int64_t>(tape.fused_bytes / static_cast<uint64_t>(opts.shard ? std::max<int64_t>(opts.shard->world, 1) : 1)),
                   tape.fused_storages);
    batch.note(bytes);  // may submit what has accumulated so far
    return true;
  }

  // Does anything that determines storage S (as of op `upto`) draw random numbers?  A pure walk
  // over the recording (no side effects): programs without RNG can be replayed at any point of the
  // call without changing what anybody gets -- they neither read nor advance a generator.
  static bool is_random_op(const TapeOp& op) {
    switch (op.kind) {
      case OpKind::Randn: case OpKind::Rand: case OpKind::UniformInplace: case OpKind::NormalInplace: return true;
      default: break;
    }
    if (!op.handle) return false;
    const auto& schema = op.handle->schema();
    for (const auto& a : schema.arguments())
      if (a.name() == "generator") return true;
    const std::string& n = schema.name();
    return n.find("dropout") != std::string::npos || n.find("rrelu") != std::string::npos ||
           n.find("rand") != std::string::npos || n.find("bernoulli") != std::string::npos ||
           n.find("multinomial") != std::string::npos || n.find("poisson") != std::string::npos;
  }
  bool deterministic_slice(Tape& tape, uint32_t S, uint32_t upto, std::vector<uint32_t>& seen_upto) {
    if (seen_upto[S] >= upto) return true;
    seen_upto[S] = upto;
    const StorageInfo& si = tape.storages[S];
    if (si.fused_done) return true;
    // The same selection as collect_storage: every op that touches S up to its last writer is
    // replayed with it -- READERS included (they must see S at their point in history), and a reader
    // can draw random numbers through its other arguments: `torch.randn(n).copy_(s)` replays the
    // (dead) randn with s.  Looking at writers only let such a storage be deferred to the end of the
    // call, i.e. moved its reader's draw behind every later tensor's (1 of 3,000 random scripts
    // differed from the reference for that reason).
    uint32_t last_writer = kNoValue;
    for (uint32_t oi : si.touching_ops) {
      if (oi >= upto) break;
      for (uint32_t v : tape.ops[oi].outputs)
        if (v != kNoValue && tape.values[v].storage == S) last_writer = oi;
    }
    if (last_writer == kNoValue) return true;
    for (uint32_t oi : si.touching_ops) {
      if (oi > last_writer) break;
      const TapeOp& op = tape.ops[oi];
      if (op.done) continue;
      if (is_random_op(op)) return false;
      for (const InputRef& in : op.inputs) {
        if (in.foreign) return false;  // (another recording: keep it simple)
        if (in.value == kNoValue || tape.values[in.value].real.defined()) continue;
        if (!deterministic_slice(tape, tape.values[in.value].storage, oi, seen_upto)) return false;
      }
    }
    return true;
  }
  // Set by the session: unfusable programs without RNG are not replayed where the walk meets them but
  // after the call's last fused submission -- their dozen ATen dispatches (Llama's rotary inv_freq:
  // ~0.25 ms of host time) then run while the GPU already works on the whole model.
  bool defer_generic = false;

  // This rank's dim-0 chunk of a fully materialised tensor (generic replay always builds the whole
  // tensor: its ops are recorded on whole tensors).
  at::Tensor chunk_of(const ValueInfo& vi, const at::Tensor& full) {
    NoInterception guard;
    const ShardGeom g = shard_of(vi, opts.shard);
    const int64_t dim = opts.shard->dim;
    if (dim > 0) {  // (Shard(d >= 1): the rows of this rank are start = begin / inner ...)
      const int64_t inner = vi.sizes[dim] ? g.pitch / vi.sizes[dim] : 0;
      const int64_t start = inner ? g.begin / inner : 0;
      return full.narrow(dim, start, g.sizes[dim]).clone(at::MemoryFormat::Contiguous);
    }
    const int64_t inner = vi.sizes[0] ? vi.numel / vi.sizes[0] : 0;
    const int64_t start = inner ? g.begin / inner : 0;
    return full.narrow(0, start, g.sizes[0]).clone();
  }

  at::Tensor materialize_value(const std::shared_ptr<Tape>& tape_ptr, uint32_t v, Prebuilt* pre = nullptr) {
    Tape& tape = *tape_ptr;
    ValueInfo& vi = tape.values[v];
    StorageInfo& si = tape.storages[vi.storage];
    if (si.fused_done) {
      at::Tensor t = real_of(tape, v);
      // (materialised whole earlier -- as a dependency, or by an unsharded call -- and asked for as a chunk now)
      return (sharding(vi) && !si.base_is_shard) ? chunk_of(vi, t) : t;
    }
    if (vi.real.defined()) return sharding(vi) ? chunk_of(vi, vi.real) : vi.real;
    if (try_fused(tape, v, pre)) {
      if (sharding(vi) && !si.base_is_shard) {  // Shard(d >= 1) of an index, table or copy program
        batch.flush();  // (the narrow reads what the kernels write)
        g_stats.narrowed_tensors++;
        return chunk_of(vi, real_of(tape, v));
      }
      return real_of(tape, v);
    }
    if (defer_generic) {
      std::vector<uint32_t> seen(tape.storages.size(), 0);
      if (deterministic_slice(tape, vi.storage, static_cast<uint32_t>(tape.ops.size()), seen)) return at::Tensor();
    }

    // generic replay, in recorded order, of everything that determines this storage.  Pending fused
    // descriptors stay in the batch (replay() submits them first if one of its inputs is among them):
    // a module's few unfusable buffers do not split the batch into extra launches.
    gens.write_back();  // ATen's own RNG kernels read the generators
    std::vector<uint8_t> mark(tape.ops.size(), 0);
    std::vector<uint32_t> visited(tape.storages.size(), 0);
    collect_storage(tape, vi.storage, static_cast<uint32_t>(tape.ops.size()), mark, visited);
    for (uint32_t oi = 0; oi < mark.size(); ++oi)
      if (mark[oi]) replay(tape, oi);
    TORCH_INTERNAL_ASSERT(vi.real.defined(), "replay did not produce `", tape.ops[vi.op].name(), "`");
    return sharding(vi) ? chunk_of(vi, vi.real) : vi.real;
  }
};

}  // namespace

at::Tensor finish_tensor(const at::Tensor& fake, at::Tensor out) {
  // requires_grad_() is not an operator and cannot be recorded: re-apply it on leaves
  // (same rule as reference deferred_init.cc:722-726)
  if (fake.is_leaf() && fake.requires_grad() && !out.requires_grad() &&
      (out.is_floating_point() || out.is_complex())) {
    out.set_requires_grad(true);
  }
  return out;
}

// Runs on the thread that walks the module (while the helper plans earlier tensors): builds the
// memory-less output tensor of `fake` -- TensorImpl, StorageImpl, autograd meta: half of what a
// tensor costs the helper -- if the analysis left on the recording says its storage will take the
// fused path.  The helper checks the geometry again and falls back to its own if anything differs.
bool prebuild_output(const at::Tensor& fake, const MaterializeOptions& opts, bool apply_shard, Prebuilt& pre) {
  if (!opts.fused || !can_materialize(fake)) return false;
  const TensorRecord* rec = fake_impl(fake)->record().get();
  if (!rec || !rec->tape || rec->value == kNoValue) return false;
  const Tape& tape = *rec->tape;
  const ValueInfo& vi = tape.values[rec->value];
  const StorageInfo& si = tape.storages[vi.storage];
  const StorageTemplate* t = si.tmpl.get();
  if (!t || !t->fast || si.fused_done || si.replayed || vi.real.defined()) return false;
  c10::Device dev = opts.device ? *opts.device : vi.device;
  if (!dev.is_cuda()) return false;
  if (!dev.has_index()) dev = c10::Device(c10::kCUDA, c10::cuda::current_device());
  const bool sharded = apply_shard && opts.shard && opts.shard->world > 1 && !vi.sizes.empty();
  if (sharded && !vi.covers_storage) return false;
  ShardGeom g;
  if (vi.covers_storage && vi.dtype == t->st.dtype) {
    g = shard_of(vi, sharded ? opts.shard : std::nullopt);
  } else {
    g.count = t->numel;
    g.sizes.assign(1, t->numel);
  }
  pre.nbytes = static_cast<size_t>(g.count) * t->isz;
  pre.out = make_output(g.sizes, t->st.dtype, dev, pre.nbytes, pre.storage);
  return true;
}

struct MaterializeSession::Impl {
  MaterializeOptions opts;
  Batch batch;
  Engine eng;
  double t_begin;
  double add_us = 0;
  bool finished = false;
  struct Deferred {
    at::Tensor fake;
    bool apply_shard;
    size_t ticket;
    int64_t shard_dim;
  };
  std::vector<Deferred> deferred;
  // this tensor's layout: the call's (rank, world) cut along `dim`, or none
  std::optional<ShardSpec> shard_for(bool apply_shard, int64_t dim) const {
    if (!apply_shard || !opts.shard) return std::nullopt;
    ShardSpec s = *opts.shard;
    s.dim = dim;
    return s;
  }
  std::function<void(size_t, at::Tensor)> sink;
  explicit Impl(const MaterializeOptions& o) : opts(o), eng{o, batch}, t_begin(now_us()) {}
};

void MaterializeSession::defer_generic_programs(std::function<void(size_t, at::Tensor)> sink) {
  impl_->sink = std::move(sink);
  impl_->eng.defer_generic = static_cast<bool>(impl_->sink);
}

MaterializeSession::MaterializeSession(const MaterializeOptions& opts) {
  g_stats = MaterializeStats{};
  g_stats.traverse_us = g_pending_traverse_us;
  g_pending_traverse_us = 0;
  g_last_descs.clear();
  impl_ = std::make_unique<Impl>(opts);
  g_call_begin_us = impl_->t_begin;
}

MaterializeSession::~MaterializeSession() {
  // also on error paths: tensors planned so far are part of the recording's state (a later call
  // returns them), so their descriptors must run; offsets already handed out must stay consumed
  if (impl_ && !impl_->finished) {
    try { impl_->batch.flush(); } catch (...) {}
    try { impl_->eng.gens.write_back(); } catch (...) {}
  }
}

at::Tensor MaterializeSession::add(const at::Tensor& t, bool apply_shard, size_t ticket, Prebuilt* pre, int64_t shard_dim) {
  g_stats.tensors++;
  if (!can_materialize(t)) return t;
  const double t0 = now_us();
  impl_->eng.opts.shard = impl_->shard_for(apply_shard, shard_dim);
  const TensorRecord* rec = fake_impl(t)->record().get();  // (`t` keeps its record, and the record the tape, alive while we work)
  at::Tensor value = impl_->eng.materialize_value(rec->tape, rec->value, pre);
  if (!value.defined()) {  // an unfusable program without RNG: replayed after the last submission (finish)
    impl_->deferred.push_back(Impl::Deferred{t, apply_shard, ticket, shard_dim});
    impl_->add_us += now_us() - t0;
    return at::Tensor();
  }
  at::Tensor out = finish_tensor(t, std::move(value));
  impl_->add_us += now_us() - t0;
  return out;
}

void MaterializeSession::finish() {
  const double t0 = now_us();
  impl_->batch.flush();
  impl_->eng.gens.write_back();
  // the deferred programs: the kernels of every fused tensor are on the stream by now
  const double t_deferred = now_us();
  impl_->eng.defer_generic = false;
  for (Impl::Deferred& d : impl_->deferred) {
    impl_->eng.opts.shard = impl_->shard_for(d.apply_shard, d.shard_dim);
    const auto rec = fake_impl(d.fake)->record();
    at::Tensor out = finish_tensor(d.fake, impl_->eng.materialize_value(rec->tape, rec->value));
    impl_->sink(d.ticket, std::move(out));
  }
  if (!impl_->deferred.empty()) {
    impl_->deferred.clear();
    impl_->batch.flush();  // (dependencies of the deferred programs that took the fused path)
    impl_->eng.gens.write_back();
  }
  g_stats.deferred_us = now_us() - t_deferred;
  impl_->finished = true;
  impl_->add_us += now_us() - t0;
  g_stats.plan_us = impl_->add_us - g_stats.launch_us;
  // whatever else happened between the first add() and now was the caller walking its modules
  g_stats.traverse_us += (now_us() - impl_->t_begin) - impl_->add_us;
}

std::vector<at::Tensor> materialize_many(const std::vector<at::Tensor>& fakes,
                                         const MaterializeOptions& opts,
                                         const std::vector<uint8_t>* shard_mask) {
  MaterializeSession session(opts);
  std::vector<at::Tensor> out(fakes.size());
  session.defer_generic_programs([&out](size_t i, at::Tensor t) { out[i] = std::move(t); });
  for (size_t i = 0; i < fakes.size(); ++i) {
    // (mask entry k > 0: shard along dim k - 1)
    const int64_t dim = shard_mask && (*shard_mask)[i] ? (*shard_mask)[i] - 1 : 0;
    at::Tensor t = session.add(fakes[i], !(shard_mask && !(*shard_mask)[i]), i, nullptr, dim);
    if (t.defined()) out[i] = std::move(t);
  }
  session.finish();
  return out;
}
std::vector<int64_t> submission_sizes(int64_t total_bytes, int64_t tensors, bool with_estimate) {
  Batch b;  // (Batch::note's cut, without the flush)
  std::vector<int64_t> out;
  if (tensors <= 0 || total_bytes <= 0) return out;
  if (with_estimate) b.expect(total_bytes, tensors);
  const int64_t each = total_bytes / tensors;
  int64_t pending = 0;
  for (int64_t i = 0; i < tensors; ++i) {
    pending += each;
    if (pending >= b.flush_threshold) {
      b.cut(pending);
      out.push_back(pending);
      pending = 0;
    }
  }
  if (pending) out.push_back(pending);
  return out;
}

void add_wrap_time(double us) { g_stats.wrap_us += us; }
// (materialize_many resets the counters: the traversal that precedes it is reported through a
// pending value that the next reset picks up)
void add_traverse_time(double us) { g_pending_traverse_us += us; }

at::Tensor materialize_flat_shard(const std::vector<at::Tensor>& fakes, const MaterializeOptions& opts, int64_t rank,
                                  int64_t world, int64_t align_numel, const std::optional<at::Tensor>& out,
                                  std::vector<int64_t>* offsets) {
  g_stats = MaterializeStats{};
  g_last_descs.clear();
  g_call_begin_us = now_us();
  Batch batch;
  Engine eng{opts, batch};
  at::Tensor result;
  try {
    result = eng.flat_shard(fakes, rank, world, align_numel, out, offsets);
  } catch (...) {
    try { batch.flush(); } catch (...) {}
    try { eng.gens.write_back(); } catch (...) {}
    throw;
  }
  eng.gens.write_back();
  g_stats.tensors = static_cast<int64_t>(fakes.size());
  return result;
}

at::Tensor materialize_one(const at::Tensor& fake, const MaterializeOptions& opts) {
  if (!can_materialize(fake)) return fake;
  return materialize_many({fake}, opts)[0];
}
std::pair<uint32_t, uint64_t> aten_stream_policy(int64_t numel, int sm, int tps) {
  const uint64_t blocks = (static_cast<uint64_t>(std::max<int64_t>(numel, 1)) + 255) / 256;
  const uint32_t S = 256u * static_cast<uint32_t>(std::min<uint64_t>(static_cast<uint64_t>(sm) * (tps / 256), blocks));
  return {S, numel > 0 ? aten_offset_increment(numel, S) : 0};
}

MaterializeStats last_stats() { return g_stats; }

std::string last_descriptors() {
  return std::string(reinterpret_cast<const char*>(g_last_descs.data()),
                     g_last_descs.size() * sizeof(TdxInitDesc));
}

at::Tensor cached_python_tensor(const at::Tensor& fake) {
  if (!can_materialize(fake)) return {};
  const auto& rec = fake_impl(fake)->record();
  return rec->tape->values[rec->value].py_wrapped;
}

void cache_python_tensor(const at::Tensor& fake, const at::Tensor& wrapped) {
  if (!can_materialize(fake)) return;
  const auto& rec = fake_impl(fake)->record();
  rec->tape->values[rec->value].py_wrapped = wrapped;
}

}  // namespace tdx
