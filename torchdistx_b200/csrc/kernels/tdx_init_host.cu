// libtdx_init.so, host side: validation, routing of descriptors to kernel families, the plan image,
// its upload and the launches -- and the C ABI (include/tdx_init.h).  No kernel is defined here: each
// kernel unit hands its kernels over as rows of the family table (tdx_device.cuh Family).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "tdx_device.cuh"

namespace tdx {

// launches of up to this many tiles per resident CTA are scheduled statically (GroupArgs::static_grabs)
constexpr unsigned long long kStaticTilesPerCta = 8;
// A launch uses the table kernel when it holds at least this many table-eligible elements: the
// table costs every CTA ~4 us.
constexpr uint64_t kLutMinLaunchElems = 1ull << 25;  // 64 MB of 16-bit output (normal; x2 for the uniform)
// the table kernel's largest work grab (the cap grows with the launch: build_plan)
constexpr unsigned long long kLutMaxGrabBytes = 1ull << 22;  // 4 MiB

// The rows of every kernel unit, joined on first use (each unit's rows are constant-initialised, so
// they are there before any dynamic initialisation runs).  Empty if two rows overlap: then some key
// would have two kernels and the routing would depend on row order.
bool overlap(const Family& a, const Family& b) {
  return a.src == b.src && (a.dtype == b.dtype || a.dtype == kAnyDtype || b.dtype == kAnyDtype) &&
         a.algo == b.algo && (a.epi & b.epi) && (a.range & b.range) && a.lut == b.lut;
}
const std::vector<Family>& families() {
  static const std::vector<Family> table = [] {
    std::vector<Family> t;
    for (const FamilyRows* u : {&kBaseFamilies, &kSsmFamilies, &kSincosFamilies, &kGatherFamilies, &kBandFamilies,
                                &kWindowFamilies, &kAtenFamilies})
      t.insert(t.end(), u->row, u->row + u->n);
    for (size_t a = 0; a < t.size(); ++a)
      for (size_t b = a + 1; b < t.size(); ++b)
        if (overlap(t[a], t[b])) {
          fprintf(stderr, "libtdx_init: kernel families %s and %s overlap\n", t[a].name, t[b].name);
          return std::vector<Family>();
        }
    return t;
  }();
  return table;
}

thread_local char g_err[256] = "";
thread_local int g_last_launches = 0;
thread_local size_t g_last_upload_bytes = 0;

int fail(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return code;
}
int cuda_fail(cudaError_t e, const char* where) {
  snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
  return static_cast<int>(e);
}

int itemsize_of(int dtype) {
  switch (dtype) {
    case TDX_F32: case TDX_RAW32: return 4;
    case TDX_BF16: case TDX_F16: case TDX_RAW16: return 2;
    case TDX_RAW8: return 1;
    case TDX_RAW64: case TDX_I64: return 8;
    default: return 0;
  }
}

bool is_aten(const TdxInitDesc& d) {
  const int a = d.algo & 0x0f;
  return a == TDX_ALGO_ATEN || a == TDX_ALGO_ATEN_WIDE;
}

int resolve_algo(const TdxInitDesc& d) {
  const int a = d.algo & 0x0f;
  // (a wide fp32 draw is the plain one; a 16-bit normal drawn on fp32 and rounded is the native one)
  if (is_aten(d)) return a == TDX_ALGO_ATEN_WIDE && d.src == TDX_SRC_UNIFORM && d.dtype != TDX_F32 ? a : TDX_ALGO_ATEN;
  if (d.src == TDX_SRC_NORMAL) {
    if (a != TDX_ALGO_DEFAULT) return a;
    return d.dtype == TDX_F32 ? TDX_ALGO_BM32 : TDX_ALGO_ICDF16;
  }
  if (d.src == TDX_SRC_UNIFORM && d.dtype != TDX_F32 && a == TDX_ALGO_WIDE32) return TDX_ALGO_WIDE32;
  return 0;
}

// Descriptors at least this large (two tiles) use the table kernel when their launch does.  The
// table is paid per CTA and per distinct parameter set, not per descriptor -- the host sorts a
// family's descriptors by parameters -- so the bound only keeps descriptors out whose tiles would
// mostly take the ragged path (a sharded k_proj of Llama-3-8B on 8 GPUs is 2^19 elements).
constexpr uint64_t kLutMinElems = 1ull << 18;

// Does the descriptor need the superset epilogue (a state-space step) or the broadcast index?
bool uses_ext(const TdxInitDesc& d) {
  if (d.src == TDX_SRC_IOTA && d.fill_bits[0] != 0) return true;
  for (int i = 0; i < d.n_epi && i < TDX_MAX_EPI; ++i) {
    const uint32_t op = d.epi[i].op & 0xffu;
    if (op >= TDX_EPI_EXP && op <= TDX_EPI_MULADD) return true;
  }
  return false;
}

// The key of a descriptor.
struct FamilyKey {
  int src, dtype, algo;
  uint8_t epi, range;  // one bit each
  bool lut;
};
bool matches(const Family& F, const FamilyKey& k) {
  return F.src == k.src && (F.dtype == kAnyDtype || F.dtype == k.dtype) && F.algo == k.algo && (F.epi & k.epi) &&
         (F.range & k.range) && F.lut == k.lut;
}
// The single row that matches (families() has no two that overlap), or -1.
int find_family(const FamilyKey& k) {
  const std::vector<Family>& F = families();
  for (size_t f = 0; f < F.size(); ++f)
    if (matches(F[f], k)) return static_cast<int>(f);
  return -1;
}

// The family whose kernel runs the descriptor: the table kernel for a large one if it has a row for
// the descriptor's key (`table`, and never a window: its work list walks plain ranges), the direct
// kernel otherwise.
int family_of(const TdxInitDesc& d, bool table = true) {
  const bool window = d.reserved & TDX_FLAG_WINDOW;
  FamilyKey k{d.src, d.dtype, resolve_algo(d), uses_ext(d) ? kEpiExt : d.n_epi ? kEpiBasic : kEpiNone,
              window ? kWindowed : kPlain, false};
  if (table && !window && !(d.algo & TDX_ALGO_NOLUT) && d.elem_count >= kLutMinElems) {
    k.lut = true;
    const int f = find_family(k);
    if (f >= 0) return f;
    k.lut = false;
  }
  return find_family(k);
}

uint64_t tiles_of(const TdxInitDesc& d, int tile_vecs) {
  if (d.elem_count == 0) return 0;
  uint64_t nvec;
  if (d.src == TDX_SRC_CONST || d.src == TDX_SRC_BAND) {  // the absolute 16-byte lines of the destination
    const uint64_t a = reinterpret_cast<uintptr_t>(d.dst);
    const uint64_t end = a + d.elem_count * itemsize_of(d.dtype);
    nvec = (end - (a & ~15ull) + 15) / 16;
  } else if (is_aten(d) && !(d.reserved & TDX_FLAG_WINDOW)) {
    // four vectors per work item (tdx_aten_kernel): the items of every k whose 4S elements meet the range
    const uint64_t S = d.fill_bits[1], epv = 16 / itemsize_of(d.dtype);
    nvec = 4 * ((d.elem_begin + d.elem_count - 1) / (4 * S) - d.elem_begin / (4 * S) + 1) * (S / epv);
  } else if (d.src == TDX_SRC_IOTA || d.src == TDX_SRC_SINCOS || d.src == TDX_SRC_GATHER ||
             (d.reserved & TDX_FLAG_WINDOW)) {  // vectors are counted from the descriptor's first element
    const uint64_t epv = 16 / itemsize_of(d.dtype);
    nvec = (d.elem_count + epv - 1) / epv;
  } else {
    const uint64_t epv = 16 / itemsize_of(d.dtype);
    nvec = (d.elem_begin + d.elem_count - 1) / epv - d.elem_begin / epv + 1;
  }
  return (nvec + tile_vecs - 1) / tile_vecs;
}

// Device-resident plan header.  Lives at the start of its plan image in the caller's workspace.
struct PlanGroup {
  unsigned long long total_tiles;
  unsigned long long prefix_off;  // byte offsets from the start of the plan image
  unsigned long long desc_off;
  uint32_t n_desc;
  uint32_t family;
  unsigned long long seed;  // seed of the group's descriptors if they all share one
  uint32_t seed_shared;
  uint32_t n_chunks;             // table kernel only: entries of the work list
  unsigned long long chunk_off;  // and its byte offset
  uint32_t n_static;             // leading entries that are pre-assigned to CTAs (GroupArgs::n_static)
  uint32_t list_ctas;            // ... to this many
  unsigned long long seg_off_off;  // byte offset of the [list_ctas + 1] segment table
};
struct PlanHeader {
  uint32_t magic;
  uint32_t n_groups;
  unsigned int counters[64];
  unsigned int done[64];
  // One per kernel family the plan uses -- a handful.  47 is what fits the 4 KiB TdxPlan
  // (static_assert in tdx_plan_upload: 520 + 47 * 72 + 128 <= 4096), fewer than there are families;
  // build_plan lays a submission that spans more out as consecutive plan images (kMaxGroups groups
  // each).  Adding a field to PlanGroup or PlanHeader means lowering this bound.
  PlanGroup groups[47];
  TdxInitDesc one;  // the plan's descriptor if it has exactly one (GroupArgs::one)
};
constexpr uint32_t kPlanMagic = 0x58445431u;  // "TDX1"
constexpr uint32_t kMaxGroups = sizeof(PlanHeader::groups) / sizeof(PlanGroup);
static_assert(kMaxGroups <= 64, "counter slots (one per group of a plan)");
// Plan images start on this boundary of the workspace (a descriptor table is 128-byte aligned).
constexpr size_t kImageAlign = 256;

// A prepared submission: one plan image per kMaxGroups kernel families, back to back in one workspace.
struct PlanSet {
  std::vector<PlanHeader> hdrs;
  std::vector<size_t> base;  // byte offset of each image (and its header) in the workspace
};

// Work list of the table kernel: at most kMaxListChunks "large" grabs (the grab cap grows with the
// launch so that this holds), a guided tail, and one partial grab per descriptor.
constexpr size_t kMaxListChunks = 8192;
constexpr size_t kMaxListTail = 4096;
constexpr size_t kMaxListCtas = 1024;  // segment table of the pre-assigned part (one entry per CTA + 1)
size_t lut_family_count() {
  static const size_t v = [] {
    size_t c = 0;
    for (const Family& F : families()) c += F.lut ? 1 : 0;
    return c;
  }();
  return v;
}
size_t plan_bytes(int n) {
  const size_t families_n = families().size();
  const size_t images = (families_n + kMaxGroups - 1) / kMaxGroups;
  // one header per image (and its alignment) + per-family prefix arrays (n + #families entries worst
  // case) + descriptors + one work list per table family (each at most kMaxListChunks + kMaxListTail
  // grabs plus one per descriptor)
  return images * (sizeof(PlanHeader) + kImageAlign) + (static_cast<size_t>(n) + families_n) * sizeof(unsigned long long) +
         static_cast<size_t>(n) * sizeof(TdxInitDesc) +
         (lut_family_count() * (kMaxListChunks + kMaxListTail) + static_cast<size_t>(n)) * sizeof(uint4) +
         lut_family_count() * kMaxListCtas * sizeof(uint32_t) +
         (32 + 128) * families_n + 64;
}

struct DeviceInfo {
  int sm_count = 0;
  std::vector<int> blocks_per_sm;  // per family
};
DeviceInfo* device_info() {
  static DeviceInfo infos[64];
  static bool ready[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  if (!ready[dev]) {
    DeviceInfo& I = infos[dev];
    if (cudaDeviceGetAttribute(&I.sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      return nullptr;
    I.blocks_per_sm.clear();
    for (const Family& F : families()) {
      int nb = 0;
      if (F.dyn_smem &&
          cudaFuncSetAttribute(reinterpret_cast<const void*>(F.fn), cudaFuncAttributeMaxDynamicSharedMemorySize,
                               F.dyn_smem) != cudaSuccess)
        return nullptr;
      if (F.dyn_smem && F.fn_any_seed &&
          cudaFuncSetAttribute(reinterpret_cast<const void*>(F.fn_any_seed),
                               cudaFuncAttributeMaxDynamicSharedMemorySize, F.dyn_smem) != cudaSuccess)
        return nullptr;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, reinterpret_cast<const void*>(F.fn), F.threads,
                                                        F.dyn_smem) != cudaSuccess)
        return nullptr;
      I.blocks_per_sm.push_back(std::max(nb, 1));
    }
    ready[dev] = true;
  }
  return &infos[dev];
}

// Builds the host image of the plan: one plan image per kMaxGroups kernel families, each with its own
// header, work counters and offsets counted from its own start.  Routing (table or direct kernel,
// riders) is decided over the whole table first, so a table that spans several images runs the
// kernels it would run in one.  Returns 0 or an error code.
// `img` is scratch that only grows (zero-filling 1.6 MB per call would cost more host time than the
// planning of a small module); `used` = bytes of the image to copy to the device.
int build_plan(const TdxInitDesc* descs, int n, std::vector<unsigned char>& img, PlanSet& plans, size_t& used) {
  if (n < 0 || (n > 0 && descs == nullptr)) return fail(TDX_E_BADARG, "descs == NULL or n < 0");
  const std::vector<Family>& F = families();
  if (F.empty()) return fail(TDX_E_BADARG, "internal: two kernel families overlap (see stderr)");
  const int nf = static_cast<int>(F.size());
  std::vector<int> fam(static_cast<size_t>(n)), per_family(F.size());
  for (int i = 0; i < n; ++i) {
    const TdxInitDesc& d = descs[i];
    const int isz = itemsize_of(d.dtype);
    if (isz == 0) return fail(TDX_E_BADARG, "unknown dtype");
    if (d.src == TDX_SRC_BAND) {  // (every width: only the element size matters)
      const uint64_t C = d.fill_bits[0] & 0xffffffffull, R = d.fill_bits[0] >> 32;
      const int32_t lo = static_cast<int32_t>(static_cast<uint32_t>(d.fill_bits[1]));
      const int32_t hi = static_cast<int32_t>(static_cast<uint32_t>(d.fill_bits[1] >> 32));
      if (C == 0 || R == 0 || C >= (1ull << 31) || R >= (1ull << 31))
        return fail(TDX_E_BADARG, "TDX_SRC_BAND: fill_bits[0] must be C | R << 32 with 0 < C, R < 2^31");
      if (lo > hi) return fail(TDX_E_BADARG, "TDX_SRC_BAND: lo > hi");
      if (d.n_epi != 0) return fail(TDX_E_BADARG, "TDX_SRC_BAND takes no epilogue");
      if (d.algo != 0 || d.reserved != 0)
        return fail(TDX_E_BADARG, "TDX_SRC_BAND: unknown flag bit (algo / reserved must be 0)");
    }
    if (d.src != TDX_SRC_CONST && d.src != TDX_SRC_BAND && d.dtype >= TDX_RAW8)
      return fail(TDX_E_BADARG, "raw dtypes are only valid with TDX_SRC_CONST and TDX_SRC_BAND");
    if (d.src == TDX_SRC_GATHER) {
      const uint64_t period = d.fill_bits[1] & 0xffffffffull, rep = d.fill_bits[1] >> 32;
      if (!(d.dtype == TDX_F32 || d.dtype == TDX_BF16 || d.dtype == TDX_F16 || (d.dtype == TDX_I64 && d.n_epi == 0)))
        return fail(TDX_E_BADARG, "TDX_SRC_GATHER writes TDX_F32 / TDX_BF16 / TDX_F16 (epilogue allowed) or TDX_I64 (none)");
      if (d.fill_bits[0] == 0) return fail(TDX_E_BADARG, "TDX_SRC_GATHER: source == NULL");
      if (d.fill_bits[0] % isz) return fail(TDX_E_BADARG, "TDX_SRC_GATHER: source not element-aligned");
      if (d.algo != 0 || d.reserved != 0 || (period == 0 && rep != 0))
        return fail(TDX_E_BADARG, "TDX_SRC_GATHER: unknown flag bit (algo / reserved must be 0; R only with P)");
    }
    if ((d.dtype == TDX_I64 && d.src != TDX_SRC_IOTA && d.src != TDX_SRC_GATHER && d.src != TDX_SRC_BAND) ||
        (d.src == TDX_SRC_IOTA && !(d.dtype == TDX_F32 || d.dtype == TDX_BF16 || d.dtype == TDX_F16 || (d.dtype == TDX_I64 && d.n_epi == 0))))
      return fail(TDX_E_BADARG, "TDX_SRC_IOTA writes TDX_F32 / TDX_BF16 / TDX_F16 (epilogue allowed) or TDX_I64 (none); TDX_I64 is IOTA-only");
    if (d.src == TDX_SRC_SINCOS) {
      const uint64_t half = d.fill_bits[0];
      if (!(d.dtype == TDX_F32 || d.dtype == TDX_BF16 || d.dtype == TDX_F16))
        return fail(TDX_E_BADARG, "TDX_SRC_SINCOS writes TDX_F32 / TDX_BF16 / TDX_F16");
      if (half == 0 || half > (1ull << 40) || (d.fill_bits[1] & ~static_cast<uint64_t>(TDX_SINCOS_COS_FIRST)))
        return fail(TDX_E_BADARG, "TDX_SRC_SINCOS: fill_bits must be {H > 0, order bit}");
      if (d.elem_count && (d.elem_begin + d.elem_count - 1) / (2 * half) >= (1ull << 24))
        return fail(TDX_E_BADARG, "TDX_SRC_SINCOS: rows must stay below 2^24 (float(r) exact)");
    }
    if (is_aten(d)) {
      const uint64_t S = d.fill_bits[1];
      if ((d.src != TDX_SRC_UNIFORM && d.src != TDX_SRC_NORMAL) ||
          !(d.dtype == TDX_F32 || d.dtype == TDX_BF16 || d.dtype == TDX_F16))
        return fail(TDX_E_BADARG, "TDX_ALGO_ATEN(_WIDE) is valid with TDX_SRC_UNIFORM / TDX_SRC_NORMAL in TDX_F32 / TDX_BF16 / TDX_F16 only");
      if (d.algo & TDX_ALGO_NOLUT) return fail(TDX_E_BADARG, "TDX_ALGO_ATEN(_WIDE) takes no TDX_ALGO_NOLUT");
      if (S == 0 || S % 256 || S >= (1ull << 31))
        return fail(TDX_E_BADARG, "TDX_ALGO_ATEN: fill_bits[1] must be the grid stride S, a multiple of 256 below 2^31");
      if (d.philox_offset % 4) return fail(TDX_E_BADARG, "TDX_ALGO_ATEN: philox_offset must be a multiple of 4");
      if (d.elem_count) {  // the last global element must stay below 2^31 (ATen's 32-bit iterator)
        uint64_t last = ~0ull;
        const uint64_t n = d.elem_count - 1;
        if (d.reserved & TDX_FLAG_WINDOW) {
          const uint64_t width = d.fill_bits[0] & 0xffffffffull, pitch = d.fill_bits[0] >> 32;
          if (width == 0 || pitch < width)
            return fail(TDX_E_BADARG, "TDX_FLAG_WINDOW: fill_bits[0] must be W | P << 32 with W > 0, P >= W");
          if (n / width < (1ull << 31) && d.elem_begin < (1ull << 31)) last = d.elem_begin + (n / width) * pitch + n % width;
        } else if (n < (1ull << 31) && d.elem_begin < (1ull << 31)) {
          last = d.elem_begin + n;
        }
        if (last >= (1ull << 31)) return fail(TDX_E_BADARG, "TDX_ALGO_ATEN: the last element must be below 2^31");
      }
    } else if (d.reserved & TDX_FLAG_WINDOW) {
      const uint64_t width = d.fill_bits[0], pitch = d.fill_bits[1];
      if (d.src != TDX_SRC_UNIFORM && d.src != TDX_SRC_NORMAL)
        return fail(TDX_E_BADARG, "TDX_FLAG_WINDOW is valid with TDX_SRC_UNIFORM / TDX_SRC_NORMAL only");
      if (width == 0 || pitch < width) return fail(TDX_E_BADARG, "TDX_FLAG_WINDOW: fill_bits must be {W > 0, P >= W}");
      if (d.elem_count) {  // the last element, elem_begin + ((n - 1) / W) * P + (n - 1) % W, must not wrap
        const uint64_t runs = (d.elem_count - 1) / width, rest = (d.elem_count - 1) % width;
        if (d.elem_begin > ~0ull - rest || runs > (~0ull - d.elem_begin - rest) / pitch)
          return fail(TDX_E_BADARG, "TDX_FLAG_WINDOW: the window's last element overflows");
      }
    }
    if (d.n_epi > TDX_MAX_EPI) return fail(TDX_E_BADARG, "n_epi > TDX_MAX_EPI");
    if (d.algo & ~(0x0f | TDX_ALGO_NOLUT)) return fail(TDX_E_BADARG, "unknown algo flag");
    if (d.elem_count && d.dst == nullptr) return fail(TDX_E_BADARG, "dst == NULL");
    if (reinterpret_cast<uintptr_t>(d.dst) % isz) return fail(TDX_E_BADARG, "dst not element-aligned");
    fam[i] = family_of(d);
    if (fam[i] < 0) return fail(TDX_E_BADARG, "no kernel for (src, dtype, algo, epilogue)");
    per_family[fam[i]]++;
  }
  // The table kernel pays 65536 evaluations per CTA up front: worth it only if the launch as a
  // whole has enough table-eligible work.  Otherwise its descriptors go to the direct twin
  // (same bits either way).
  {
    std::vector<uint64_t> lut_elems(F.size());
    for (int i = 0; i < n; ++i)
      if (F[fam[i]].lut) lut_elems[fam[i]] += descs[i].elem_count;
    for (int i = 0; i < n; ++i) {
      const int f = fam[i];
      // break-even: ~64 MB for the normal, whose direct kernel is the slowest, ~128 MB for the uniform
      const uint64_t need = kLutMinLaunchElems * (F[f].src == TDX_SRC_UNIFORM ? 2 : 1);
      if (!F[f].lut || lut_elems[f] >= need) continue;
      const int twin = family_of(descs[i], /*table=*/false);
      if (twin < 0) continue;
      fam[i] = twin;
      per_family[f]--;
      per_family[twin]++;
    }
  }
  // A module's constant fills (norm weights, biases: KBs) and index programs ride in the largest
  // table launch's work list instead of costing a launch of their own -- unless they are a real share
  // of the bytes.
  {
    const int fill_family = find_family({TDX_SRC_CONST, TDX_F32, 0, kEpiNone, kPlain, false});
    const int iota_family = find_family({TDX_SRC_IOTA, TDX_F32, 0, kEpiNone, kPlain, false});
    const auto rides = [&](int f) { return f == fill_family || f == iota_family; };
    int riders = 0, host = -1;
    uint64_t ride_bytes = 0, host_bytes = 0;
    std::vector<uint64_t> bytes_of(F.size());
    for (int i = 0; i < n; ++i) {
      const uint64_t bytes = descs[i].elem_count * itemsize_of(descs[i].dtype);
      bytes_of[fam[i]] += bytes;
      if (rides(fam[i])) {
        ++riders;
        ride_bytes += bytes;
      }
    }
    for (int f = 0; f < nf; ++f)
      if (F[f].lut && per_family[f] > 0 && bytes_of[f] > host_bytes) {
        host = f;
        host_bytes = bytes_of[f];
      }
    if (riders && host >= 0 && ride_bytes * 16 <= host_bytes) {
      for (int i = 0; i < n; ++i)
        if (rides(fam[i])) {
          per_family[fam[i]]--;
          fam[i] = host;
          per_family[host]++;
        }
    }
  }
  plans.hdrs.clear();
  plans.base.clear();
  PlanHeader hdr;
  memset(&hdr, 0, sizeof(hdr));
  hdr.magic = kPlanMagic;
  if (img.size() < plan_bytes(n)) img.resize(plan_bytes(n));
  int sm_count = 132;  // (H100 SXM; the device's own count when it can be queried)
  if (DeviceInfo* info = device_info()) sm_count = info->sm_count;
  std::vector<int> order;
  thread_local std::vector<uint32_t> seg_fill;
  order.reserve(static_cast<size_t>(n));
  const size_t hdr_end = (sizeof(PlanHeader) + 15) & ~static_cast<size_t>(15);
  size_t start = 0, off = hdr_end;  // the current image's offset in the workspace; `off` counts from it
  unsigned char* image = img.data();
  for (int f = 0; f < nf; ++f) {
    if (!per_family[f]) continue;
    if (hdr.n_groups == kMaxGroups) {  // this image is full: the next family opens another
      memcpy(image, &hdr, sizeof(hdr));
      plans.hdrs.push_back(hdr);
      plans.base.push_back(start);
      start = (start + off + kImageAlign - 1) & ~(kImageAlign - 1);
      image = img.data() + start;
      off = hdr_end;
      memset(&hdr, 0, sizeof(hdr));
      hdr.magic = kPlanMagic;
    }
    PlanGroup& G = hdr.groups[hdr.n_groups++];
    G.family = f;
    G.n_desc = per_family[f];
    // (8-byte prefix sums: the table kernel's segment table before this group ends on a 4-byte boundary)
    off = (off + 15) & ~static_cast<size_t>(15);
    G.prefix_off = off;
    auto* prefix = reinterpret_cast<unsigned long long*>(image + off);
    off += (static_cast<size_t>(G.n_desc) + 1) * sizeof(unsigned long long);
    off = (off + 127) & ~static_cast<size_t>(127);  // (a descriptor = one cache line: lut_prefetch_desc)
    G.desc_off = off;
    auto* out = reinterpret_cast<TdxInitDesc*>(image + off);
    off += static_cast<size_t>(G.n_desc) * sizeof(TdxInitDesc);
    unsigned long long acc = 0;
    uint32_t k = 0;
    G.seed_shared = 1;
    // Table kernel: a CTA rebuilds its 65536-entry table (~10 us) whenever the parameters change
    // from one grab to the next, so descriptors with equal parameters are made neighbours (GPT-2's
    // alternating std 0.02 / 0.02/sqrt(2L) would otherwise cost a rebuild per tensor).  The order
    // inside a family is free: every descriptor is self-contained.
    order.clear();
    for (int i = 0; i < n; ++i)
      if (fam[i] == f) order.push_back(i);
    if (F[f].lut)
      std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        const TdxInitDesc &x = descs[a], &y = descs[b];
        const bool xr = x.src != TDX_SRC_CONST && x.src != TDX_SRC_IOTA, yr = y.src != TDX_SRC_CONST && y.src != TDX_SRC_IOTA;
        if (xr != yr) return yr;  // (folded fills and index programs first)
        if (!xr) return false;
        if (x.p0 != y.p0) return x.p0 < y.p0;
        if (x.p1 != y.p1) return x.p1 < y.p1;
        if (x.n_epi != y.n_epi) return x.n_epi < y.n_epi;
        return x.n_epi != 0 && memcmp(x.epi, y.epi, sizeof(TdxEpiStep) * x.n_epi) < 0;
      });
    bool have_seed = false;
    for (int i : order) {
      if (descs[i].src != TDX_SRC_CONST && descs[i].src != TDX_SRC_IOTA) {
        if (!have_seed) G.seed = descs[i].philox_seed;
        else if (descs[i].philox_seed != G.seed) G.seed_shared = 0;
        have_seed = true;
      }
      prefix[k] = acc;
      out[k] = descs[i];
      // (an image of one group of one descriptor launches it inline: the last image of a split table
      // can be one even when the table is not)
      if (G.n_desc == 1) hdr.one = descs[i];
      acc += tiles_of(descs[i], F[f].tile_vecs);
      ++k;
    }
    prefix[k] = acc;
    G.total_tiles = acc;
    if (F[f].lut) {
      // Work list of the table kernel (for_each_listed_chunk).  Head: everything but four tiles per
      // CTA of tail (two leave the CTAs far apart at the end of a large launch, eight cost more grabs
      // than they buy balance) is cut into one
      // contiguous, equal share per CTA -- a share is a few grabs, broken only where a descriptor
      // ends -- and CTA b owns entries [seg[b], seg[b + 1]).  Tail: guided sizes handed out by the
      // work counter (grab = remaining / (2 * CTAs), between one tile and the cap), which is what
      // lets the CTAs finish together whatever their speeds were.  Fewer grabs matter: a grab ends
      // in a barrier that re-aligns the warps of a CTA, and the lock-step phase that follows
      // costs throughput.  Small launches (fewer than 16 tiles per CTA) are all tail.
      off = (off + 15) & ~static_cast<size_t>(15);
      G.chunk_off = off;
      auto* list = reinterpret_cast<uint4*>(image + off);
      const unsigned long long ctas = static_cast<unsigned long long>(std::max(sm_count, 1));
      const unsigned long long cap =
          std::max<unsigned long long>(kLutMaxGrabBytes / (F[f].tile_vecs * 16ull), (acc + kMaxListChunks - 1) / kMaxListChunks);
      unsigned long long static_tiles = 0;
      if (ctas < kMaxListCtas && acc >= ctas * 16ull) static_tiles = acc - ctas * 4ull;
      seg_fill.assign(static_cast<size_t>(ctas) + 1, 0u);  // seg_fill[b] = first entry of CTA b
      unsigned long long remaining = acc;
      uint32_t nc = 0, cta = 0;
      unsigned long long room = static_tiles / ctas + (0 < static_tiles % ctas ? 1 : 0);  // CTA 0's share
      for (uint32_t di = 0; di < G.n_desc; ++di) {
        unsigned long long t = 0;
        const unsigned long long nt = prefix[di + 1] - prefix[di];
        while (t < nt) {
          unsigned long long sz;
          if (cta < ctas && static_tiles) {  // pre-assigned part
            sz = std::min<unsigned long long>(std::min(nt - t, room), 0xffffffffull);
          } else {
            sz = std::min(std::min(std::max(remaining / (2ull * ctas), 1ull), cap), nt - t);
          }
          if (start + off + (static_cast<size_t>(nc) + 1) * sizeof(uint4) > img.size())
            return fail(TDX_E_WORKSPACE, "internal: work list exceeds its bound");
          list[nc++] = make_uint4(di, static_cast<uint32_t>(sz), static_cast<uint32_t>(t),
                                  static_cast<uint32_t>(t >> 32));
          t += sz;
          remaining -= sz;
          if (cta < ctas && static_tiles) {
            room -= sz;
            if (room == 0) {
              ++cta;
              seg_fill[cta] = nc;
              room = static_tiles / ctas + (cta < static_tiles % ctas ? 1 : 0);
            }
          }
        }
      }
      G.n_chunks = nc;
      off += static_cast<size_t>(nc) * sizeof(uint4);
      G.n_static = 0;
      G.list_ctas = static_cast<uint32_t>(ctas);
      G.seg_off_off = off;
      if (static_tiles && cta == ctas) {
        if (start + off + (static_cast<size_t>(ctas) + 1) * sizeof(uint32_t) > img.size())
          return fail(TDX_E_WORKSPACE, "internal: segment table exceeds its bound");
        memcpy(image + off, seg_fill.data(), (static_cast<size_t>(ctas) + 1) * sizeof(uint32_t));
        G.n_static = seg_fill[ctas];
        off += (static_cast<size_t>(ctas) + 1) * sizeof(uint32_t);
      }
    }
  }
  memcpy(image, &hdr, sizeof(hdr));
  plans.hdrs.push_back(hdr);
  plans.base.push_back(start);
  used = start + off;
  return 0;
}

// ---- pinned staging ring for plan uploads ------------------------------------------------------
struct StageSlot {
  void* host = nullptr;
  size_t cap = 0;
  cudaEvent_t done = nullptr;
  int device = -1;
  bool pending = false;
};
constexpr int kStageSlots = 8;
thread_local StageSlot g_stage[kStageSlots];
thread_local int g_stage_pos = 0;

int stage(const void* src, size_t bytes, cudaStream_t stream, void* dst_device, void** pinned_out) {
  StageSlot& s = g_stage[g_stage_pos];
  g_stage_pos = (g_stage_pos + 1) % kStageSlots;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
  if (s.pending) {  // the copy that last used this slot must have left it
    e = cudaEventSynchronize(s.done);
    if (e != cudaSuccess) return cuda_fail(e, "cudaEventSynchronize(staging)");
    s.pending = false;
  }
  if (s.done == nullptr || s.device != dev) {
    if (s.done) cudaEventDestroy(s.done);
    e = cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming);
    if (e != cudaSuccess) return cuda_fail(e, "cudaEventCreate(staging)");
    s.device = dev;
  }
  if (s.cap < bytes) {
    if (s.host) cudaFreeHost(s.host);
    s.cap = std::max<size_t>(bytes * 2, 64 << 10);
    e = cudaHostAlloc(&s.host, s.cap, cudaHostAllocPortable);
    if (e != cudaSuccess) { s.host = nullptr; s.cap = 0; return cuda_fail(e, "cudaHostAlloc(staging)"); }
  }
  memcpy(s.host, src, bytes);
  e = cudaMemcpyAsync(dst_device, s.host, bytes, cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) return cuda_fail(e, "cudaMemcpyAsync(plan)");
  e = cudaEventRecord(s.done, stream);
  if (e != cudaSuccess) return cuda_fail(e, "cudaEventRecord(staging)");
  s.pending = true;
  *pinned_out = s.host;
  return 0;
}

// Launches the groups of one plan image whose device copy starts at `image`; adds them to `launches`.
int launch_groups(const PlanHeader& hdr, void* image, cudaStream_t stream, int& launches) {
  DeviceInfo* info = device_info();
  if (!info) return fail(TDX_E_NODEVICE, "no CUDA device / occupancy query failed");
  auto* base = static_cast<unsigned char*>(image);
  auto* dev_hdr = reinterpret_cast<PlanHeader*>(base);
  for (uint32_t gi = 0; gi < hdr.n_groups; ++gi) {
    const PlanGroup& G = hdr.groups[gi];
    if (G.total_tiles == 0) continue;
    const Family& F = families()[G.family];
    GroupArgs a;
    a.tile_prefix = reinterpret_cast<const unsigned long long*>(base + G.prefix_off);
    a.descs = reinterpret_cast<const TdxInitDesc*>(base + G.desc_off);
    a.total_tiles = G.total_tiles;
    a.counter = &dev_hdr->counters[gi];  // zero: uploaded so, and put back by the kernel (leave_grid)
    a.done = &dev_hdr->done[gi];
    a.n_desc = G.n_desc;
    a.inline_desc = (hdr.n_groups == 1 && G.n_desc == 1) ? 1u : 0u;  // (hdr.one is set for one-descriptor plans)
    a.one = hdr.one;
    a.seed_shared = G.seed_shared;
    {
      uint32_t k0 = static_cast<uint32_t>(G.seed), k1 = static_cast<uint32_t>(G.seed >> 32);
      for (int r = 0; r < 10; ++r) {
        a.rk[2 * r] = k0;
        a.rk[2 * r + 1] = k1;
        k0 += kPhiloxW0;
        k1 += kPhiloxW1;
      }
    }
    const unsigned long long resident =
        static_cast<unsigned long long>(info->sm_count) * info->blocks_per_sm[G.family];
    // 256-thread kernels: full-size grabs only when every resident CTA still gets a few of them
    int tpc = F.tiles_per_chunk;
    a.static_grabs = 0;
    if (!F.lut) {
      if (G.total_tiles <= resident * kStaticTilesPerCta) {
        // small launch: one grab of consecutive tiles per CTA, assigned by block index
        tpc = static_cast<int>((G.total_tiles + resident - 1) / resident);
        a.static_grabs = 1;
      } else {
        const unsigned long long want = G.total_tiles / (resident * 2ull);
        tpc = static_cast<int>(std::min<unsigned long long>(std::max<unsigned long long>(want, 1ull), tpc));
      }
    }
    a.tiles_per_chunk = static_cast<uint32_t>(tpc);
    a.n_chunks = G.n_chunks;
    a.chunks = reinterpret_cast<const uint4*>(base + G.chunk_off);
    a.n_static = G.n_static;
    a.seg_off = reinterpret_cast<const uint32_t*>(base + G.seg_off_off);
    const unsigned long long chunks = F.lut ? G.n_chunks : (G.total_tiles + tpc - 1) / tpc;
    const unsigned int grid = static_cast<unsigned int>(std::min(chunks, resident));
    if (G.n_static && grid != G.list_ctas) return fail(TDX_E_BADARG, "internal: work list was cut for another grid");
    const KernelFn fn = (F.fn_any_seed && !G.seed_shared) ? F.fn_any_seed : F.fn;
    fn<<<grid, F.threads, F.dyn_smem, stream>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, F.name);
    ++launches;
  }
  return 0;
}

// ---- host destinations: the cut into staged passes (tdx_init_submit_host) ----------------------------

thread_local int g_last_host_copies = 0;

bool windowed(const TdxInitDesc& d) { return d.reserved & TDX_FLAG_WINDOW; }
uint64_t window_width(const TdxInitDesc& d) { return is_aten(d) ? d.fill_bits[0] & 0xffffffffull : d.fill_bits[0]; }
uint64_t window_pitch(const TdxInitDesc& d) { return is_aten(d) ? d.fill_bits[0] >> 32 : d.fill_bits[1]; }

// The descriptor of global elements [begin, begin + count) of `d`'s tensor as one plain range.
TdxInitDesc plain_part(const TdxInitDesc& d, uint64_t begin, uint64_t count, void* dst) {
  TdxInitDesc p = d;
  p.dst = dst;
  p.elem_begin = begin;
  p.elem_count = count;
  if (windowed(d)) {
    p.reserved &= ~TDX_FLAG_WINDOW;
    p.fill_bits[0] = 0;  // (ATen's stream keeps its grid stride in fill_bits[1])
    if (!is_aten(d)) p.fill_bits[1] = 0;
  }
  return p;
}

// The descriptors that write local elements [first, first + count) of `d` at `dst`: one for a plain
// descriptor; for a window a partial first run, the whole runs and a partial last run, as the planner
// emits a window (planner_engine.cc emit_window).
int piece_descs(const TdxInitDesc& d, uint64_t first, uint64_t count, unsigned char* dst, TdxInitDesc out[3]) {
  const uint64_t isz = itemsize_of(d.dtype);
  if (!windowed(d)) {
    out[0] = plain_part(d, d.elem_begin + first, count, dst);
    return 1;
  }
  const uint64_t W = window_width(d), P = window_pitch(d);
  int k = 0;
  uint64_t a = first;
  const uint64_t b = first + count;
  auto global = [&](uint64_t l) { return d.elem_begin + (l / W) * P + l % W; };
  if (a % W) {
    const uint64_t c = std::min(W - a % W, b - a);
    out[k++] = plain_part(d, global(a), c, dst + (a - first) * isz);
    a += c;
  }
  const uint64_t runs = (b - a) / W;
  if (runs > 1) {
    out[k] = d;
    out[k].dst = dst + (a - first) * isz;
    out[k].elem_begin = global(a);
    out[k++].elem_count = runs * W;
    a += runs * W;
  } else if (runs == 1) {
    out[k++] = plain_part(d, global(a), W, dst + (a - first) * isz);
    a += W;
  }
  if (a < b) out[k++] = plain_part(d, global(a), b - a, dst + (a - first) * isz);
  return k;
}

// The table family that would take a plain range of `d` if it were large enough (-1: none): such a piece
// needs room for the table kernel's work list in its pass's workspace.
int table_family_of(const TdxInitDesc& d) {
  if (d.algo & TDX_ALGO_NOLUT) return -1;
  const TdxInitDesc p = plain_part(d, d.elem_begin, kLutMinElems, d.dst);
  const int f = family_of(p);
  return f >= 0 && families()[f].lut ? f : -1;
}

// Bytes of workspace build_plan can use for a pass of `n` descriptors of which those of `tables`
// distinct table families may take the table kernel: the same terms as plan_bytes, counted for this
// pass (groups <= descriptors) instead of for the largest table.
size_t pass_workspace_bytes(size_t n, size_t tables) {
  const size_t groups = std::min(n, families().size());
  const size_t images = (groups + kMaxGroups - 1) / kMaxGroups;
  return images * (sizeof(PlanHeader) + kImageAlign) + groups * (sizeof(unsigned long long) + 15 + 127) +
         n * (sizeof(unsigned long long) + sizeof(TdxInitDesc) + sizeof(uint4)) +
         tables * ((kMaxListChunks + kMaxListTail) * sizeof(uint4) + 15 + (kMaxListCtas + 1) * sizeof(uint32_t));
}

// The cut of a table for a staging buffer of `staging_bytes` (see tdx_init_submit_host).  A pass's
// plan workspace sits at the head of the buffer; its pieces are placed from the end down, each at the
// highest offset that keeps its destination's address mod 16, until the next one would reach into the
// workspace the pass needs with it.
int host_cut(const TdxInitDesc* descs, int n, size_t staging_bytes, std::vector<TdxHostPiece>& pieces,
             int& passes) {
  pieces.clear();
  passes = 0;
  // (one vector at any address mod 16 above the workspace of a one-descriptor pass)
  if (staging_bytes < pass_workspace_bytes(1, 0) + 32)
    return fail(TDX_E_BADARG, "staging buffer smaller than one vector plus a one-descriptor pass's workspace");
  size_t top = staging_bytes, in_pass = 0;  // lowest staging byte used by the pass; its descriptors
  std::vector<int> tables;                  // table families the pass has room for
  bool open = false;
  for (int i = 0; i < n; ++i) {
    const TdxInitDesc& d = descs[i];
    const uint64_t isz = itemsize_of(d.dtype);
    const int table = table_family_of(d);
    uint64_t l = 0;
    while (l < d.elem_count) {
      if (!open) {
        top = staging_bytes;
        in_pass = 0;
        tables.clear();
        open = true;
        ++passes;
      }
      const uint64_t m = (reinterpret_cast<uintptr_t>(d.dst) + l * isz) % 16, rest = d.elem_count - l;
      // elements that fit above a workspace of `ws` bytes, at an offset congruent to m
      auto fit = [&](size_t ws) -> uint64_t {
        const size_t base = ((ws + 15 - m) & ~static_cast<size_t>(15)) + m;
        return base < top ? (top - base) / isz : 0;
      };
      const bool have_table = table >= 0 && std::find(tables.begin(), tables.end(), table) != tables.end();
      // a piece of a window can be three descriptors; one run's part of it is one
      uint64_t c = fit(pass_workspace_bytes(in_pass + (windowed(d) ? 3 : 1), tables.size()));
      int nd = windowed(d) ? 3 : 1;
      if (c == 0 && windowed(d)) {
        c = std::min(fit(pass_workspace_bytes(in_pass + 1, tables.size())), window_width(d) - l % window_width(d));
        nd = 1;
      }
      c = std::min(c, rest);
      bool add_table = false;
      if (table >= 0 && !have_table && c >= kLutMinElems) {  // large enough for the table kernel
        const uint64_t t = std::min<uint64_t>(fit(pass_workspace_bytes(in_pass + nd, tables.size() + 1)), rest);
        if (t >= kLutMinElems) {
          c = t;
          add_table = true;
        } else {
          c = kLutMinElems - 1;
        }
      }
      if (c == 0) {
        if (in_pass == 0) return fail(TDX_E_BADARG, "internal: a pass has no room for one element");
        open = false;  // the next pass takes it
        continue;
      }
      if (add_table) tables.push_back(table);
      const size_t off = ((top - c * isz - m) & ~static_cast<size_t>(15)) + m;
      pieces.push_back(TdxHostPiece{i, passes - 1, l, c, off});
      top = off;
      in_pass += nd;
      l += c;
    }
  }
  return 0;
}

}  // namespace tdx

extern "C" {

TDX_C_API size_t tdx_init_workspace_bytes(int n) { return tdx::plan_bytes(n < 0 ? 0 : n); }

TDX_C_API int tdx_init_host_cut(const TdxInitDesc* descs, int n, size_t staging_bytes, TdxHostPiece* pieces,
                                int max_pieces, int* n_pieces, int* n_passes) {
  if (n_pieces == nullptr || n_passes == nullptr) return tdx::fail(TDX_E_BADARG, "n_pieces / n_passes == NULL");
  {
    thread_local std::vector<unsigned char> img;
    thread_local tdx::PlanSet plans;
    size_t used = 0;
    if (int rc = tdx::build_plan(descs, n, img, plans, used)) return rc;
  }
  std::vector<TdxHostPiece> cut;
  int passes = 0;
  if (int rc = tdx::host_cut(descs, n, staging_bytes, cut, passes)) return rc;
  if (pieces)
    memcpy(pieces, cut.data(), std::min<size_t>(cut.size(), max_pieces < 0 ? 0 : max_pieces) * sizeof(TdxHostPiece));
  *n_pieces = static_cast<int>(cut.size());
  *n_passes = passes;
  return 0;
}

TDX_C_API int tdx_init_host_piece_descs(const TdxInitDesc* d, const TdxHostPiece* piece, void* staging,
                                        TdxInitDesc out[3]) {
  if (d == nullptr || piece == nullptr || out == nullptr) return tdx::fail(TDX_E_BADARG, "NULL argument");
  if (tdx::itemsize_of(d->dtype) == 0) return tdx::fail(TDX_E_BADARG, "unknown dtype");
  if (piece->elem_count == 0 || piece->elem_first + piece->elem_count > d->elem_count)
    return tdx::fail(TDX_E_BADARG, "the piece is not inside its descriptor");
  if (tdx::windowed(*d) && tdx::window_width(*d) == 0) return tdx::fail(TDX_E_BADARG, "TDX_FLAG_WINDOW: W == 0");
  return tdx::piece_descs(*d, piece->elem_first, piece->elem_count,
                          static_cast<unsigned char*>(staging) + piece->staging_off, out);
}

TDX_C_API int tdx_init_submit_host(const TdxInitDesc* descs, int n, void* staging, size_t staging_bytes,
                                   void* stream) {
  tdx::g_last_launches = 0;
  tdx::g_last_host_copies = 0;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (staging == nullptr || reinterpret_cast<uintptr_t>(staging) % 16)
    return tdx::fail(TDX_E_BADARG, "staging == NULL or not 16-byte aligned");
  thread_local std::vector<unsigned char> img;
  thread_local tdx::PlanSet plans;
  size_t used = 0;
  if (int rc = tdx::build_plan(descs, n, img, plans, used)) return rc;
  {
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, staging) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
      cudaGetLastError();
      return tdx::fail(TDX_E_BADARG, "staging is not device memory");
    }
    for (int i = 0; i < n; ++i) {
      if (descs[i].elem_count == 0) continue;
      if (cudaPointerGetAttributes(&attr, descs[i].dst) != cudaSuccess) {
        cudaGetLastError();
        return tdx::fail(TDX_E_BADARG, "cudaPointerGetAttributes(dst) failed");
      }
      if (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)
        return tdx::fail(TDX_E_BADARG, "tdx_init_submit_host: dst is device memory (tdx_init_launch takes it)");
    }
  }
  std::vector<TdxHostPiece> cut;
  int passes = 0;
  if (int rc = tdx::host_cut(descs, n, staging_bytes, cut, passes)) return rc;
  // every pass's table, laid out before anything is enqueued (its workspace must fit under its pieces)
  std::vector<std::vector<TdxInitDesc>> tables(static_cast<size_t>(passes));
  std::vector<size_t> floor(static_cast<size_t>(passes), staging_bytes);
  auto* base = static_cast<unsigned char*>(staging);
  for (const TdxHostPiece& p : cut) {
    TdxInitDesc part[3];
    const int k = tdx::piece_descs(descs[p.desc], p.elem_first, p.elem_count, base + p.staging_off, part);
    tables[p.pass].insert(tables[p.pass].end(), part, part + k);
    floor[p.pass] = std::min<size_t>(floor[p.pass], p.staging_off);
  }
  for (int p = 0; p < passes; ++p) {
    if (int rc = tdx::build_plan(tables[p].data(), static_cast<int>(tables[p].size()), img, plans, used)) return rc;
    if (used > floor[p]) return tdx::fail(TDX_E_WORKSPACE, "internal: a pass's workspace reaches into its pieces");
  }
  size_t next = 0;
  int launches = 0;
  for (int p = 0; p < passes; ++p) {
    if (int rc = tdx::build_plan(tables[p].data(), static_cast<int>(tables[p].size()), img, plans, used)) return rc;
    tdx::g_last_upload_bytes = used;
    void* pinned = nullptr;
    if (int rc = tdx::stage(img.data(), used, s, staging, &pinned)) return rc;
    for (size_t q = 0; q < plans.hdrs.size(); ++q)
      if (int rc = tdx::launch_groups(plans.hdrs[q], base + plans.base[q], s, launches)) return rc;
    for (; next < cut.size() && cut[next].pass == p; ++next) {
      const TdxHostPiece& c = cut[next];
      const size_t isz = tdx::itemsize_of(descs[c.desc].dtype);
      cudaError_t e = cudaMemcpyAsync(static_cast<unsigned char*>(descs[c.desc].dst) + c.elem_first * isz,
                                      base + c.staging_off, c.elem_count * isz, cudaMemcpyDeviceToHost, s);
      if (e != cudaSuccess) return tdx::cuda_fail(e, "cudaMemcpyAsync(device to host)");
      ++tdx::g_last_host_copies;
    }
  }
  tdx::g_last_launches = launches;
  return 0;
}

TDX_C_API int tdx_last_host_copies(void) { return tdx::g_last_host_copies; }

TDX_C_API int tdx_plan_upload(const TdxInitDesc* descs, int n, void* workspace,
                              size_t workspace_bytes, void* stream, TdxPlan* plan) {
  static_assert(sizeof(tdx::PlanHeader) <= sizeof(TdxPlan), "TdxPlan too small");
  thread_local std::vector<unsigned char> img;
  thread_local tdx::PlanSet plans;
  if (plan == nullptr) return tdx::fail(TDX_E_BADARG, "plan == NULL");
  size_t used = 0;
  if (int rc = tdx::build_plan(descs, n, img, plans, used)) return rc;
  if (plans.hdrs.size() != 1)
    return tdx::fail(TDX_E_BADARG, "tdx_plan_upload: the descriptors span more kernel families than one plan holds "
                                   "(47); tdx_init_launch takes them");
  memcpy(plan, &plans.hdrs[0], sizeof(tdx::PlanHeader));
  if (workspace == nullptr || workspace_bytes < used)
    return tdx::fail(TDX_E_WORKSPACE, "workspace too small (see tdx_init_workspace_bytes)");
  tdx::g_last_upload_bytes = used;
  cudaError_t e = cudaMemcpyAsync(workspace, img.data(), used, cudaMemcpyHostToDevice,
                                  static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return tdx::cuda_fail(e, "cudaMemcpyAsync(plan)");
  // the staging image is reused by the next call on this thread: make sure the copy has left it
  e = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return tdx::cuda_fail(e, "cudaStreamSynchronize(plan upload)");
  return 0;
}

TDX_C_API int tdx_plan_launch(const TdxPlan* plan, void* workspace, void* stream) {
  if (workspace == nullptr) return tdx::fail(TDX_E_WORKSPACE, "workspace == NULL");
  if (plan == nullptr) return tdx::fail(TDX_E_BADARG, "plan == NULL");
  tdx::PlanHeader hdr;
  memcpy(&hdr, plan, sizeof(hdr));
  if (hdr.magic != tdx::kPlanMagic) return tdx::fail(TDX_E_BADARG, "plan was not produced by tdx_plan_upload");
  int launches = 0;
  if (int rc = tdx::launch_groups(hdr, workspace, static_cast<cudaStream_t>(stream), launches)) return rc;
  tdx::g_last_launches = launches;
  return 0;
}

// The host image of the plan tdx_init_prepare() built on this thread, waiting for tdx_init_submit().
namespace tdx {
thread_local std::vector<unsigned char> g_prepared_img;
thread_local PlanSet g_prepared_plans;
thread_local size_t g_prepared_used = 0;
thread_local bool g_prepared = false;
}  // namespace tdx

TDX_C_API int tdx_init_prepare(const TdxInitDesc* descs, int n, size_t* workspace_bytes) {
  tdx::g_prepared = false;
  if (workspace_bytes == nullptr) return tdx::fail(TDX_E_BADARG, "workspace_bytes == NULL");
  if (int rc = tdx::build_plan(descs, n, tdx::g_prepared_img, tdx::g_prepared_plans, tdx::g_prepared_used)) return rc;
  *workspace_bytes = tdx::g_prepared_plans.hdrs[0].n_groups ? tdx::g_prepared_used : 0;
  tdx::g_prepared = true;
  return 0;
}

TDX_C_API int tdx_init_submit(void* workspace, size_t workspace_bytes, void* stream) {
  if (!tdx::g_prepared) return tdx::fail(TDX_E_BADARG, "tdx_init_submit without tdx_init_prepare on this thread");
  tdx::g_prepared = false;
  const tdx::PlanSet& plans = tdx::g_prepared_plans;
  if (plans.hdrs[0].n_groups == 0) {
    tdx::g_last_launches = 0;
    return 0;
  }
  const size_t used = tdx::g_prepared_used;
  if (workspace == nullptr || workspace_bytes < used)
    return tdx::fail(TDX_E_WORKSPACE, "workspace too small (see tdx_init_prepare)");
  // The plan image goes through a small ring of pinned staging buffers so that the copy is truly
  // asynchronous: the host can go on planning the next batch while the GPU works on this one.
  tdx::g_last_upload_bytes = used;
  void* pinned = nullptr;
  if (int rc = tdx::stage(tdx::g_prepared_img.data(), used, static_cast<cudaStream_t>(stream), workspace, &pinned))
    return rc;
  int launches = 0;
  for (size_t p = 0; p < plans.hdrs.size(); ++p)
    if (int rc = tdx::launch_groups(plans.hdrs[p], static_cast<unsigned char*>(workspace) + plans.base[p],
                                    static_cast<cudaStream_t>(stream), launches))
      return rc;
  tdx::g_last_launches = launches;
  return 0;
}

TDX_C_API int tdx_init_launch(const TdxInitDesc* descs, int n, void* workspace,
                              size_t workspace_bytes, void* stream) {
  size_t need = 0;
  if (int rc = tdx_init_prepare(descs, n, &need)) return rc;
  if (need == 0) {
    tdx::g_prepared = false;
    tdx::g_last_launches = 0;
    return 0;
  }
  if (workspace == nullptr || workspace_bytes < need) {
    tdx::g_prepared = false;
    return tdx::fail(TDX_E_WORKSPACE, "workspace too small (see tdx_init_workspace_bytes)");
  }
  return tdx_init_submit(workspace, workspace_bytes, stream);
}

TDX_C_API int tdx_last_launch_count(void) { return tdx::g_last_launches; }
TDX_C_API size_t tdx_last_upload_bytes(void) { return tdx::g_last_upload_bytes; }

TDX_C_API int tdx_elems_per_block(int dtype, int src, int algo) {
  if (src == TDX_SRC_CONST) return 0;
  if (dtype == TDX_F32) return 4;
  if (dtype != TDX_BF16 && dtype != TDX_F16) return 0;
  if ((algo & 0x0f) == TDX_ALGO_WIDE32) return 4;  // BM32 == WIDE32
  return 8;
}

TDX_C_API int tdx_abi_version(void) { return TDX_ABI_VERSION; }
TDX_C_API const char* tdx_last_error(void) { return tdx::g_err; }

}  // extern "C"
