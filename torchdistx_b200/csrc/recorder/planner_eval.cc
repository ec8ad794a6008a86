// Symbolic evaluation of a storage's recorded program (a State), its lowering to descriptors, and
// the questions answered from them without a GPU: plan_info, storage_history, analyze_tape.
#include "planner_internal.h"

#include <ATen/Functions.h>

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstring>
#include <limits>

#include "fake_tensor.h"

namespace tdx {

using c10::IValue;
using c10::ScalarType;
using torch::jit::Stack;

namespace {
thread_local c10::Device g_fold_device = c10::Device(c10::kCPU);
}  // namespace

FoldOn::FoldOn(c10::Device d) : prev(g_fold_device) { g_fold_device = d; }
FoldOn::~FoldOn() { g_fold_device = prev; }

namespace {

// The Tape::rng entry of an RNG op (made on first sight).
uint32_t rng_slot_of(Tape& tape, uint32_t op_idx) {
  TapeOp& op = tape.ops[op_idx];
  if (op.rng_slot == kNoValue) {
    RngSlot s;
    s.op = op_idx;
    if (op.handle) {
      const size_t pos = find_arg(op, "generator");
      s.explicit_generator = pos != static_cast<size_t>(-1) && pos < op.args.size() && op.args[pos].isGenerator();
    }
    op.rng_slot = static_cast<uint32_t>(tape.rng.size());
    tape.rng.push_back(s);
  }
  return op.rng_slot;
}

State make_opaque() { return State{}; }

constexpr size_t kMaxPlanEpi = 12;

bool is_ssm_step(uint32_t op) {
  op &= 0xffu;
  return op >= TDX_EPI_EXP && op <= TDX_EPI_MULADD;
}

// Does the program use the state-space extension (a new step or a broadcast index)?  Only such
// programs may grow past TDX_MAX_EPI steps and be compacted: every other keeps its descriptor.
bool uses_ssm(const Sym& sy) {
  if (sy.period != 0) return true;
  for (const TdxEpiStep& s : sy.epi)
    if (is_ssm_step(s.op)) return true;
  return false;
}

using EpiSteps = c10::SmallVector<TdxEpiStep, TDX_MAX_EPI>;

// The epilogue a segment emits: its steps if they fit (always so for programs without the
// extension); otherwise MUL followed by ADD (same rounding) merged into MULADD.  false: it does not
// fit a descriptor, and the program is replayed through ATen.
bool emit_epi(const Sym& sy, EpiSteps& out) {
  out.assign(sy.epi.begin(), sy.epi.end());
  if (out.size() <= TDX_MAX_EPI) return true;
  if (!uses_ssm(sy)) return false;
  EpiSteps m;
  for (size_t i = 0; i < sy.epi.size(); ++i) {
    const TdxEpiStep& s = sy.epi[i];
    if (i + 1 < sy.epi.size() && (s.op & 0xffu) == TDX_EPI_MUL && (sy.epi[i + 1].op & 0xffu) == TDX_EPI_ADD &&
        (s.op & TDX_EPI_NOROUND) == (sy.epi[i + 1].op & TDX_EPI_NOROUND)) {
      TdxEpiStep f;
      f.op = TDX_EPI_MULADD | (s.op & TDX_EPI_NOROUND);
      f.a = s.a;
      f.b = sy.epi[i + 1].a;
      m.push_back(f);
      ++i;
      continue;
    }
    m.push_back(s);
  }
  if (m.size() > TDX_MAX_EPI) return false;
  out = std::move(m);
  return true;
}

// The factor ATen's CUDA kernel multiplies an fp32 tensor by for `t / c` with a scalar c: the reciprocal
// of the double c, rounded once to fp32.  Not 1.0f / float(c): for a c that fp32 cannot hold the two
// differ (c = 0.001: 1000.0 against 999.99994, so `exp(arange(n)) / 0.001` was off by an ulp).
double div_multiplier(double c) { return static_cast<double>(static_cast<float>(1.0 / c)); }

bool same_step(const TdxEpiStep& x, const TdxEpiStep& y) {
  return x.op == y.op && std::memcmp(&x.a, &y.a, sizeof(float)) == 0 && std::memcmp(&x.b, &y.b, sizeof(float)) == 0;
}

// Element bits of `v` converted to `dtype` (the conversion at::full performs), without building a
// tensor.  Returns false for dtypes that are not handled here.
bool scalar_bits(const c10::Scalar& v, ScalarType dtype, unsigned char* out, size_t* isz) {
  auto put = [&](auto x) { std::memcpy(out, &x, sizeof(x)); *isz = sizeof(x); return true; };
  switch (dtype) {
    case ScalarType::Float: return put(v.to<float>());
    case ScalarType::Double: return put(v.to<double>());
    case ScalarType::BFloat16: return put(v.to<c10::BFloat16>());
    case ScalarType::Half: return put(v.to<c10::Half>());
    case ScalarType::Long: return put(v.to<int64_t>());
    case ScalarType::Int: return put(v.to<int32_t>());
    case ScalarType::Short: return put(v.to<int16_t>());
    case ScalarType::Char: return put(v.to<int8_t>());
    case ScalarType::Byte: return put(v.to<uint8_t>());
    case ScalarType::Bool: return put(v.to<bool>());
    default: return false;
  }
}

// The value `v` holds once it has been stored in a tensor of `dtype` (what `full(v, dtype=...)` /
// `fill_` keep of it: ATen converts with Scalar::to<scalar_t>()), as a Scalar again.  Lets a dtype
// cast of a constant be folded on the host, exactly: full(v, A).to(B) == B(A(v)).  false: a dtype
// or a value (out-of-range float -> integer) this does not model.
bool stored_value(const c10::Scalar& v, ScalarType dtype, c10::Scalar& out) {
  try {
    switch (dtype) {
      case ScalarType::Float: out = static_cast<double>(v.to<float>()); return true;
      case ScalarType::Double: out = v.to<double>(); return true;
      case ScalarType::BFloat16: out = static_cast<double>(static_cast<float>(v.to<c10::BFloat16>())); return true;
      case ScalarType::Half: out = static_cast<double>(static_cast<float>(v.to<c10::Half>())); return true;
      case ScalarType::Long: out = v.to<int64_t>(); return true;
      case ScalarType::Int: out = static_cast<int64_t>(v.to<int32_t>()); return true;
      case ScalarType::Short: out = static_cast<int64_t>(v.to<int16_t>()); return true;
      case ScalarType::Char: out = static_cast<int64_t>(v.to<int8_t>()); return true;
      case ScalarType::Byte: out = static_cast<int64_t>(v.to<uint8_t>()); return true;
      case ScalarType::Bool: out = v.to<bool>(); return true;
      default: return false;
    }
  } catch (...) {
    return false;
  }
}

// While a tape is analysed at the end of its recording (analyze_tape) the target device is not
// known yet, and a constant chain must be folded with the target device's arithmetic: such
// storages are evaluated when they are materialised instead.  The same holds for programs that
// read a real tensor's value (it may be mutated before the materialisation: the version check
// must see that).
thread_local bool g_analysis_only = false;
thread_local bool g_analysis_deferred = false;  // the last evaluation met one of those

// The 1-element tensor form of a constant state (needed to fold further ops through ATen).
void ensure_cval(Sym& st, ScalarType dtype) {
  if (st.cval.defined() || !st.has_scalar) return;
  c10::impl::ExcludeDispatchKeyGuard a{c10::DispatchKey::DeferredInit};
  c10::impl::ExcludeDispatchKeyGuard b{c10::DispatchKey::Fake};
  st.cval = at::full({1}, st.cscalar, at::TensorOptions().dtype(dtype).device(g_fold_device));
}

bool is_fused_float(ScalarType t) {
  return t == ScalarType::Float || t == ScalarType::BFloat16 || t == ScalarType::Half;
}

// Value of argument `pos` of a recorded op as a double, if it is a number or a real 1-element
// tensor (the form Python scalars take in mul_.Tensor / add_.Tensor).
std::optional<double> scalar_arg(const TapeOp& op, size_t pos) {
  if (pos >= op.args.size()) return std::nullopt;
  const IValue& v = op.args[pos];
  if (v.isDouble()) return v.toDouble();
  if (v.isInt()) return static_cast<double>(v.toInt());
  if (v.isBool()) return v.toBool() ? 1.0 : 0.0;
  if (v.isTensor()) {
    size_t slot = 0;  // which tensor slot of the frame is this argument?
    for (size_t i = 0; i < pos; ++i) {
      if (op.args[i].isTensor()) ++slot;
      else if (op.args[i].isList())
        for (const IValue& e : op.args[i].toListRef()) slot += e.isTensor();
    }
    if (slot >= op.inputs.size()) return std::nullopt;
    const at::Tensor& t = op.inputs[slot].real;
    if (!t.defined() || t.numel() != 1 || !t.is_cpu() || t.is_complex()) return std::nullopt;
    // A Python number the argument parser wrapped into a 0-dim tensor is nobody else's to mutate:
    // its value can be read when the tape is analysed.  Any other real tensor is read when the
    // storage is materialised (it may change until then: the version check must see that).
    if (g_analysis_only && !t.unsafeGetTensorImpl()->is_wrapped_number()) {
      g_analysis_deferred = true;
      return std::nullopt;
    }
    if (!t.is_inference() && static_cast<int64_t>(t._version()) != op.inputs[slot].real_version)
      return std::nullopt;  // mutated since recording: let generic replay raise the error
    return t.item<double>();
  }
  return std::nullopt;
}

// The addend of add / sub with a scalar (args 1 and 2: c and alpha): ATen's CUDA kernel computes
// x + alpha * c with alpha and c cast to fp32, and the product contracts into one FMA with the sum.  A step
// x + p equals that only when p = float(alpha) * float(c) is exact in fp32 (then every evaluation order
// rounds once, at the sum); otherwise nullopt, and ATen replays the op.  `negate`: sub (alpha's sign flipped).
std::optional<double> add_addend(const TapeOp& op, bool negate) {
  const auto c = scalar_arg(op, 1), alpha = scalar_arg(op, 2);
  if (!c || !alpha) return std::nullopt;
  const double p = static_cast<double>(static_cast<float>(*c)) * static_cast<double>(static_cast<float>(*alpha));
  if (static_cast<double>(static_cast<float>(p)) != p) return std::nullopt;
  return negate ? -p : p;
}

// ATen casts uniform_'s bounds to the tensor dtype before use
// ($TORCH/include/ATen/native/cuda/DistributionTemplates.h uniform_kernel, and the CPU twin).
double round_to_dtype(double x, ScalarType t) {
  switch (t) {
    case ScalarType::Float: return static_cast<double>(static_cast<float>(x));
    case ScalarType::BFloat16: return static_cast<double>(static_cast<float>(c10::BFloat16(static_cast<float>(x))));
    case ScalarType::Half: return static_cast<double>(static_cast<float>(c10::Half(static_cast<float>(x))));
    default: return x;
  }
}

// Runs the recorded operator on `self` (a 1-element tensor standing for a constant segment), with
// the recorded scalar arguments: exact ATen semantics for constant folding.  `dtype` is the
// segment's dtype before the op; on success it is the result's.
bool fold_const(const TapeOp& op, Sym& st, ScalarType& dtype, bool inplace) {
  if (g_analysis_only) {
    g_analysis_deferred = true;
    return false;
  }
  ensure_cval(st, dtype);
  st.has_scalar = false;
  if (!op.handle || !st.cval.defined()) return false;
  if (inplace) {
    // Segments are split by copying (`w[i].zero_()` makes three of one): their constants are handles
    // to ONE 1-element tensor until somebody writes.  An in-place op replayed on a shared constant
    // would reach every segment that holds it (`full(c); w[i].zero_(); w.add_(1)` added 1 twice to
    // the two outer segments; `w[a:b].mul_(2)` doubled the whole tensor): write to a private copy.
    NoInterception guard;
    st.cval = st.cval.clone();
  }
  Stack stack;
  size_t slot = 0;
  bool ok = true, first_tensor = true;
  for (const IValue& a : op.args) {
    if (a.isTensor()) {
      if (slot >= op.inputs.size()) return false;
      const InputRef& in = op.inputs[slot++];
      if (first_tensor) {
        if (st.cval.device() != g_fold_device) {
          NoInterception guard;
          st.cval = st.cval.to(g_fold_device);
        }
        stack.emplace_back(st.cval);
        first_tensor = false;
      } else if (in.real.defined() && in.real.numel() == 1 && in.real.is_cpu()) {
        stack.emplace_back(in.real);
      } else if (!in.real.defined() && in.value == kNoValue && !in.foreign) {
        stack.emplace_back(at::Tensor());
      } else {
        ok = false;
      }
    } else if (a.isList()) {
      for (const IValue& e : a.toListRef()) ok &= !e.isTensor();
      stack.push_back(a);
    } else if (a.isDevice()) {
      stack.emplace_back(g_fold_device);
    } else {
      stack.push_back(a);
    }
  }
  if (!ok) return false;
  NoInterception guard;
  op.handle->callBoxed(stack);
  if (stack.empty() || !stack.back().isTensor()) return false;
  at::Tensor out = stack.back().toTensor();
  if (out.numel() != 1) return false;
  st.cval = inplace ? st.cval : out;
  dtype = st.cval.scalar_type();
  return true;
}

// ---- segment bookkeeping ------------------------------------------------------------------------
// The elements of the storage a value names, if they are one contiguous run.
bool range_of(const ValueInfo& v, int64_t& begin, int64_t& end) {
  int64_t expect = 1;
  for (int64_t d = static_cast<int64_t>(v.sizes.size()) - 1; d >= 0; --d) {
    if (v.sizes[d] == 1) continue;
    if (v.strides[d] != expect) return false;
    expect *= v.sizes[d];
  }
  begin = v.storage_offset;
  end = v.storage_offset + v.numel;
  return true;
}

// Cuts the segments at `at` so that none straddles it.
void split_at(SegList& segs, int64_t at) {
  for (size_t i = 0; i < segs.size(); ++i) {
    if (segs[i].begin < at && at < segs[i].end) {
      Seg right = segs[i];
      right.begin = at;
      segs[i].end = at;
      segs.insert(segs.begin() + static_cast<std::ptrdiff_t>(i) + 1, std::move(right));
      return;
    }
  }
}

// [b, e) now holds `st` (an op that overwrites what was there).
void overwrite(State& s, int64_t b, int64_t e, Sym st, int64_t origin) {
  if (b >= e) return;
  split_at(s.segs, b);
  split_at(s.segs, e);
  SegList out;
  out.reserve(s.segs.size() + 1);
  bool placed = false;
  for (Seg& g : s.segs) {
    if (g.begin >= b && g.end <= e) {
      if (!placed) {
        Seg n;
        n.begin = b;
        n.end = e;
        n.origin = origin;
        n.st = std::move(st);
        out.push_back(std::move(n));
        placed = true;
      }
      continue;
    }
    out.push_back(std::move(g));
  }
  s.segs = std::move(out);
}

void merge_rng_chain(State& st, const State& other) {
  for (const RngPass& r : other.rng_chain) {
    bool have = false;
    for (const RngPass& q : st.rng_chain) have |= q.op == r.op;
    if (!have) st.rng_chain.push_back(r);
  }
}

// The state of the recorded tensor argument `k` of `op` as of the op, if it is one segment over its
// whole storage, named by the argument from element 0 on.  nullptr otherwise.
const Seg* whole_arg(Tape& tape, const TapeOp& op, size_t k, uint32_t op_idx, uint32_t S, State& st) {
  if (k >= op.inputs.size() || op.inputs[k].foreign || op.inputs[k].value == kNoValue) return nullptr;
  const ValueInfo& v = tape.values[op.inputs[k].value];
  int64_t b = 0, e = 0;
  if (v.storage == S || !range_of(v, b, e) || b != 0) return nullptr;
  st = eval_storage(tape, v.storage, op_idx);
  if (st.opaque || st.dtype != v.dtype || st.segs.size() != 1) return nullptr;
  const Seg& g = st.segs[0];
  if (g.begin != 0 || g.end != e || g.origin != 0) return nullptr;
  return &g;
}

// `st` becomes one segment `sy` over the whole storage `out` names, in `dtype`, with the RNG passes of
// `srcs` (a new storage: a factory, or an out-of-place op).
void fill_whole(State& st, const ValueInfo& out, ScalarType dtype, Sym sy, std::initializer_list<const State*> srcs = {}) {
  State res;
  res.opaque = false;
  res.dtype = dtype;
  for (const State* s : srcs) merge_rng_chain(res, *s);
  Seg g;
  g.end = out.numel;
  g.st = std::move(sy);
  res.segs.push_back(std::move(g));
  st = std::move(res);
}

// Appends an epilogue step; false: the program has as many steps as a descriptor can take.
bool push_epi(Sym& sy, uint32_t code, double a, double b = 0) {
  if (sy.epi.size() >= ((is_ssm_step(code) || uses_ssm(sy)) ? kMaxPlanEpi : TDX_MAX_EPI)) return false;
  TdxEpiStep s;
  s.op = code;  // every step rounds to the tensor dtype, like the in-place ATen op it stands for
  s.a = static_cast<float>(a);
  s.b = static_cast<float>(b);
  sy.epi.push_back(s);
  return true;
}

// clamp(min, max) / clamp_(min, max), either bound may be None.
bool push_clamp(Sym& sy, const TapeOp& op) {
  const bool has_min = !op.args[1].isNone(), has_max = !op.args[2].isNone();
  const auto lo = scalar_arg(op, 1), hi = scalar_arg(op, 2);
  return !((has_min && !lo) || (has_max && !hi)) &&
         push_epi(sy, TDX_EPI_CLAMP, has_min ? *lo : -std::numeric_limits<double>::infinity(),
                  has_max ? *hi : std::numeric_limits<double>::infinity());
}

// Is the second tensor argument of `op` a recorded tensor (`a * b`, `a + b`), not a scalar?
bool second_is_recorded(const TapeOp& op) {
  return op.inputs.size() > 1 && (op.inputs[1].value != kNoValue || op.inputs[1].foreign);
}

// ---- the rules: each applies one kind of op to `st`, or returns false (the state is then opaque) --

// The three ops of a sinusoidal position table (Whisper `sinusoids`, M2M100 / MusicGen
// `get_embedding`, GPT-J / CodeGen `create_sinusoidal_positions`):
//   P = rows * cols   a [R, 1] view of a plain arange(R) (int64, or cast to fp32) times a [1, H] view
//                     of a 1-D fp32 index program of at most TDX_MAX_EPI steps, either order (einsum
//                     "i,j->ij" records the same mul);
//   sin(P), cos(P)    out of place;
//   cat([sin(P), cos(P)], dim=-1), or [cos(P), sin(P)], over the same P.
// Any other mul of two recorded tensors, einsum, sin / cos, or cat is opaque, as before.
bool sincos_transition(Tape& tape, const TapeOp& op, uint32_t op_idx, uint32_t S, const ValueInfo& out, State& st) {
  const bool ok2d = out.covers_storage && out.dtype == ScalarType::Float && out.sizes.size() == 2;
  if (op.kind == OpKind::MulOut || op.kind == OpKind::EinsumOut) {
    // einsum "i,j->ij" of two 1-D operands (GPT-J, CodeGen) is that mul of their [R, 1] and [1, H]
    // views (ATen's einsum multiplies when nothing is summed), rows first
    bool outer_eq = false;
    if (op.kind == OpKind::EinsumOut && !op.args.empty() && op.args[0].isString()) {
      std::string eq;
      for (char ch : op.args[0].toStringRef())
        if (ch != ' ') eq += ch;
      outer_eq = eq.size() == 7 && eq[1] == ',' && eq[3] == '-' && eq[4] == '>' && eq[0] != eq[2] &&
                 std::isalpha(static_cast<unsigned char>(eq[0])) && std::isalpha(static_cast<unsigned char>(eq[2])) &&
                 eq[5] == eq[0] && eq[6] == eq[2];
    }
    const int64_t R = ok2d ? out.sizes[0] : 0, H = ok2d ? out.sizes[1] : 0;
    if (R < 2 || H < 2 || R >= (int64_t{1} << 24) || op.inputs.size() != 2 ||
        (op.kind == OpKind::EinsumOut && !outer_eq))
      return false;
    State side[2];
    const Seg* g[2] = {nullptr, nullptr};
    int row = op.kind == OpKind::EinsumOut ? 0 : -1;
    for (int k = 0; k < 2; ++k) {
      g[k] = whole_arg(tape, op, static_cast<size_t>(k), op_idx, S, side[k]);
      if (!g[k]) return false;
      const ValueInfo& v = tape.values[op.inputs[static_cast<size_t>(k)].value];
      if (op.kind == OpKind::EinsumOut) {
        if (v.sizes.size() != 1 || v.sizes[0] != (k == 0 ? R : H)) return false;
        continue;
      }
      if (v.sizes.size() != 2) return false;
      if (v.sizes[0] == R && v.sizes[1] == 1) row = row < 0 ? k : 2;
      else if (!(v.sizes[0] == 1 && v.sizes[1] == H)) return false;
    }
    if (row < 0 || row > 1) return false;
    const Sym &rs = g[row]->st, &cs = g[1 - row]->st;
    const ScalarType rdt = side[row].dtype, cdt = side[1 - row].dtype;
    EpiSteps epi;
    const bool rows_ok = rs.src == Sym::Iota && rs.period == 0 && rs.p0 == 0.0 && rs.p1 == 1.0 && rs.epi.empty() &&
                         (rdt == ScalarType::Long || rdt == ScalarType::Float);
    const bool cols_ok = cs.src == Sym::Iota && cs.period == 0 && cdt == ScalarType::Float && emit_epi(cs, epi);
    if (!rows_ok || !cols_ok) return false;
    Sym sy;
    sy.src = Sym::Outer;
    sy.p0 = cs.p0;
    sy.p1 = cs.p1;
    sy.epi.assign(epi.begin(), epi.end());
    sy.half = H;
    sy.outer_storage = S;
    fill_whole(st, out, ScalarType::Float, std::move(sy), {&side[0], &side[1]});
    return true;
  }
  if (op.kind == OpKind::SinOut || op.kind == OpKind::CosOut) {
    State src;
    const Seg* g = ok2d ? whole_arg(tape, op, 0, op_idx, S, src) : nullptr;
    if (!g || g->st.src != Sym::Outer || g->st.trig != 0 || g->end != out.numel || src.dtype != ScalarType::Float)
      return false;
    src.segs[0].st.trig = op.kind == OpKind::SinOut ? 1 : 2;
    st = std::move(src);
    return true;
  }
  // cat
  const int64_t dim = op.args.size() > 1 && op.args[1].isInt() ? op.args[1].toInt() : 0;
  if (!ok2d || op.inputs.size() != 2 || !(dim == 1 || dim == -1) || out.sizes[1] % 2) return false;
  State side[2];
  const Seg* g[2] = {nullptr, nullptr};
  for (int k = 0; k < 2; ++k) {
    g[k] = whole_arg(tape, op, static_cast<size_t>(k), op_idx, S, side[k]);
    const ValueInfo* v = g[k] ? &tape.values[op.inputs[static_cast<size_t>(k)].value] : nullptr;
    if (!v || v->sizes.size() != 2 || v->sizes[0] != out.sizes[0] || v->sizes[1] * 2 != out.sizes[1] ||
        g[k]->st.src != Sym::Outer || g[k]->st.trig == 0 || g[k]->st.half != v->sizes[1])
      return false;
  }
  const Sym &a = g[0]->st, &b = g[1]->st;
  bool same = a.outer_storage == b.outer_storage && a.trig != b.trig && a.p0 == b.p0 && a.p1 == b.p1 &&
              a.half == b.half && a.epi.size() == b.epi.size();
  for (size_t i = 0; same && i < a.epi.size(); ++i) same = same_step(a.epi[i], b.epi[i]);
  if (!same) return false;
  Sym sy = a;
  sy.src = Sym::Sincos;
  sy.cos_first = a.trig == 2;
  sy.trig = 0;
  sy.outer_storage = kNoValue;
  fill_whole(st, out, ScalarType::Float, std::move(sy), {&side[0], &side[1]});
  return true;
}

// Largest source (bytes, in the destination dtype) a copy of a host-built tensor takes onto the fused
// path: the bytes travel with every submission and every InitPlan that holds them (RWKV's time_*
// vectors are KBs; the embedding limit of InitPlan is the same 1 MB).
constexpr int64_t kMaxGatherBytes = int64_t{1} << 20;

bool is_gather_dtype(ScalarType t) { return is_fused_float(t) || t == ScalarType::Long; }

// dst.copy_(real), `real` a tensor built eagerly while recording (from Python lists or numpy): the
// elements `out` names become its elements, converted to dst's dtype by ATen on the host (the
// conversion copy_ itself performs: round to nearest even).  The value is read when the storage is
// evaluated for materialisation -- never while the recording is analysed -- and only if the tensor
// is unchanged since recording; otherwise the copy is opaque and generic replay raises the version
// error.  Forms: the source the size of `out`, or broadcast to it (one block of walking dimensions,
// the broadcast geometry {P, R}); `out` a contiguous range of the storage, or a strided view inside
// one segment that is uninitialised or already such a copy (Pegasus / Marian write the two halves
// of a table into column slices: the segment becomes one host image).  false: opaque.
bool gather_copy(const TapeOp& op, const ValueInfo& out, State& st) {
  if (g_analysis_only) {
    g_analysis_deferred = true;
    return false;
  }
  const InputRef& in = op.inputs[1];
  const at::Tensor& real = in.real;
  if (st.opaque || out.dtype != st.dtype || st.segs.empty() || !is_gather_dtype(out.dtype) || !real.is_cpu() ||
      !(is_gather_dtype(real.scalar_type()) || real.scalar_type() == ScalarType::Double))
    return false;
  if (!real.is_inference() && static_cast<int64_t>(real._version()) != in.real_version)
    return false;  // mutated since recording: generic replay raises the error
  NoInterception guard;
  at::Tensor e;
  try {
    e = real.expand(c10::IntArrayRef(out.sizes));
  } catch (const c10::Error&) {
    return false;
  }
  // the real tensor must be contiguous once its broadcast and size-1 dimensions are left out
  int64_t expect = 1;
  for (int64_t d = real.dim() - 1; d >= 0; --d) {
    if (real.size(d) == 1 || real.stride(d) == 0) continue;
    if (real.stride(d) != expect) return false;
    expect *= real.size(d);
  }
  // broadcast geometry: P elements walked by one block of dimensions, each repeated R times
  int first = -1, last = -1;
  for (int d = 0; d < static_cast<int>(e.dim()); ++d)
    if (e.size(d) > 1 && e.stride(d) != 0) {
      if (first < 0) first = d;
      last = d;
    }
  int64_t P = 1, R = 1;
  for (int d = 0; d < static_cast<int>(e.dim()); ++d) {
    if (first >= 0 && d >= first && d <= last) {
      if (e.size(d) > 1 && e.stride(d) == 0) return false;  // a broadcast dimension inside the block
      P *= e.size(d);
    } else if (d > last) {
      R *= e.size(d);
    }
  }
  const int64_t isz = static_cast<int64_t>(c10::elementSize(out.dtype));
  if (P * isz > kMaxGatherBytes || R >= (int64_t{1} << 32)) return false;
  at::Tensor c = e;
  for (int d = 0; d < static_cast<int>(c.dim()); ++d)
    if (c.size(d) > 1 && c.stride(d) == 0) c = c.narrow(d, 0, 1);
  Sym sy;
  sy.src = Sym::Gather;
  int64_t b = 0, end = 0;
  if (range_of(out, b, end)) {
    if (b < 0 || end > st.segs.back().end) return false;
    sy.gsrc = c.reshape({-1}).to(out.dtype, /*non_blocking=*/false, /*copy=*/true).contiguous();
    if (P != out.numel) {
      sy.period = P;
      sy.repeat = R > 1 ? R : 0;
    }
    overwrite(st, b, end, std::move(sy), b);
    return true;
  }
  // a strided view: written into a host image of the one segment it lies in
  int64_t lo = out.storage_offset, hi = out.storage_offset + 1;
  for (size_t d = 0; d < out.sizes.size(); ++d) {
    if (out.sizes[d] == 0) return true;  // (nothing is written)
    if (out.sizes[d] > 1 && out.strides[d] <= 0) return false;
    hi += (out.sizes[d] - 1) * out.strides[d];
  }
  for (Seg& g : st.segs) {
    if (!(g.begin <= lo && hi <= g.end)) continue;
    const int64_t n = g.end - g.begin;
    if (n * isz > kMaxGatherBytes) return false;
    at::Tensor image;
    if (g.st.src == Sym::Uninit) {
      image = at::zeros({n}, at::TensorOptions().dtype(out.dtype));
    } else if (g.st.src == Sym::Gather && g.st.period == 0 && g.st.epi.empty() && g.origin == g.begin &&
               g.st.gsrc.numel() == n) {
      image = g.st.gsrc.clone();
    } else {
      return false;
    }
    image.as_strided(c10::IntArrayRef(out.sizes), c10::IntArrayRef(out.strides), lo - g.begin).copy_(e);
    sy.gsrc = std::move(image);
    g.st = std::move(sy);
    g.origin = g.begin;
    return true;
  }
  return false;
}

// The smallest mask (rows and columns) that becomes a band.  A smaller `tril` / `triu` keeps the
// path it had before bands existed: ATen replays it, and an InitPlan stores its few bytes by value
// (so that such a plan keeps the format older readers take).
constexpr int64_t kMinBandSide = 16;

// The value of a constant segment as it is stored in `dtype`.  A constant that only exists as a
// 1-element tensor is read back (never while the recording is analysed: the fold device is not known).
bool const_value(const Sym& sy, ScalarType dtype, c10::Scalar& out) {
  if (sy.has_scalar) return stored_value(sy.cscalar, dtype, out);
  if (!sy.cval.defined()) return false;
  if (g_analysis_only) {
    g_analysis_deferred = true;
    return false;
  }
  NoInterception guard;
  return stored_value(sy.cval.cpu().item(), dtype, out);
}

bool is_zero_value(const c10::Scalar& v, ScalarType dtype) {
  unsigned char b[16] = {};
  size_t isz = 0;
  if (!scalar_bits(v, dtype, b, &isz)) return false;
  for (size_t i = 0; i < isz; ++i)
    if (b[i]) return false;
  return true;
}

// The causal-mask programs (GPT-BigCode, GPT-Neo, ImageGPT, OpenAI GPT, Bark, CLVP):
//   tril(x, k) / triu(x, k), out of place or in place, of x one constant segment over a contiguous
//                     [..., R, C] storage: the band [-R, k] / [k, C] of the constant, 0 outside;
//   tril / triu of such a band whose outside value is 0 (bit for bit): the bounds intersect;
//   bitwise_xor(A, B) of two bool bands of the same geometry, true inside and false outside, nested
//                     with one shared bound (GPT-Neo's local layers: [-R, 0] xor [-R, -w] = [1 - w, 0]).
// A band that covers no diagonal is the constant outside value.  Everything else of these kinds
// (another source, a band with a non-zero outside, non-nested xor, a non-contiguous argument, a
// mask under kMinBandSide) is opaque, as before.
bool band_transition(Tape& tape, const TapeOp& op, uint32_t op_idx, uint32_t S, const ValueInfo& out, State& st) {
  const size_t nd = out.sizes.size();
  const int64_t R = nd >= 2 ? out.sizes[nd - 2] : 0, C = nd >= 2 ? out.sizes[nd - 1] : 0;
  if (R < kMinBandSide || C < kMinBandSide || R >= (int64_t{1} << 31) || C >= (int64_t{1} << 31)) return false;
  // the result: one segment over the whole storage (an empty band is the constant outside value)
  auto result = [&](const State& src, ScalarType dtype, Sym sy) {
    sy.band_rows = R;
    sy.band_cols = C;
    sy.band_lo = std::max<int64_t>(sy.band_lo, -R);
    sy.band_hi = std::min<int64_t>(sy.band_hi, C);
    if (sy.band_lo > sy.band_hi || sy.band_hi < 1 - R || sy.band_lo > C - 1) {
      Sym k;
      k.src = Sym::Const;
      k.cscalar = sy.band_out;
      k.has_scalar = true;
      sy = std::move(k);
    }
    fill_whole(st, out, dtype, std::move(sy), {&src});
    return true;
  };
  if (op.kind != OpKind::XorOut) {
    const bool lower = op.kind == OpKind::TrilOut || op.kind == OpKind::TrilInplace;
    const bool inplace = op.kind == OpKind::TrilInplace || op.kind == OpKind::TriuInplace;
    const size_t pd = op.handle ? find_arg(op, "diagonal") : static_cast<size_t>(-1);
    const int64_t k = pd == static_cast<size_t>(-1) || pd >= op.args.size() ? 0 : op.args[pd].toInt();
    State src;
    const Seg* g = nullptr;
    int64_t b = 0, e = 0;
    if (inplace) {  // the whole storage, one segment numbered from its first element
      if (!st.opaque && st.dtype == out.dtype && st.segs.size() == 1 && range_of(out, b, e) && b == 0 &&
          st.segs[0].begin == 0 && st.segs[0].end == e && st.segs[0].origin == 0) {
        src = std::move(st);
        g = &src.segs[0];
      }
    } else if (out.covers_storage) {
      g = whole_arg(tape, op, 0, op_idx, S, src);
      if (g && (src.dtype != out.dtype || tape.values[op.inputs[0].value].sizes != out.sizes)) g = nullptr;
    }
    if (!g) return false;
    Sym sy;
    sy.src = Sym::Band;
    if (g->st.src == Sym::Const) {
      if (!const_value(g->st, out.dtype, sy.band_in) || !stored_value(c10::Scalar(0), out.dtype, sy.band_out))
        return false;
      sy.band_lo = -R;
      sy.band_hi = C;
    } else if (g->st.src == Sym::Band && g->st.band_rows == R && g->st.band_cols == C &&
               is_zero_value(g->st.band_out, out.dtype)) {
      sy = g->st;
    } else {
      return false;
    }
    if (lower) sy.band_hi = std::min(sy.band_hi, k);
    else sy.band_lo = std::max(sy.band_lo, k);
    return result(src, out.dtype, std::move(sy));
  }
  // bitwise_xor of two bool bands
  if (!out.covers_storage || out.dtype != ScalarType::Bool || op.inputs.size() != 2) return false;
  State side[2];
  const Seg* g[2] = {nullptr, nullptr};
  for (int j = 0; j < 2; ++j) {
    g[j] = whole_arg(tape, op, static_cast<size_t>(j), op_idx, S, side[j]);
    const ValueInfo* v = g[j] ? &tape.values[op.inputs[static_cast<size_t>(j)].value] : nullptr;
    if (!v || v->sizes != out.sizes || side[j].dtype != ScalarType::Bool || g[j]->st.src != Sym::Band ||
        g[j]->st.band_rows != R || g[j]->st.band_cols != C || !g[j]->st.band_in.toBool() ||
        g[j]->st.band_out.toBool())
      return false;
  }
  const Sym &a = g[0]->st, &c = g[1]->st;
  Sym sy = a;
  if (a.band_lo == c.band_lo) {  // (lo, min(hi)] ... (lo, max(hi)]: the diagonals one band adds
    sy.band_lo = std::min(a.band_hi, c.band_hi) + 1;
    sy.band_hi = std::max(a.band_hi, c.band_hi);
  } else if (a.band_hi == c.band_hi) {
    sy.band_lo = std::min(a.band_lo, c.band_lo);
    sy.band_hi = std::max(a.band_lo, c.band_lo) - 1;
  } else {
    return false;
  }
  merge_rng_chain(side[0], side[1]);
  return result(side[0], ScalarType::Bool, std::move(sy));
}

// Factories: one segment over the whole (new) storage.
bool factory_rule(Tape& tape, const TapeOp& op, uint32_t op_idx, const ValueInfo& out, State& st) {
  if (!out.covers_storage) return false;
  Sym sy;
  switch (op.kind) {
    case OpKind::Empty:
      break;
    case OpKind::Zeros:
    case OpKind::Ones:
    case OpKind::Full: {
      sy.src = Sym::Const;
      sy.has_scalar = true;
      if (op.kind == OpKind::Zeros) sy.cscalar = 0;
      else if (op.kind == OpKind::Ones) sy.cscalar = 1;
      else {
        const size_t pos = find_arg(op, "fill_value");
        if (pos == static_cast<size_t>(-1) || !op.args[pos].isScalar()) return false;
        sy.cscalar = op.args[pos].toScalar();
      }
      break;
    }
    case OpKind::Randn:
    case OpKind::Rand:
      if (!is_fused_float(out.dtype)) return false;
      sy.src = op.kind == OpKind::Randn ? Sym::Normal : Sym::Uniform;
      sy.p0 = 0.0;
      sy.p1 = 1.0;
      sy.rng_op = op_idx;
      fill_whole(st, out, out.dtype, std::move(sy));
      st.rng_chain.push_back(RngPass{op_idx, out.numel, rng_slot_of(tape, op_idx)});
      return true;
    default: {  // Arange
      // arange([start,] end[, step]) with integer start / step: exact in int64, and in fp32 as long as
      // every value stays below 2^24 (then no question of how the kernel rounds start + i * step)
      if (!(out.dtype == ScalarType::Long || out.dtype == ScalarType::Float)) return false;
      const size_t ps = find_arg(op, "start"), pt = find_arg(op, "step");
      const auto start = ps == static_cast<size_t>(-1) ? std::optional<double>(0.0) : scalar_arg(op, ps);
      const auto step = pt == static_cast<size_t>(-1) ? std::optional<double>(1.0) : scalar_arg(op, pt);
      const double kExact = out.dtype == ScalarType::Float ? 16777216.0 : 9007199254740992.0;
      if (!start || !step || *start != std::floor(*start) || *step != std::floor(*step) ||
          std::fabs(*start) + std::fabs(*step) * static_cast<double>(out.numel) >= kExact)
        return false;
      sy.src = Sym::Iota;
      sy.p0 = *start;
      sy.p1 = *step;
    }
  }
  fill_whole(st, out, out.dtype, std::move(sy));
  return true;
}

// dst.copy_(src): the range `out` names becomes src's elements.
bool copy_rule(Tape& tape, const TapeOp& op, uint32_t op_idx, uint32_t S, const ValueInfo& out, State& st) {
  if (op.inputs.size() >= 2 && op.inputs[1].value == kNoValue && !op.inputs[1].foreign && op.inputs[1].real.defined())
    return gather_copy(op, out, st);  // from a real (host-built) tensor
  int64_t b = 0, e = 0;
  if (st.opaque || out.dtype != st.dtype || !range_of(out, b, e) || st.segs.empty() || b < 0 ||
      e > st.segs.back().end || op.inputs.size() < 2 || op.inputs[1].value == kNoValue)
    return false;
  const ValueInfo& in = tape.values[op.inputs[1].value];
  int64_t sb = 0, se = 0;
  if (in.numel != out.numel || in.dtype != out.dtype || in.storage == S || !range_of(in, sb, se) ||
      in.sizes != out.sizes)  // (no broadcasting, no dtype conversion)
    return false;
  State src = eval_storage(tape, in.storage, op_idx);
  if (src.opaque || src.dtype != in.dtype || src.segs.empty() || sb < 0 || se > src.segs.back().end) return false;
  for (Seg& g : src.segs) {
    const int64_t gb = std::max(g.begin, sb), ge = std::min(g.end, se);
    if (gb >= ge) continue;
    overwrite(st, b + (gb - sb), b + (ge - sb), g.st, g.origin - sb + b);
  }
  merge_rng_chain(st, src);  // the source's passes must have their streams when dst is built
  return true;
}

// In-place writers and steps through `out` (the whole tensor or a contiguous view of part of it).
bool inplace_rule(Tape& tape, const TapeOp& op, uint32_t op_idx, const ValueInfo& out, State& st) {
  int64_t b = 0, e = 0;
  if (st.opaque || out.dtype != st.dtype || !range_of(out, b, e) || st.segs.empty() || b < 0 ||
      e > st.segs.back().end)
    return false;
  if (op.kind == OpKind::UniformInplace || op.kind == OpKind::NormalInplace) {
    if (!is_fused_float(out.dtype)) return false;
    const bool uni = op.kind == OpKind::UniformInplace;
    const auto a = scalar_arg(op, 1), c = scalar_arg(op, 2);
    if (!a || !c) return false;
    Sym sy;
    sy.src = uni ? Sym::Uniform : Sym::Normal;
    if (uni) {
      TORCH_CHECK(*a <= *c, "uniform_ expects to return a [from, to) range, but found from=", fmt_double(*a),
                  " > to=", fmt_double(*c));
      sy.p0 = round_to_dtype(*a, out.dtype);
      sy.p1 = round_to_dtype(*c, out.dtype);
    } else {
      TORCH_CHECK(*c >= 0.0, "normal expects std >= 0.0, but found std ", fmt_double(*c));
      sy.p0 = *a;
      sy.p1 = *c;
    }
    sy.rng_op = op_idx;
    overwrite(st, b, e, std::move(sy), b);
    st.rng_chain.push_back(RngPass{op_idx, out.numel, rng_slot_of(tape, op_idx)});
    return true;
  }
  if (op.kind == OpKind::FillInplace || op.kind == OpKind::ZeroInplace) {
    Sym sy;
    sy.src = Sym::Const;
    if (op.kind == OpKind::ZeroInplace) {
      sy.cscalar = 0;
      sy.has_scalar = true;
    } else if (op.args.size() > 1 && op.args[1].isScalar()) {
      sy.cscalar = op.args[1].toScalar();
      sy.has_scalar = true;
    } else if (op.inputs.size() > 1 && op.inputs[1].real.defined() &&
               op.inputs[1].real.numel() == 1 && op.inputs[1].real.is_cpu()) {
      if (g_analysis_only) {
        g_analysis_deferred = true;
        return false;
      }
      NoInterception guard;
      sy.cval = op.inputs[1].real.detach().to(out.dtype).reshape({1}).clone();
    } else {
      return false;
    }
    overwrite(st, b, e, std::move(sy), b);
    return true;
  }
  // elementwise: applies to every segment inside [b, e)
  split_at(st.segs, b);
  split_at(st.segs, e);
  for (Seg& g : st.segs) {
    if (g.begin < b || g.end > e) continue;
    Sym& sy = g.st;
    if (sy.src == Sym::Uninit) return false;
    if (sy.src == Sym::Const) {
      ScalarType dt = st.dtype;
      if (!fold_const(op, sy, dt, /*inplace=*/true) || dt != st.dtype) return false;
      continue;
    }
    if (sy.src == Sym::Iota && st.dtype != ScalarType::Float) return false;
    if (sy.src == Sym::Outer || sy.src == Sym::Sincos || sy.src == Sym::Band) return false;  // (no step folds onto them)
    if (sy.src == Sym::Gather && !is_fused_float(st.dtype)) return false;  // (int64: a copy only)
    bool ok = true;
    if (op.kind == OpKind::MulInplace) {
      const auto c = scalar_arg(op, 1);
      ok = c && push_epi(sy, TDX_EPI_MUL, *c);
    } else if (op.kind == OpKind::AddInplace || op.kind == OpKind::SubInplace) {
      // x - alpha * c is computed by ATen as x + (-alpha) * c (sub is add with the sign of alpha flipped)
      const auto p = add_addend(op, op.kind == OpKind::SubInplace);
      ok = p && push_epi(sy, TDX_EPI_ADD, *p);
    } else if (op.kind == OpKind::NegInplace) {
      ok = push_epi(sy, TDX_EPI_MUL, -1.0);
    } else if (op.kind == OpKind::DivInplace) {
      // fp32 only, like DivOut below: ATen's CUDA kernel multiplies by the reciprocal of the divisor
      const auto c = scalar_arg(op, 1);
      ok = c && st.dtype == ScalarType::Float && *c != 0.0 && push_epi(sy, TDX_EPI_MUL, div_multiplier(*c));
    } else if (op.kind == OpKind::ErfinvInplace) {
      ok = push_epi(sy, TDX_EPI_ERFINV, 0);
    } else if (op.kind == OpKind::ExpInplace || op.kind == OpKind::LogInplace || op.kind == OpKind::Expm1Inplace) {
      ok = push_epi(sy, op.kind == OpKind::ExpInplace ? TDX_EPI_EXP : op.kind == OpKind::LogInplace ? TDX_EPI_LOG
                                                                                                   : TDX_EPI_EXPM1, 0);
    } else {  // clamp_
      ok = push_clamp(sy, op);
    }
    if (!ok) return false;
  }
  return true;
}

// `a + b` of two recorded tensors: only the inverse of softplus, `dt + log(-expm1(-dt))` (Mamba's dt
// bias), is modelled.  Both sides must be one program over the same elements of one source (same RNG
// op, or the same index program), b's = a's followed by exactly neg, expm1, neg, log.
bool softplus_add_rule(Tape& tape, const TapeOp& op, uint32_t op_idx, uint32_t S, const ValueInfo& out, State& st) {
  const auto alpha = scalar_arg(op, 2);
  State side[2];
  for (int k = 0; k < 2; ++k) {
    if (op.inputs[k].foreign) return false;
    const ValueInfo& v = tape.values[op.inputs[k].value];
    if (!v.covers_storage || v.storage == S || v.dtype != out.dtype || v.sizes != out.sizes) return false;
    side[k] = eval_storage(tape, v.storage, op_idx);
    if (side[k].opaque || side[k].dtype != v.dtype || side[k].segs.size() != 1) return false;
  }
  const Seg &sa = side[0].segs[0], &sb = side[1].segs[0];
  const Sym &a = sa.st, &bs = sb.st;
  static const uint32_t kTail[4] = {TDX_EPI_MUL, TDX_EPI_EXPM1, TDX_EPI_MUL, TDX_EPI_LOG};
  bool ok = alpha && *alpha == 1.0 && a.src == bs.src && (a.rng() || a.src == Sym::Iota) && sa.origin == sb.origin &&
            sa.begin == sb.begin && sa.end == sb.end && a.p0 == bs.p0 && a.p1 == bs.p1 && a.period == bs.period &&
            a.repeat == bs.repeat && a.wide == bs.wide && a.src_noround == bs.src_noround &&
            (!a.rng() || a.rng_op == bs.rng_op) && bs.epi.size() == a.epi.size() + 4;
  for (size_t i = 0; ok && i < a.epi.size(); ++i) ok = same_step(a.epi[i], bs.epi[i]);
  for (size_t i = 0; ok && i < 4; ++i) {
    const TdxEpiStep& s = bs.epi[a.epi.size() + i];
    ok = s.op == kTail[i] && (s.op != TDX_EPI_MUL || s.a == -1.0f);
  }
  if (!ok) return false;
  st = std::move(side[0]);
  merge_rng_chain(st, side[1]);
  return push_epi(st.segs[0].st, TDX_EPI_INV_SOFTPLUS, 0);
}

// A broadcast arange made contiguous: `arange(n)[None, :].expand(D, -1).contiguous()` (Mamba's A_log),
// `arange(n)[:, None].expand(-1, m).clone()`, `arange(n).repeat(D, 1)`.
bool broadcast_arange_rule(Tape& tape, const TapeOp& op, uint32_t op_idx, uint32_t S, const ValueInfo& in,
                           const ValueInfo& out, State& st) {
  State src = eval_storage(tape, in.storage, op_idx);
  if (src.opaque || src.segs.size() != 1 || src.dtype != in.dtype || out.dtype != in.dtype || in.storage == S ||
      in.storage_offset != 0)
    return false;
  const Seg& g = src.segs[0];
  const int64_t n = g.end;
  if (g.st.src != Sym::Iota || g.st.period != 0 || g.begin != 0 || g.origin != 0 || n <= 1) return false;
  int64_t repeat = 0;
  if (op.kind == OpKind::RepeatOut) {  // of the 1-D arange: element i is index i % n
    if (in.sizes.size() != 1 || in.sizes[0] != n || in.strides[0] != 1) return false;
  } else {  // the view: one dimension walks the arange with stride 1, every other has stride 0
    int walk = -1;
    for (size_t d = 0; d < in.sizes.size(); ++d) {
      if (in.sizes[d] == 1 || in.strides[d] == 0) continue;
      if (walk >= 0 || in.strides[d] != 1 || in.sizes[d] != n) return false;
      walk = static_cast<int>(d);
    }
    if (walk < 0) return false;
    repeat = 1;
    for (size_t d = static_cast<size_t>(walk) + 1; d < in.sizes.size(); ++d) repeat *= in.sizes[d];
  }
  Sym sy = g.st;
  sy.period = n;
  sy.repeat = repeat > 1 ? repeat : 0;
  fill_whole(st, out, out.dtype, std::move(sy));
  return true;
}

// Out-of-place elementwise ops and casts: a new storage whose state derives from the argument's.
bool unary_rule(Tape& tape, const TapeOp& op, uint32_t op_idx, uint32_t S, const ValueInfo& in, const ValueInfo& out,
                State& st) {
  if (op.kind == OpKind::RepeatOut) return false;
  int64_t b = 0, e = 0;
  if (in.numel != out.numel || in.storage == S || !range_of(in, b, e)) return false;
  State src = eval_storage(tape, in.storage, op_idx);
  if (src.opaque || src.dtype != in.dtype || src.segs.empty() || b < 0 || e > src.segs.back().end) return false;
  // restrict to the argument's elements and renumber from 0
  st = State{};
  st.opaque = false;
  st.dtype = src.dtype;
  st.rng_chain = std::move(src.rng_chain);
  for (Seg& g : src.segs) {
    const int64_t gb = std::max(g.begin, b), ge = std::min(g.end, e);
    if (gb >= ge) continue;
    Seg n = std::move(g);
    n.begin = gb - b;
    n.end = ge - b;
    n.origin -= b;
    st.segs.push_back(std::move(n));
  }
  if (op.kind == OpKind::CloneOut || op.kind == OpKind::ContiguousOut) {
    // a copy: same elements (an RNG segment keeps its op, hence its Philox stream: the clone is
    // bit-identical to its source, as deepcopy semantics require)
    return out.dtype == st.dtype;
  }
  ScalarType new_dtype = st.dtype;
  for (Seg& g : st.segs) {
    Sym& sy = g.st;
    if (sy.src == Sym::Uninit) {
      if (op.kind != OpKind::CastOut) return false;
      new_dtype = out.dtype;
      continue;
    }
    if (sy.src == Sym::Const) {
      if (op.kind == OpKind::CastOut && sy.has_scalar && !sy.cval.defined()) {
        // a dtype cast of a plain constant (`ones(n).to(bf16)`, every norm weight of a model
        // converted with Module.to): exact on the host, no 1-element tensor, no device round trip
        c10::Scalar kept, probe;
        if (stored_value(sy.cscalar, st.dtype, kept) && stored_value(kept, out.dtype, probe)) {
          sy.cscalar = kept;
          new_dtype = out.dtype;
          continue;
        }
      }
      ScalarType dt = st.dtype;
      if (!fold_const(op, sy, dt, /*inplace=*/false) || dt != out.dtype) return false;
      new_dtype = out.dtype;
      continue;
    }
    if (sy.src == Sym::Gather) {
      if (op.kind == OpKind::CastOut) {
        // a cast of the copy (`Module.to(torch.bfloat16)`): the source converted on the host, as ATen
        // converts (round to nearest even); after an epilogue step it would be a second rounding
        if (!sy.epi.empty() || !is_gather_dtype(out.dtype)) return false;
        if (out.dtype != st.dtype) {
          NoInterception guard;
          sy.gsrc = sy.gsrc.to(out.dtype);
        }
        new_dtype = out.dtype;
        continue;
      }
      if (!is_fused_float(st.dtype)) return false;
      // (any other step: as for an RNG source, below)
    }
    if (sy.src == Sym::Band) {
      // a mask cast at the end (`tril(ones(n, n)).bool()`, Module.to(dtype)): both values converted
      // on the host, exactly, as for a constant
      c10::Scalar in_v, out_v;
      if (op.kind != OpKind::CastOut || !stored_value(sy.band_in, out.dtype, in_v) ||
          !stored_value(sy.band_out, out.dtype, out_v))
        return false;
      sy.band_in = in_v;
      sy.band_out = out_v;
      new_dtype = out.dtype;
      continue;
    }
    if (sy.src == Sym::Outer || sy.src == Sym::Sincos) {
      // a table cast at the end (`Module.to(torch.bfloat16)`): rounded once at the store
      if (!(sy.src == Sym::Sincos && op.kind == OpKind::CastOut && st.dtype == ScalarType::Float &&
            is_fused_float(out.dtype)))
        return false;
      new_dtype = out.dtype;
      continue;
    }
    if (sy.src == Sym::Iota) {
      // index programs: everything after the arange runs in fp32 (the kernel's epilogue)
      if (op.kind == OpKind::CastOut) {
        if (out.dtype == st.dtype) continue;
        if (st.dtype == ScalarType::Float && (out.dtype == ScalarType::BFloat16 || out.dtype == ScalarType::Half)) {
          // `inv_freq.to(torch.bfloat16)` (Module.to(dtype) converts floating buffers too): the fp32
          // program, rounded once at the store.  Terminal: nothing folds onto a 16-bit index program
          // (every later elementwise transition asks for fp32).
          new_dtype = out.dtype;
          continue;
        }
        if (!(st.dtype == ScalarType::Long && out.dtype == ScalarType::Float && sy.epi.empty()) ||
            std::fabs(sy.p0) + std::fabs(sy.p1) * static_cast<double>(out.numel) >= 16777216.0)
          return false;
        new_dtype = out.dtype;  // int64 -> fp32 of values below 2^24: exact
        continue;
      }
      // (exp / log / expm1 of an int64 arange promote it to fp32 first, like `/ c` does)
      const bool ssm_unary = op.kind == OpKind::ExpOut || op.kind == OpKind::LogOut || op.kind == OpKind::Expm1Out;
      const double extent = static_cast<double>(sy.period ? sy.period : out.numel);
      if (out.dtype != ScalarType::Float ||
          !(st.dtype == ScalarType::Float ||
            (st.dtype == ScalarType::Long && (op.kind == OpKind::DivOut || op.kind == OpKind::MulOut || ssm_unary) &&
             sy.epi.empty())) ||
          std::fabs(sy.p0) + std::fabs(sy.p1) * extent >= 16777216.0)
        return false;
      // (an int64 arange divided or multiplied by a float is promoted to fp32 first, like ATen does:
      // Whisper's `-c * arange(H)` is float(i) * float(c))
      new_dtype = out.dtype;
    }
    if (op.kind == OpKind::ExpOut || op.kind == OpKind::LogOut || op.kind == OpKind::Expm1Out ||
        op.kind == OpKind::ClampOut) {
      // index programs in fp32 (checked above), RNG programs in their own dtype
      if (sy.src != Sym::Iota && out.dtype != st.dtype) return false;
      const bool ok = op.kind == OpKind::ClampOut
                          ? push_clamp(sy, op)
                          : push_epi(sy, op.kind == OpKind::ExpOut ? TDX_EPI_EXP
                                         : op.kind == OpKind::LogOut ? TDX_EPI_LOG : TDX_EPI_EXPM1, 0);
      if (!ok) return false;
      continue;
    }
    if (op.kind == OpKind::DivOut || op.kind == OpKind::PowScalarOut || op.kind == OpKind::ReciprocalOut) {
      // fp32 only, with the arithmetic of ATen's CUDA kernels: `t / c` multiplies by the reciprocal of
      // c (BinaryDivTrueKernel.cu; div_multiplier), `c ** t` is powf(c, t) (PowKernel.cu), reciprocal
      // is 1.0f / t
      if (out.dtype != ScalarType::Float || (sy.src != Sym::Iota && st.dtype != ScalarType::Float)) return false;
      bool ok = false;
      if (op.kind == OpKind::DivOut) {
        const auto c = scalar_arg(op, 1);
        const size_t pm = find_arg(op, "rounding_mode");
        ok = c && pm == static_cast<size_t>(-1) && push_epi(sy, TDX_EPI_MUL, div_multiplier(*c));
      } else if (op.kind == OpKind::PowScalarOut) {
        const auto base = scalar_arg(op, 0);
        ok = base && *base != 1.0 && push_epi(sy, TDX_EPI_RPOW, *base);
      } else {
        ok = push_epi(sy, TDX_EPI_RECIP, 0);
      }
      if (!ok) return false;
      continue;
    }
    if (sy.src == Sym::Iota && (op.kind == OpKind::MulOut || op.kind == OpKind::AddOut)) {
      bool ok;
      if (op.kind == OpKind::MulOut) {
        const auto c = scalar_arg(op, 1);
        ok = c && push_epi(sy, TDX_EPI_MUL, *c);
      } else {
        const auto p = add_addend(op, false);
        ok = p && push_epi(sy, TDX_EPI_ADD, *p);
      }
      if (!ok) return false;
      continue;
    }
    // RNG source followed by an elementwise op
    if (op.kind == OpKind::CastOut) {
      if (out.dtype == st.dtype) continue;  // a copy
      // fp32 -> bf16/fp16: the values must be exactly `source.to(dtype)` (the fp32 source may be
      // materialised too, e.g. `m.to(torch.bfloat16)` keeps both alive while recording), so the
      // descriptor keeps the fp32 stream/arithmetic and rounds once, at this point of the chain
      if (st.dtype != ScalarType::Float || !(out.dtype == ScalarType::BFloat16 || out.dtype == ScalarType::Half) ||
          sy.wide)
        return false;
      sy.wide = true;
      bool direct = false;  // did the RNG op write the very storage this cast reads?
      for (uint32_t ov : tape.ops[sy.rng_op].outputs) direct |= ov != kNoValue && tape.values[ov].storage == in.storage;
      if (direct) {
        sy.wide_src_storage = in.storage;
        sy.wide_cast_op = op_idx;
      }
      // everything before the cast ran in fp32; the cast itself is the rounding of the last
      // pre-cast step (or of the generated value, if there was none)
      sy.src_noround = !sy.epi.empty();
      for (size_t i = 0; i + 1 < sy.epi.size(); ++i) sy.epi[i].op |= TDX_EPI_NOROUND;
      new_dtype = out.dtype;
      continue;
    }
    if (out.dtype != st.dtype) return false;  // type promotion: not modelled
    bool ok;
    if (op.kind == OpKind::MulOut) {
      const auto c = scalar_arg(op, 1);
      ok = c && push_epi(sy, TDX_EPI_MUL, *c);
    } else if (op.kind == OpKind::NegOut) {
      ok = push_epi(sy, TDX_EPI_MUL, -1.0);
    } else if (op.kind == OpKind::SubOut || op.kind == OpKind::AddOut) {
      const auto p = add_addend(op, op.kind == OpKind::SubOut);
      ok = p && push_epi(sy, TDX_EPI_ADD, *p);
    } else {
      ok = false;  // (every kind admitted above is handled before this point)
    }
    if (!ok) return false;
  }
  if (new_dtype != out.dtype) return false;
  st.dtype = new_dtype;
  return true;
}

// Applies one recorded op whose output lives on the storage being evaluated: the rule of its kind.
void transition(Tape& tape, uint32_t op_idx, uint32_t S, State& st) {
  TapeOp& op = tape.ops[op_idx];
  // the output of this op on S
  uint32_t out_v = kNoValue;
  for (uint32_t v : op.outputs)
    if (v != kNoValue && tape.values[v].storage == S) out_v = v;
  const ValueInfo& out = tape.values[out_v];
  const bool ok = [&] {
    switch (op.kind) {
      case OpKind::Empty: case OpKind::Zeros: case OpKind::Ones: case OpKind::Full: case OpKind::Randn:
      case OpKind::Rand: case OpKind::Arange:
        return factory_rule(tape, op, op_idx, out, st);
      case OpKind::Alias: case OpKind::View: case OpKind::HookVariableData:
      case OpKind::HookSetData:  // `p.data = t`: p now names t's storage; its elements are t's
        return true;  // same elements under another tensor object
      case OpKind::CopyInplace:
        return copy_rule(tape, op, op_idx, S, out, st);
      case OpKind::UniformInplace: case OpKind::NormalInplace: case OpKind::FillInplace: case OpKind::ZeroInplace:
      case OpKind::MulInplace: case OpKind::AddInplace: case OpKind::ErfinvInplace: case OpKind::ClampInplace:
      case OpKind::SubInplace: case OpKind::NegInplace: case OpKind::DivInplace: case OpKind::ExpInplace:
      case OpKind::LogInplace: case OpKind::Expm1Inplace:
        return inplace_rule(tape, op, op_idx, out, st);
      case OpKind::EinsumOut: case OpKind::SinOut: case OpKind::CosOut: case OpKind::CatOut:
        return sincos_transition(tape, op, op_idx, S, out, st);
      case OpKind::TrilOut: case OpKind::TriuOut: case OpKind::TrilInplace: case OpKind::TriuInplace:
      case OpKind::XorOut:
        return band_transition(tape, op, op_idx, S, out, st);
      case OpKind::MulOut: case OpKind::AddOut: case OpKind::CloneOut: case OpKind::CastOut: case OpKind::DivOut:
      case OpKind::PowScalarOut: case OpKind::ReciprocalOut: case OpKind::SubOut: case OpKind::NegOut:
      case OpKind::ExpOut: case OpKind::LogOut: case OpKind::Expm1Out: case OpKind::ClampOut:
      case OpKind::RepeatOut: case OpKind::ContiguousOut: {
        // (the outer product of a position table is a mul of two recorded tensors)
        if (op.kind == OpKind::MulOut && second_is_recorded(op)) return sincos_transition(tape, op, op_idx, S, out, st);
        if (op.inputs.empty() || op.inputs[0].value == kNoValue || !out.covers_storage) return false;
        if (op.kind == OpKind::AddOut && second_is_recorded(op)) return softplus_add_rule(tape, op, op_idx, S, out, st);
        const ValueInfo& in = tape.values[op.inputs[0].value];
        const bool copy = op.kind == OpKind::CloneOut || op.kind == OpKind::ContiguousOut;
        bool broadcast = false;  // a dimension of more than one element with stride 0
        for (size_t d = 0; d < in.sizes.size(); ++d) broadcast |= in.sizes[d] > 1 && in.strides[d] == 0;
        if ((copy && broadcast) || (op.kind == OpKind::RepeatOut && in.numel != out.numel))
          return broadcast_arange_rule(tape, op, op_idx, S, in, out, st);
        return unary_rule(tape, op, op_idx, S, in, out, st);
      }
      default:
        return false;
    }
  }();
  if (!ok) st = make_opaque();
}

bool is_pure_alias(OpKind k) {
  return k == OpKind::Alias || k == OpKind::View || k == OpKind::HookVariableData || k == OpKind::HookSetData;
}

// A reader of an intermediate state does not pin its argument to generic replay if nobody will ever
// have to RUN it: every tensor it produced has a final state the planner can derive symbolically
// (e.g. `original = buf.clone()` followed by `buf.copy_(...)`, `original.copy_(...)`: HF's rotary
// embeddings).  Deriving such a state evaluates the argument as of the reader, never its final state.
thread_local int g_reader_depth = 0;
bool reader_resolves_symbolically(Tape& tape, const TapeOp& op) {
  if (g_reader_depth >= 4) return false;
  struct Depth {
    Depth() { ++g_reader_depth; }
    ~Depth() { --g_reader_depth; }
  } depth;
  for (uint32_t v : op.outputs) {
    if (v == kNoValue) continue;
    const ValueInfo& ov = tape.values[v];
    if (ov.real.defined() || tape.storages[ov.storage].replayed) return false;
    if (eval_storage(tape, ov.storage, static_cast<uint32_t>(tape.ops.size())).opaque) return false;
  }
  return true;
}

}  // namespace

size_t find_arg(const TapeOp& op, const char* name) {
  const auto& args = op.handle->schema().arguments();
  for (size_t i = 0; i < args.size(); ++i)
    if (args[i].name() == name) return i;
  return static_cast<size_t>(-1);
}

State eval_storage(Tape& tape, uint32_t S, uint32_t upto) {
  const StorageInfo& si = tape.storages[S];
  State st;
  bool any = false;
  // index of the last op (< upto) that changes the CONTENT of S (aliases only re-describe it)
  uint32_t last_writer = kNoValue;
  for (uint32_t oi : si.touching_ops) {
    if (oi >= upto) break;
    const TapeOp& op = tape.ops[oi];
    if (is_pure_alias(op.kind)) continue;
    for (uint32_t v : op.outputs)
      if (v != kNoValue && tape.values[v].storage == S) last_writer = oi;
  }
  for (uint32_t oi : si.touching_ops) {
    if (oi >= upto) break;
    const TapeOp& op = tape.ops[oi];
    bool writes = false;
    for (uint32_t v : op.outputs) writes |= (v != kNoValue && tape.values[v].storage == S);
    if (!writes) {
      // A reader that saw an intermediate state which a later op overwrote must run at its own
      // point in history: only generic replay can do that.  (`p.data = t` names p's old storage
      // as an argument but never reads it.)
      if (op.kind != OpKind::HookSetData && !op.done && last_writer != kNoValue && oi < last_writer &&
          !reader_resolves_symbolically(tape, op))
        return make_opaque();
      continue;
    }
    if (op.done && op.kind == OpKind::Generic) return make_opaque();
    any = true;
    transition(tape, oi, S, st);
    if (st.opaque) return st;
  }
  if (!any) return make_opaque();
  return st;
}

bool wide_observable(const Tape& tape, const Sym& sy) {
  if (!sy.wide) return false;
  if (sy.wide_src_storage == kNoValue) return true;
  const StorageInfo& a = tape.storages[sy.wide_src_storage];
  if (a.live > 0 || a.fused_done || a.replayed) return true;
  for (uint32_t oi : a.touching_ops) {
    if (oi == sy.wide_cast_op) continue;
    const TapeOp& op = tape.ops[oi];
    if (op.kind == OpKind::HookSetData) continue;  // `p.data = cast`: names the old storage, never reads it
    bool writes = false;
    for (uint32_t v : op.outputs) writes |= v != kNoValue && tape.values[v].storage == sy.wide_src_storage;
    bool produces = false;  // (metadata queries such as _has_compatible_shallow_copy_type yield no tensor)
    for (uint32_t v : op.outputs) produces |= v != kNoValue;
    if (!writes && produces) return true;  // another reader whose result could be asked for
  }
  return false;
}

// ATen launches a draw as one trivially 1-D iterator with 32-bit indexing when it runs on a contiguous
// tensor with N < 2^31 and 1 + (N - 1) * itemsize < 2^31 (TensorIteratorBase::can_use_32bit_indexing).
std::string aten_draw_refusal(const Tape& tape, const RngChain& chain) {
  constexpr int64_t kMax32 = (int64_t{1} << 31) - 1;
  for (const RngPass& r : chain) {
    const TapeOp& op = tape.ops[r.op];
    const std::string name = op.name();
    if (op.outputs.empty() || op.outputs[0] == kNoValue) return name + " has no recorded result";
    const ValueInfo& v = tape.values[op.outputs[0]];
    const int64_t isz = static_cast<int64_t>(c10::elementSize(v.dtype));
    if (v.numel != r.numel) return name + " drew on a tensor of another size";
    if (v.numel > kMax32 || (v.numel > 0 && (v.numel - 1) > (kMax32 - 1) / isz))
      return name + " of " + std::to_string(v.numel) + " " + c10::toString(v.dtype) +
             " elements needs 64-bit indexing";
    int64_t expect = 1;
    for (size_t k = v.sizes.size(); k-- > 0;) {
      if (v.sizes[k] != 1 && v.strides[k] != expect) return name + " drew through a non-contiguous view";
      expect *= v.sizes[k];
    }
  }
  return "";
}

bool aten_exact_step(uint32_t op) {
  switch (op & 0xffu) {
    case TDX_EPI_MUL: case TDX_EPI_ADD: case TDX_EPI_ERFINV: case TDX_EPI_CLAMP: case TDX_EPI_EXP:
    case TDX_EPI_LOG: case TDX_EPI_EXPM1: case TDX_EPI_INV_SOFTPLUS: case TDX_EPI_MULADD:
      return true;
    default:
      return false;
  }
}

// ---------------------------------------------------------------------------------------------
// lowering: a State as descriptors
// ---------------------------------------------------------------------------------------------
namespace {

int tdx_dtype_of(ScalarType t) {
  switch (t) {
    case ScalarType::Float: return TDX_F32;
    case ScalarType::BFloat16: return TDX_BF16;
    case ScalarType::Half: return TDX_F16;
    default: return -1;
  }
}

// One segment of `st` as a descriptor: everything but dst / elem_begin / elem_count / seed / offset.
// false: the segment is not expressible as one.  `may_sync`: a constant that only exists as a (device)
// tensor may be read back (the materialise path; never the analysis at the end of the recording).
bool lower_seg(const Seg& sg, const State& st, bool may_sync, FastSeg& f) {
  const Sym& sy = sg.st;
  const size_t isz = c10::elementSize(st.dtype);
  f.begin = sg.begin;
  f.end = sg.end;
  f.origin = sg.origin;
  f.sym = &sy;
  TdxInitDesc& d = f.proto;
  std::memset(&d, 0, sizeof(d));
  if (sy.src == Sym::Const) {
    if (!(isz == 1 || isz == 2 || isz == 4 || isz == 8)) return false;
    d.src = TDX_SRC_CONST;
    d.dtype = raw_dtype(isz);
    unsigned char pat[16], one[16];
    size_t got = 0;
    if (!(sy.has_scalar && scalar_bits(sy.cscalar, st.dtype, one, &got) && got == isz)) {
      if (!may_sync) return false;
      Sym tmp = sy;
      ensure_cval(tmp, st.dtype);
      if (!tmp.cval.defined()) return false;
      NoInterception guard;
      std::memcpy(one, tmp.cval.cpu().contiguous().data_ptr(), isz);
    }
    for (size_t i = 0; i < 16; i += isz) std::memcpy(pat + i, one, isz);
    std::memcpy(d.fill_bits, pat, 16);
  } else if (sy.src == Sym::Iota) {
    if (!(tdx_dtype_of(st.dtype) >= 0 || (st.dtype == ScalarType::Long && sy.epi.empty()))) return false;
    EpiSteps epi;
    if (!emit_epi(sy, epi)) return false;
    d.src = TDX_SRC_IOTA;
    d.dtype = st.dtype == ScalarType::Long ? TDX_I64 : static_cast<uint8_t>(tdx_dtype_of(st.dtype));
    d.p0 = sy.p0;
    d.p1 = sy.p1;
    d.fill_bits[0] = static_cast<uint64_t>(sy.period);  // broadcast geometry (0, 0: the plain arange)
    d.fill_bits[1] = static_cast<uint64_t>(sy.repeat);
    d.n_epi = static_cast<uint8_t>(epi.size());
    for (size_t i = 0; i < epi.size(); ++i) d.epi[i] = epi[i];
    f.indexed = true;
  } else if (sy.src == Sym::Sincos) {
    if (tdx_dtype_of(st.dtype) < 0 || sy.epi.size() > TDX_MAX_EPI) return false;
    d.src = TDX_SRC_SINCOS;
    d.dtype = static_cast<uint8_t>(tdx_dtype_of(st.dtype));
    d.p0 = sy.p0;  // the column program
    d.p1 = sy.p1;
    d.fill_bits[0] = static_cast<uint64_t>(sy.half);
    d.fill_bits[1] = sy.cos_first ? TDX_SINCOS_COS_FIRST : 0u;
    d.n_epi = static_cast<uint8_t>(sy.epi.size());
    for (size_t i = 0; i < sy.epi.size(); ++i) d.epi[i] = sy.epi[i];
    f.indexed = true;
  } else if (sy.src == Sym::Gather) {
    EpiSteps epi;
    if (!is_gather_dtype(st.dtype) || !sy.gsrc.defined() || !emit_epi(sy, epi)) return false;
    d.src = TDX_SRC_GATHER;
    d.dtype = st.dtype == ScalarType::Long ? TDX_I64 : static_cast<uint8_t>(tdx_dtype_of(st.dtype));
    d.fill_bits[0] = 0;  // (the device address of the staged source: Batch::flush)
    d.fill_bits[1] = static_cast<uint64_t>(sy.period) | (static_cast<uint64_t>(sy.repeat) << 32);
    d.n_epi = static_cast<uint8_t>(epi.size());
    for (size_t i = 0; i < epi.size(); ++i) d.epi[i] = epi[i];
    f.indexed = true;
    f.gather = sy.gsrc;
  } else if (sy.src == Sym::Band) {
    unsigned char in[16] = {}, outside[16] = {};
    size_t gi = 0, go = 0;
    if (!(isz == 1 || isz == 2 || isz == 4 || isz == 8) || !scalar_bits(sy.band_in, st.dtype, in, &gi) ||
        !scalar_bits(sy.band_out, st.dtype, outside, &go) || gi != isz || go != isz)
      return false;
    d.src = TDX_SRC_BAND;
    d.dtype = raw_dtype(isz);
    d.fill_bits[0] = static_cast<uint64_t>(sy.band_cols) | (static_cast<uint64_t>(sy.band_rows) << 32);
    d.fill_bits[1] = static_cast<uint64_t>(static_cast<uint32_t>(static_cast<int32_t>(sy.band_lo))) |
                     (static_cast<uint64_t>(static_cast<uint32_t>(static_cast<int32_t>(sy.band_hi))) << 32);
    std::memcpy(&d.philox_seed, in, isz);  // (the source draws no random numbers: the two values)
    std::memcpy(&d.philox_offset, outside, isz);
    f.indexed = true;
  } else if (sy.src == Sym::Outer) {
    return false;  // (an intermediate of a table: only the table is a descriptor)
  } else {
    if (tdx_dtype_of(st.dtype) < 0) return false;
    EpiSteps epi;
    if (!emit_epi(sy, epi)) return false;
    f.indexed = true;
    d.src = sy.src == Sym::Uniform ? TDX_SRC_UNIFORM : TDX_SRC_NORMAL;
    d.dtype = static_cast<uint8_t>(tdx_dtype_of(st.dtype));
    d.p0 = sy.p0;
    d.p1 = sy.p1;
    d.n_epi = static_cast<uint8_t>(epi.size());
    for (size_t i = 0; i < epi.size(); ++i) d.epi[i] = epi[i];
    if (sy.src_noround) d.reserved |= TDX_FLAG_SRC_NOROUND;
    f.wide = sy.wide;
    f.rng_slot = kNoValue;
    for (const RngPass& r : st.rng_chain)
      if (r.op == sy.rng_op) f.rng_slot = r.slot;
    if (f.rng_slot == kNoValue) return false;
  }
  return true;
}

}  // namespace

// Lays a state out for emission (StorageTemplate's fast form).  false: some segment is not
// expressible as a descriptor (lower_seg).
bool build_fast(const StorageInfo& si, StorageTemplate& t, bool may_sync) {
  t.fast = false;
  t.segs.clear();
  const State& st = t.st;
  if (st.opaque) return false;
  const size_t isz = c10::elementSize(st.dtype);
  if (isz == 0 || si.nbytes % isz) return false;
  const int64_t numel = static_cast<int64_t>(si.nbytes / isz);
  if (numel == 0 || st.segs.empty() || st.segs.back().end != numel) return false;
  for (const Seg& sg : st.segs) {
    if (sg.st.src == Sym::Uninit) continue;
    FastSeg f;
    if (!lower_seg(sg, st, may_sync, f)) return false;
    t.segs.push_back(std::move(f));
  }
  t.isz = static_cast<uint8_t>(isz);
  t.numel = numel;
  t.fast = true;
  return true;
}

PlanInfo plan_info(const at::Tensor& fake, RngStream rng) {
  PlanInfo info;
  if (!can_materialize(fake)) {
    info.source = "real";
    return info;
  }
  info.deferred = true;
  const auto rec = fake_impl(fake)->record();
  Tape& tape = *rec->tape;
  const ValueInfo& vi = tape.values[rec->value];
  info.dtype = c10::toString(vi.dtype);
  info.numel = vi.numel;
  info.sizes.assign(vi.sizes.begin(), vi.sizes.end());
  info.device = vi.device.str();
  info.requires_grad = fake.is_leaf() && fake.requires_grad();
  const StorageInfo& si = tape.storages[vi.storage];
  if (vi.real.defined() || si.fused_done) {
    info.source = "materialized";
    return info;
  }
  // fold constants where the tensor will live, if that device exists here (a plan built on a
  // machine without a GPU folds 16-bit constant arithmetic with the CPU kernels' rounding)
  FoldOn fold_on(vi.device.is_cuda() && at::hasCUDA() ? vi.device : c10::Device(c10::kCPU));
  State fresh;
  if (!si.tmpl) fresh = eval_storage(tape, vi.storage, static_cast<uint32_t>(tape.ops.size()));
  const State& st = si.tmpl ? si.tmpl->st : fresh;
  static const char* names[] = {"uninit", "const", "uniform", "normal", "iota", "outer", "sincos", "gather", "band"};
  // the epilogue every segment emits (a state-space program that does not compact is replayed; the
  // outer product of a position table, or its sin / cos alone, is never a descriptor)
  std::vector<EpiSteps> emitted(st.segs.size());
  bool fits = true;
  for (size_t i = 0; i < st.segs.size(); ++i)
    fits &= emit_epi(st.segs[i].st, emitted[i]) && st.segs[i].st.src != Sym::Outer;
  if (st.opaque || st.segs.empty() || !fits) {
    info.source = "opaque";
    // best effort: the first op on the storage the planner does not model
    for (uint32_t oi : si.touching_ops) {
      const TapeOp& op = tape.ops[oi];
      if (op.kind == OpKind::Generic) {
        info.first_unfusable_op = op.name();
        break;
      }
    }
    return info;
  }
  const size_t isz = c10::elementSize(st.dtype);
  // the segment that writes the most elements names the tensor's source
  const Seg* main = &st.segs.front();
  for (const Seg& g : st.segs)
    if (g.end - g.begin > main->end - main->begin) main = &g;
  info.source = names[main->st.src];
  // a plan names whole tensors only, and its segments are the descriptors the engine would emit:
  // the analysis's, or each segment lowered now
  info.fusible = !si.replayed && vi.covers_storage && vi.dtype == st.dtype;
  const bool analysed = si.tmpl && si.tmpl->fast;
  size_t next_lowered = 0;
  info.p0 = main->st.p0;
  info.p1 = main->st.p1;
  const EpiSteps& main_epi = emitted[static_cast<size_t>(main - &st.segs.front())];
  info.n_epilogue = static_cast<int>(main_epi.size());
  info.rng_ops = static_cast<int>(st.rng_chain.size());
  info.wide = wide_observable(tape, main->st);
  info.src_noround = main->st.src_noround;
  for (const TdxEpiStep& e : main_epi) info.epilogue.emplace_back(static_cast<int>(e.op), e.a, e.b);
  for (const RngPass& r : st.rng_chain) {
    info.rng_numels.push_back(r.numel);
    info.rng_op_ids.push_back(static_cast<int64_t>((tape.uid << 32) | r.op));
  }
  for (const Seg& g : st.segs) {
    FastSeg own;
    const FastSeg* f = nullptr;
    if (g.st.src != Sym::Uninit) {
      if (analysed) f = &si.tmpl->segs[next_lowered++];
      else if (lower_seg(g, st, /*may_sync=*/true, own)) f = &own;
      else info.fusible = false;
    }
    PlanSegment ps;
    ps.begin = g.begin;
    ps.end = g.end;
    ps.origin = g.origin;
    ps.source = names[g.st.src];
    ps.p0 = g.st.p0;
    ps.p1 = g.st.p1;
    ps.wide = wide_observable(tape, g.st);
    ps.aten_wide = rng == RngStream::Aten && g.st.rng() && g.st.wide;
    ps.src_noround = g.st.src_noround;
    if (g.st.src == Sym::Gather) {
      ps.gather_period = g.st.period;
      ps.gather_repeat = g.st.repeat;
      ps.gather_bytes.assign(static_cast<const char*>(g.st.gsrc.data_ptr()), g.st.gsrc.nbytes());
    } else {
      ps.iota_period = g.st.period;
      ps.iota_repeat = g.st.repeat;
    }
    if (g.st.src == Sym::Sincos) {
      ps.sincos_half = g.st.half;
      ps.sincos_cos_first = g.st.cos_first;
    }
    if (g.st.src == Sym::Band) {
      ps.band_rows = g.st.band_rows;
      ps.band_cols = g.st.band_cols;
      ps.band_lo = g.st.band_lo;
      ps.band_hi = g.st.band_hi;
      if (f) {  // (the two element bit patterns, in the low isz bytes)
        ps.band_in = f->proto.philox_seed;
        ps.band_out = f->proto.philox_offset;
      }
    }
    for (const TdxEpiStep& e : emitted[static_cast<size_t>(&g - &st.segs.front())])
      ps.epilogue.emplace_back(static_cast<int>(e.op), e.a, e.b);
    if (g.st.rng()) {
      for (size_t i = 0; i < st.rng_chain.size(); ++i)
        if (st.rng_chain[i].op == g.st.rng_op) ps.rng_pass = static_cast<int>(i);
    }
    if (g.st.src == Sym::Const && f) {  // (the element's bits, in the low isz bytes of the fill pattern)
      ps.const_bytes.assign(reinterpret_cast<const char*>(f->proto.fill_bits), isz);
      if (&g == main) info.const_bytes = ps.const_bytes;
    }
    info.segments.push_back(std::move(ps));
  }
  if (rng == RngStream::Aten) {  // (the engine's aten_fusible, on the same chain and epilogues)
    static const char* steps[] = {"?", "mul", "add", "erfinv", "clamp", "pow", "reciprocal", "exp", "log", "expm1",
                                  "inverse softplus", "mul+add"};
    info.aten_refusal = aten_draw_refusal(tape, st.rng_chain);
    for (size_t i = 0; i < st.segs.size() && info.aten_refusal.empty(); ++i) {
      if (!st.segs[i].st.rng()) continue;
      for (const TdxEpiStep& e : emitted[i]) {
        if (aten_exact_step(e.op)) continue;
        const uint32_t k = e.op & 0xffu;
        info.aten_refusal = std::string("a draw feeds a ") + (k < 12 ? steps[k] : "?") +
                            " step, which ATen's stream does not compute bit for bit";
        break;
      }
    }
    if (!info.aten_refusal.empty()) info.fusible = false;
  }
  return info;
}

void analyze_tape(Tape& tape) noexcept {
  struct Flag {
    Flag() { g_analysis_only = true; }
    ~Flag() { g_analysis_only = false; }
  } flag;
  const uint32_t n_ops = static_cast<uint32_t>(tape.ops.size());
  for (uint32_t S = 0; S < tape.storages.size(); ++S) {
    StorageInfo& si = tape.storages[S];
    if (si.tmpl || si.fused_done) continue;
    g_analysis_deferred = false;
    try {
      NoInterception guard;
      State st = eval_storage(tape, S, n_ops);
      // constant chains fold with the TARGET device's arithmetic and programs that read a real
      // tensor see its value at materialisation time: both are evaluated then
      if (g_analysis_deferred) continue;
      auto t = std::make_shared<StorageTemplate>();
      t->st = std::move(st);
      build_fast(si, *t, /*may_sync=*/false);
      if (t->fast && si.live > 0) {
        tape.fused_bytes += static_cast<uint64_t>(t->numel) * t->isz;
        tape.fused_storages++;
      }
      si.tmpl = std::move(t);
    } catch (...) {
      // (e.g. uniform_ with from > to: the error is raised when the tensor is materialised)
    }
  }
}

std::vector<std::string> storage_history(const at::Tensor& fake) {
  std::vector<std::string> out;
  if (!can_materialize(fake)) return out;
  const auto rec = fake_impl(fake)->record();
  Tape& tape = *rec->tape;
  const StorageInfo& si = tape.storages[tape.values[rec->value].storage];
  for (uint32_t oi : si.touching_ops) {
    const TapeOp& op = tape.ops[oi];
    std::string line = op.name();
    bool writes = false, covers = true;
    for (uint32_t v : op.outputs)
      if (v != kNoValue && tape.values[v].storage == tape.values[rec->value].storage) {
        writes = true;
        covers = covers && tape.values[v].covers_storage;
      }
    if (is_pure_alias(op.kind)) line += covers ? " [alias]" : " [view]";
    else line += writes ? (covers ? " [writes]" : " [writes part]") : " [reads]";
    out.push_back(line);
  }
  return out;
}

}  // namespace tdx
