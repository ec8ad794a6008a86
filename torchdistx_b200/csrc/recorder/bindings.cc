// torchdistx_b200._C -- the native surface behind torchdistx_b200.fake / .deferred_init.
//
// Exports the same 8 functions as the reference's `_C` module
// (reference src/python/torchdistx/_C.pyi:9-16; _C/deferred_init.cc:99-105; _C/fake.cc:40-51):
//   enter_deferred_init, leave_deferred_init, enter_fake_mode, leave_fake_mode, is_fake,
//   can_materialize, materialize_tensor, meta_like
// plus the batched / sharded entry points this engine adds (materialize_tensors, stats,
// philox state access for cross-rank seed agreement).
//
// Python-object fidelity (reference _C/deferred_init.cc:61-95 materializeVariable):
//   * a real tensor is returned unchanged (same object);
//   * a fake tensor materialised twice returns the same Python object;
//   * the result has the Python class of the fake tensor (e.g. torch.nn.Parameter).
// torch 2.11 no longer exposes pyobj_slot()->init_pyobj/check_pyobj, so the class is applied with
// torch.Tensor._make_subclass and identity is kept by caching the wrapped tensor on the tape.
#include <torch/csrc/utils/device_lazy_init.h>
#include <torch/extension.h>

#include <algorithm>
#include <chrono>

#include "fake_tensor.h"
#include "planner.h"
#include "tape.h"
#include "tdx_init.h"

namespace py = pybind11;

namespace {

void py_enter_fake_mode(bool fake_cuda) {
  tdx::enter_fake_mode(fake_cuda);
  // Without a usable CUDA device the Python arg parser would try (and fail) to initialise CUDA for
  // every `device="cuda"` factory call.
  if (fake_cuda && !at::hasCUDA()) torch::utils::set_requires_device_init(at::kCUDA, false);
}

void py_leave_fake_mode() {
  tdx::leave_fake_mode();
  if (!tdx::fake_mode_active() && !at::hasCUDA())
    torch::utils::set_requires_device_init(at::kCUDA, true);
}

tdx::RngStream rng_stream(const std::string& rng) {
  if (rng == "aten") return tdx::RngStream::Aten;
  if (rng != "fused") throw py::value_error("rng must be \"fused\" or \"aten\", got \"" + rng + "\"");
  return tdx::RngStream::Fused;
}

tdx::MaterializeOptions make_options(const py::object& device, const py::object& shard, bool fused,
                                     const std::string& rng = "fused") {
  tdx::MaterializeOptions o;
  o.rng = rng_stream(rng);
  if (!device.is_none()) o.device = py::cast<c10::Device>(device);
  if (!shard.is_none()) {
    auto t = py::cast<std::pair<int64_t, int64_t>>(shard);
    TORCH_CHECK_VALUE(t.second >= 1 && t.first >= 0 && t.first < t.second,
                      "shard must be (rank, world_size) with 0 <= rank < world_size");
    o.shard = tdx::ShardSpec{t.first, t.second};
  }
  o.fused = fused;
  return o;
}

// `out` as a Python object of `like`'s class (no identity bookkeeping: see wrap_like).
py::object wrap_only(const py::handle& like, const at::Tensor& out) {
  PyTypeObject* type = Py_TYPE(like.ptr());
  if (reinterpret_cast<PyObject*>(type) == reinterpret_cast<PyObject*>(THPVariableClass)) return py::cast(out);
  if (reinterpret_cast<PyObject*>(type) == ParameterClass && out.use_count() > 0 &&
      out.unsafeGetTensorImpl()->pyobj_slot()->load_pyobj() == nullptr && !out.grad_fn()) {
    // A fresh leaf that Python has never seen: it can be born a Parameter (what
    // Tensor._make_subclass does, minus the detach() and the trip through the argument parser --
    // a microsecond per tensor, hundreds of tensors per call).
    py::object r = py::reinterpret_steal<py::object>(THPVariable_Wrap(out, type));
    if (!r) throw py::error_already_set();
    return r;
  }
  static py::object make_subclass = py::module_::import("torch").attr("Tensor").attr("_make_subclass");
  return make_subclass(py::reinterpret_borrow<py::object>(reinterpret_cast<PyObject*>(type)), py::cast(out),
                       out.requires_grad());
}

// Gives `out` the Python class of `like` and remembers the result for identity.
py::object wrap_like(const py::handle& like, const at::Tensor& fake, const at::Tensor& out) {
  at::Tensor cached = tdx::cached_python_tensor(fake);
  if (cached.defined()) return py::cast(cached);
  py::object result;
  PyTypeObject* type = Py_TYPE(like.ptr());
  if (reinterpret_cast<PyObject*>(type) == reinterpret_cast<PyObject*>(THPVariableClass)) {
    result = py::cast(out);
  } else if (reinterpret_cast<PyObject*>(type) == ParameterClass && out.use_count() > 0 &&
             out.unsafeGetTensorImpl()->pyobj_slot()->load_pyobj() == nullptr && !out.grad_fn()) {
    // A fresh leaf that Python has never seen: it can be born a Parameter (what
    // Tensor._make_subclass does, minus the detach() and the trip through the argument parser --
    // a microsecond per tensor, hundreds of tensors per call).
    result = py::reinterpret_steal<py::object>(THPVariable_Wrap(out, type));
    if (!result) throw py::error_already_set();
  } else {
    static py::object make_subclass = py::module_::import("torch").attr("Tensor").attr("_make_subclass");
    result = make_subclass(py::reinterpret_borrow<py::object>(reinterpret_cast<PyObject*>(type)),
                           py::cast(out), out.requires_grad());
  }
  tdx::cache_python_tensor(fake, py::cast<at::Tensor>(result));
  return result;
}

py::object py_materialize_tensor(const py::object& var, const py::object& device,
                                 const py::object& shard, bool fused, const std::string& rng) {
  if (!THPVariable_Check(var.ptr())) {
    throw py::type_error(std::string("`var` has to be a `Variable`, but got `") +
                         Py_TYPE(var.ptr())->tp_name + "`.");
  }
  const at::Tensor& t = THPVariable_Unpack(var.ptr());
  if (!tdx::can_materialize(t)) return var;  // real tensors: a no-op returning the same object
  {
    at::Tensor cached = tdx::cached_python_tensor(t);
    if (cached.defined()) return py::cast(cached);
  }
  const tdx::MaterializeOptions opts = make_options(device, shard, fused, rng);
  at::Tensor out;
  {
    py::gil_scoped_release nogil;
    out = tdx::materialize_one(t, opts);
  }
  return wrap_like(var, t, out);
}

py::list py_materialize_tensors(const py::list& vars, const py::object& device,
                                const py::object& shard, bool fused, const py::object& shard_mask,
                                const std::string& rng) {
  std::vector<at::Tensor> fakes;
  fakes.reserve(vars.size());
  for (const py::handle& h : vars) {
    if (!THPVariable_Check(h.ptr()))
      throw py::type_error(std::string("expected a list of tensors, but got `") +
                           Py_TYPE(h.ptr())->tp_name + "`.");
    fakes.push_back(THPVariable_Unpack(h.ptr()));
  }
  const tdx::MaterializeOptions opts = make_options(device, shard, fused, rng);
  // tensors that were already handed out keep their identity and are not touched again
  std::vector<uint8_t> mask_all;
  if (!shard_mask.is_none()) {
    // (True / False, or 1 + the dimension to cut along)
    for (const py::handle& h : py::cast<py::list>(shard_mask)) {
      const int64_t k = PyBool_Check(h.ptr()) ? (h.ptr() == Py_True ? 1 : 0) : py::cast<int64_t>(h);
      TORCH_CHECK_VALUE(k >= 0 && k < 256, "shard_mask entries are bools or 1 + a dimension");
      mask_all.push_back(static_cast<uint8_t>(k));
    }
    TORCH_CHECK_VALUE(mask_all.size() == fakes.size(), "shard_mask must have one flag per tensor");
  }
  std::vector<at::Tensor> todo;
  std::vector<size_t> todo_idx;
  std::vector<uint8_t> mask;
  for (size_t i = 0; i < fakes.size(); ++i) {
    if (tdx::can_materialize(fakes[i]) && !tdx::cached_python_tensor(fakes[i]).defined()) {
      todo.push_back(fakes[i]);
      todo_idx.push_back(i);
      if (!mask_all.empty()) mask.push_back(mask_all[i]);
    }
  }
  std::vector<at::Tensor> done;
  {
    py::gil_scoped_release nogil;
    done = tdx::materialize_many(todo, opts, mask_all.empty() ? nullptr : &mask);
  }
  const auto t0 = std::chrono::steady_clock::now();
  py::list result(fakes.size());
  size_t k = 0;
  for (size_t i = 0; i < fakes.size(); ++i) {
    if (!tdx::can_materialize(fakes[i])) {
      result[i] = vars[i];
    } else if (k < todo_idx.size() && todo_idx[k] == i) {
      result[i] = wrap_like(vars[i], fakes[i], done[k]);
      ++k;
    } else {
      result[i] = py::cast(tdx::cached_python_tensor(fakes[i]));
    }
  }
  tdx::add_wrap_time(std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count());
  return result;
}

// Whole-module entry point: the traversal of materialize_module (children first, then the module's
// own parameters, then its buffers; reference deferred_init.py:104-124) done natively, and streamed:
// every tensor goes to the planner the moment the walk finds it, so the first kernels run while the
// rest of the tree is still being walked (for a 300-tensor model the walk costs ~0.4 ms of host time,
// as much as the kernels of a 1/8 shard).  Results get their Python class and go back into the
// modules' dicts after the last submission -- that part overlaps the GPU too.
struct PendingSlot {
  py::dict dict;  // the module's _parameters or _buffers
  py::object key;
  py::object var;  // the fake tensor object (its Python class is what the result must have)
  at::Tensor fake;
  size_t ticket;  // of the planner's result; kNoTicket: the tensor was handed out before
  // The output the walking thread built itself (PipelinedMaterialize::add), already wearing its Python
  // class; confirmed against the planner's result after the join.
  at::Tensor speculative;
  py::object speculative_wrapped;
};
constexpr size_t kNoTicket = static_cast<size_t>(-1);

void walk_and_feed(const py::handle& module, bool buffers_only, const py::object& check_fn, bool sharded,
                   tdx::PipelinedMaterialize& session, std::vector<PendingSlot>& pending) {
  // interned once: attr("...") would build a Python string per call, three times per module
  static PyObject* const k_modules = PyUnicode_InternFromString("_modules");
  static PyObject* const k_groups[2] = {PyUnicode_InternFromString("_parameters"),
                                        PyUnicode_InternFromString("_buffers")};
  py::dict children = py::reinterpret_steal<py::dict>(PyObject_GetAttr(module.ptr(), k_modules));
  if (!children) throw py::error_already_set();
  std::vector<PyObject*> seen;  // Module.children() yields each distinct child once
  for (auto item : children) {
    if (item.second.is_none()) continue;
    if (std::find(seen.begin(), seen.end(), item.second.ptr()) != seen.end()) continue;
    seen.push_back(item.second.ptr());
    walk_and_feed(item.second, buffers_only, check_fn, sharded, session, pending);
  }
  if (!check_fn.is_none() && !py::cast<bool>(check_fn(module))) return;
  for (int gi = 0; gi < 2; ++gi) {
    const bool is_parameter = gi == 0;
    if (buffers_only && is_parameter) continue;
    py::dict d = py::reinterpret_steal<py::dict>(PyObject_GetAttr(module.ptr(), k_groups[gi]));
    if (!d) throw py::error_already_set();
    for (auto item : d) {
      if (item.second.is_none()) continue;
      if (!THPVariable_Check(item.second.ptr()))
        throw py::type_error(std::string("expected a tensor, but got `") + Py_TYPE(item.second.ptr())->tp_name + "`.");
      const at::Tensor& t = THPVariable_Unpack(item.second.ptr());
      if (!tdx::can_materialize(t)) continue;  // real tensors stay where they are
      PendingSlot p{d, py::reinterpret_borrow<py::object>(item.first),
                    py::reinterpret_borrow<py::object>(item.second), t, kNoTicket, {}, {}};
      // tensors that were already handed out keep their identity and are not touched again
      // (parameters are chunked, buffers replicated -- no isinstance(): which dict it came from says it)
      if (!tdx::cached_python_tensor(t).defined()) {
        p.ticket = session.add(t, /*apply_shard=*/!sharded || is_parameter, &p.speculative);
        if (p.speculative.defined()) p.speculative_wrapped = wrap_only(p.var, p.speculative);
      }
      pending.push_back(std::move(p));
    }
  }
}

void py_materialize_module(const py::object& module, bool buffers_only, const py::object& check_fn,
                           const py::object& device, const py::object& shard, bool fused, const std::string& rng) {
  const tdx::MaterializeOptions opts = make_options(device, shard, fused, rng);
  std::vector<PendingSlot> pending;
  pending.reserve(512);
  std::vector<py::object> wrapped;
  double wrap_us = 0;
  const auto t_walk = std::chrono::steady_clock::now();
  // plans on a helper thread while this one keeps walking
  auto session_ptr = std::make_unique<tdx::PipelinedMaterialize>(opts);
  tdx::PipelinedMaterialize& session = *session_ptr;
  try {
    walk_and_feed(module, buffers_only, check_fn, !shard.is_none(), session, pending);
    session.finish();
    tdx::add_traverse_time(std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_walk).count());
    // Results get their Python identity as they become ready.  Nothing is assigned before every
    // tensor has been planned: a failure leaves the module as it was (the reference's per-tensor loop
    // would leave it half-built).
    wrapped.resize(pending.size());
    for (size_t i = 0; i < pending.size(); ++i) {
      PendingSlot& p = pending[i];
      if (p.ticket == kNoTicket) {
        wrapped[i] = py::cast(tdx::cached_python_tensor(p.fake));
        continue;
      }
      if (p.speculative.defined()) continue;  // wrapped during the walk; confirmed after the join
      at::Tensor out;
      if (session.ready(p.ticket)) {
        out = session.result(p.ticket);
      } else {
        py::gil_scoped_release nogil;  // the helper may need the GIL (Python-level dispatch during a replay)
        out = session.result(p.ticket);
      }
      const auto t0 = std::chrono::steady_clock::now();
      wrapped[i] = wrap_like(p.var, p.fake, out);
      wrap_us += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
    }
    {
      py::gil_scoped_release nogil;
      session.join();
    }
    // the speculative wraps: almost always the planner returned the very tensor the walk had built
    for (size_t i = 0; i < pending.size(); ++i) {
      PendingSlot& p = pending[i];
      if (!p.speculative.defined()) continue;
      at::Tensor out = session.result(p.ticket);
      if (out.unsafeGetTensorImpl() == p.speculative.unsafeGetTensorImpl() && !tdx::cached_python_tensor(p.fake).defined()) {
        tdx::cache_python_tensor(p.fake, py::cast<at::Tensor>(p.speculative_wrapped));
        wrapped[i] = std::move(p.speculative_wrapped);
      } else {
        p.speculative_wrapped = py::object();
        wrapped[i] = wrap_like(p.var, p.fake, out);
      }
    }
    const auto t0 = std::chrono::steady_clock::now();
    // (assignment through the dict, like Module.__setattr__ does for an existing entry)
    for (size_t i = 0; i < pending.size(); ++i) pending[i].dict[pending[i].key] = wrapped[i];
    wrap_us += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
    tdx::add_wrap_time(wrap_us);
  } catch (const c10::ValueError&) {
    // Same wording as the reference's loop (deferred_init.py:104-113), which turns the ValueError of
    // `_C.materialize_tensor(tensor)` into "'<key>' has already been materialized.".
    const size_t bad = session.failed_ticket();
    std::string key;
    for (const PendingSlot& p : pending)
      if (p.ticket == bad && bad != kNoTicket) key = py::cast<std::string>(py::str(p.key));
    {
      py::gil_scoped_release nogil;
      session_ptr.reset();
    }
    if (key.empty()) throw;
    throw py::value_error("'" + key + "' has already been materialized.");
  } catch (...) {
    // the helper may be inside a replay that needs the GIL: never wait for it while holding it
    py::gil_scoped_release nogil;
    session_ptr.reset();
    throw;
  }
  {
    py::gil_scoped_release nogil;
    session_ptr.reset();
  }
  {
    // What the call replaced: ~300 fake Parameter objects (their TensorImpls, meta twins, records) die
    // here, with the GIL, on the calling thread -- a background thread that needs the GIL for them
    // starves the caller the moment it returns to Python (measured: milliseconds).  The recording
    // they kept alive (~3000 recorded call frames for Llama-3-8B, ~0.5 ms of destructors, no Python
    // objects of its own) is handed to the reaper thread.
    std::vector<std::shared_ptr<tdx::Tape>> tapes;
    for (PendingSlot& p : pending) {
      if (!tdx::can_materialize(p.fake)) continue;
      const auto& rec = tdx::fake_impl(p.fake)->record();
      if (rec->tape && (tapes.empty() || tapes.back() != rec->tape) &&
          std::find(tapes.begin(), tapes.end(), rec->tape) == tapes.end())
        tapes.push_back(rec->tape);
    }
    pending.clear();
    wrapped.clear();
    // (a recording nobody else refers to any more: its tensors are released here, under the GIL --
    // see drop_tensor_refs -- and only memory is left for the reaper)
    for (const auto& t : tapes)
      if (t.use_count() == 1) tdx::drop_tensor_refs(*t);
    tdx::release_in_background(std::move(tapes));
  }
}

py::tuple py_materialize_flat_shard(const py::list& vars, int64_t rank, int64_t world, int64_t align_numel,
                                    const py::object& device, const py::object& out, const std::string& rng) {
  std::vector<at::Tensor> fakes;
  fakes.reserve(vars.size());
  for (const py::handle& h : vars) {
    if (!THPVariable_Check(h.ptr()))
      throw py::type_error(std::string("expected a list of tensors, but got `") + Py_TYPE(h.ptr())->tp_name + "`.");
    fakes.push_back(THPVariable_Unpack(h.ptr()));
  }
  const tdx::MaterializeOptions opts = make_options(device, py::none(), true, rng);
  std::optional<at::Tensor> out_t;
  if (!out.is_none()) out_t = py::cast<at::Tensor>(out);
  std::vector<int64_t> offsets;
  at::Tensor shard;
  {
    py::gil_scoped_release nogil;
    shard = tdx::materialize_flat_shard(fakes, opts, rank, world, align_numel, out_t, &offsets);
  }
  return py::make_tuple(shard, offsets);
}

py::dict py_last_stats() {
  const tdx::MaterializeStats s = tdx::last_stats();
  py::dict d;
  d["tensors"] = s.tensors;
  d["fused_tensors"] = s.fused_tensors;
  d["generic_ops"] = s.generic_ops;
  d["narrowed_tensors"] = s.narrowed_tensors;
  d["aten_stream_tensors"] = s.aten_stream_tensors;
  d["host_bytes"] = s.host_bytes;
  d["host_copies"] = s.host_copies;
  d["elided_rng_ops"] = s.elided_rng_ops;
  d["kernel_launches"] = s.kernel_launches;
  d["bytes_written"] = s.bytes_written;
  d["descriptors"] = s.descriptors;
  d["plan_us"] = s.plan_us;
  d["launch_us"] = s.launch_us;
  d["wrap_us"] = s.wrap_us;
  d["traverse_us"] = s.traverse_us;
  d["assign_us"] = s.assign_us;
  d["eval_us"] = s.eval_us;
  d["alloc_us"] = s.alloc_us;
  d["submissions"] = s.submissions;
  d["upload_bytes"] = s.upload_bytes;
  d["first_submit_us"] = s.first_submit_us;
  d["last_submit_us"] = s.last_submit_us;
  d["template_hits"] = s.template_hits;
  d["prebuilt_outputs"] = s.prebuilt_outputs;
  d["deferred_us"] = s.deferred_us;
  d["helper_start_us"] = s.helper_start_us;
  d["helper_done_us"] = s.helper_done_us;
  return d;
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "torchdistx_b200 native runtime (fake tensors, deferred-init tape, fused materialiser)";
  // ---- the reference's 8-function surface --------------------------------------------------
  m.def("enter_deferred_init", &tdx::enter_deferred_init);
  m.def("leave_deferred_init", &tdx::leave_deferred_init);
  m.def("enter_fake_mode", &py_enter_fake_mode, py::arg("fake_cuda") = false);
  m.def("leave_fake_mode", &py_leave_fake_mode);
  m.def("is_fake", [](const at::Tensor& t) { return tdx::is_fake(t); });
  m.def("can_materialize", [](const at::Tensor& t) { return tdx::can_materialize(t); });
  m.def("materialize_tensor", &py_materialize_tensor, py::arg("tensor"),
        py::arg("device") = py::none(), py::arg("shard") = py::none(), py::arg("fused") = true,
        py::arg("rng") = "fused");
  m.def("meta_like", &tdx::meta_like);
  m.def("aten_stream_policy", &tdx::aten_stream_policy, py::arg("numel"), py::arg("sm"), py::arg("tps"));
  // ---- engine additions ------------------------------------------------------------------
  m.def("materialize_tensors", &py_materialize_tensors, py::arg("tensors"),
        py::arg("device") = py::none(), py::arg("shard") = py::none(), py::arg("fused") = true,
        py::arg("shard_mask") = py::none(), py::arg("rng") = "fused");
  m.def("materialize_module", &py_materialize_module, py::arg("module"), py::arg("buffers_only") = false,
        py::arg("check_fn") = py::none(), py::arg("device") = py::none(), py::arg("shard") = py::none(),
        py::arg("fused") = true, py::arg("rng") = "fused");
  m.def("materialize_flat_shard", &py_materialize_flat_shard, py::arg("tensors"), py::arg("rank"), py::arg("world"),
        py::arg("align_numel") = 0, py::arg("device") = py::none(), py::arg("out") = py::none(),
        py::arg("rng") = "fused");
  m.def("plan_info", [](const at::Tensor& t, const std::string& rng) {
    const tdx::PlanInfo i = tdx::plan_info(t, rng_stream(rng));
    py::dict d;
    d["deferred"] = i.deferred;
    d["fusible"] = i.fusible;
    d["source"] = i.source;
    d["dtype"] = i.dtype;
    d["numel"] = i.numel;
    d["p0"] = i.p0;
    d["p1"] = i.p1;
    d["n_epilogue"] = i.n_epilogue;
    d["rng_ops"] = i.rng_ops;
    d["wide"] = i.wide;
    d["src_noround"] = i.src_noround;
    d["first_unfusable_op"] = i.first_unfusable_op;
    d["sizes"] = i.sizes;
    d["device"] = i.device;
    d["requires_grad"] = i.requires_grad;
    d["epilogue"] = i.epilogue;
    d["const_bytes"] = py::bytes(i.const_bytes);
    d["rng_numels"] = i.rng_numels;
    d["rng_op_ids"] = i.rng_op_ids;
    py::list segs;
    for (const tdx::PlanSegment& g : i.segments) {
      py::dict sd;
      sd["begin"] = g.begin;
      sd["end"] = g.end;
      sd["origin"] = g.origin;
      sd["source"] = g.source;
      sd["p0"] = g.p0;
      sd["p1"] = g.p1;
      sd["wide"] = g.wide;
      sd["src_noround"] = g.src_noround;
      sd["epilogue"] = g.epilogue;
      sd["const_bytes"] = py::bytes(g.const_bytes);
      sd["rng_pass"] = g.rng_pass;
      sd["iota_period"] = g.iota_period;
      sd["iota_repeat"] = g.iota_repeat;
      sd["sincos_half"] = g.sincos_half;
      sd["sincos_cos_first"] = g.sincos_cos_first;
      sd["gather_period"] = g.gather_period;
      sd["gather_repeat"] = g.gather_repeat;
      sd["gather_bytes"] = py::bytes(g.gather_bytes);
      sd["band_rows"] = g.band_rows;
      sd["band_cols"] = g.band_cols;
      sd["band_lo"] = g.band_lo;
      sd["band_hi"] = g.band_hi;
      sd["band_in"] = g.band_in;
      sd["band_out"] = g.band_out;
      if (rng == "aten") sd["aten_wide"] = g.aten_wide;
      segs.append(sd);
    }
    d["segments"] = segs;
    if (rng == "aten") d["aten_refusal"] = i.aten_refusal;
    return d;
  }, py::arg("tensor"), py::arg("rng") = "fused");
  m.def("_drain", [] {
    py::gil_scoped_release nogil;  // the helper may need the GIL to let go of Python objects
    tdx::drain_background();
  });
  m.def("_submission_sizes", &tdx::submission_sizes, py::arg("total_bytes"), py::arg("tensors"), py::arg("with_estimate") = true);
  m.def("storage_history", &tdx::storage_history);
  m.def("last_stats", &py_last_stats);
  m.def("last_descriptors", [] { return py::bytes(tdx::last_descriptors()); });
  m.def("kernel_abi_version", [] { return tdx_abi_version(); });
}
