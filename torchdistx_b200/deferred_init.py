"""Deferred module initialisation with a GPU-native materialiser.

Drop-in for ``torchdistx.deferred_init`` (reference src/python/torchdistx/deferred_init.py:19-124):
``deferred_init``, ``is_deferred``, ``materialize_tensor`` and ``materialize_module`` keep their
signatures, traversal order, return values and errors.

What differs is underneath ``materialize_*``.  The reference calls ``_C.materialize_tensor`` once
per tensor and each call replays the recorded aten ops one by one through the dispatcher
(reference deferred_init.py:104-113 -> deferred_init.cc:506-528).  Here ``materialize_module``
collects every tensor of the module tree (same order: children first, then the module's own
parameters, then its buffers) and hands the whole list to the native engine, which folds each
tensor's recorded program into one fused descriptor and runs all of them with a handful of
sm_90a kernel launches (``include/tdx_init.h``).  The extra keyword-only arguments select the
target device and dim-0 sharding:

    materialize_module(m, device="cuda")                       # recorded on cpu, built on the GPU
    materialize_module(m, device="cuda", shard=(rank, world))  # each rank builds only its rows
    materialize_module(m, device_mesh=tp_mesh, parallelize_plan=plan)  # tensor-parallel blocks
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple, TypeVar, Union

import torch
from torch import Tensor
from torch.nn import Module

import atexit

from . import _C
from . import fake  # noqa: F401  (installs the fake-aware Tensor.__repr__)

# materialize_module leaves the teardown of a finished recording to the engine's helper thread;
# it must be done with Python objects before the interpreter goes away
atexit.register(_C._drain)



def _install_value_readers() -> None:
    """``Tensor.item()`` on a deferred tensor materialises it and goes on recording (it is an operator:
    the native handler sees it).  ``tolist()`` and ``numpy()`` read memory directly and never reach
    the dispatcher, so a constructor that computes hyper-parameters from a tensor -- stochastic-depth
    rates, ``torch.linspace(0, rate, depth).tolist()`` in ConvNeXt / Swin / timm-style models -- fails
    under the reference with "Cannot access data pointer of Tensor that doesn't have storage".  Here
    they behave like ``item()``: the value is needed now, so the tensor is built now."""
    for name in ("tolist", "numpy"):
        original = getattr(torch.Tensor, name)
        if getattr(original, "_tdx_deferred_aware", False):
            continue

        def reader(self, *args, _original=original, **kwargs):
            if _C.can_materialize(self):
                self = _C.materialize_tensor(self, None, None)
            return _original(self, *args, **kwargs)

        reader._tdx_deferred_aware = True  # type: ignore[attr-defined]
        reader.__name__, reader.__doc__ = name, original.__doc__
        setattr(torch.Tensor, name, reader)


_install_value_readers()

__all__ = [
    "deferred_init",
    "is_deferred",
    "materialize_tensor",
    "materialize_module",
    "materialize_flat_shard",
    "last_materialize_stats",
    "last_descriptors",
    "plan_report",
]

M = TypeVar("M", bound=Module)
DeviceLike = Union[str, torch.device, None]
Shard = Optional[Tuple[int, int]]


def deferred_init(module_fn: Callable[..., M], *args, **kwargs) -> M:
    """Runs ``module_fn(*args, **kwargs)`` with every tensor fake and every operation recorded.

    The returned module owns no memory; build it later with :func:`materialize_module` or
    :func:`materialize_tensor`.  Operations performed on the module after this function returns
    are not recorded.
    """
    _C.enter_deferred_init()
    try:
        return module_fn(*args, **kwargs)
    finally:
        _C.leave_deferred_init()


def is_deferred(obj: Union[Tensor, Module]) -> bool:
    """``True`` if the tensor -- or any parameter or buffer of the module -- still awaits
    materialisation."""
    if isinstance(obj, Tensor):
        return _C.can_materialize(obj)
    if isinstance(obj, Module):
        return any(_C.can_materialize(t) for t in obj.parameters()) or any(
            _C.can_materialize(t) for t in obj.buffers()
        )
    raise ValueError("`obj` must be of type `Tensor` or `Module`.")


def _device(device: DeviceLike) -> Optional[torch.device]:
    return None if device is None else torch.device(device)


def materialize_tensor(tensor: Tensor, *, device: DeviceLike = None, shard: Shard = None, rng: str = "fused") -> Tensor:
    """Materialises ``tensor``; a real tensor is returned unchanged.

    Repeated calls return the same tensor object (the recording keeps a reference to it, so drop
    the fake tensor when it is no longer needed).  ``rng``: see :func:`materialize_module`.
    """
    return _C.materialize_tensor(tensor, _device(device), shard, True, rng)


def materialize_module(
    module: Module,
    buffers_only: bool = False,
    check_fn: Optional[Callable[[Module], bool]] = None,
    *,
    device: DeviceLike = None,
    shard: Shard = None,
    device_mesh=None,
    as_dtensor: bool = False,
    parallelize_plan: Optional[Dict[str, object]] = None,
    rng: str = "fused",
) -> None:
    """Materialises ``module`` and its descendants in place.

    Args:
        module: the module to materialise.
        buffers_only: materialise buffers only, leave parameters fake.
        check_fn: called with every (sub)module; modules for which it returns ``False`` are
            skipped (their children are still visited).
        device: build the tensors on this device instead of the recorded one.
        shard: ``(rank, world_size)``: build only this rank's ``torch.chunk(..., dim=0)`` slice of
            every parameter (buffers and 0-dim tensors are replicated).  All ranks must hold the
            same generator state; see :func:`torchdistx_b200.parallel.sync_rng`.
        device_mesh: a 1-D ``torch.distributed.device_mesh.DeviceMesh``: shorthand for
            ``shard=(mesh.get_local_rank(), mesh.size())`` on this rank's device of the mesh, with the
            generator state agreed over the mesh's process group first (the path's one collective,
            16 bytes).  The layout is FSDP2's / DTensor's ``Shard(0)``
            ($TORCH/distributed/fsdp/_fully_shard/_fsdp_param.py:381-402).
        as_dtensor: with ``device_mesh``: wrap every dim-0-sharded parameter as a
            ``DTensor(mesh, [Shard(0)])`` over its local chunk (no copy, no communication).
        parallelize_plan: with ``device_mesh``: the dict ``torch.distributed.tensor.parallel.
            parallelize_module`` takes.  Every parameter the plan reaches is built as this rank's
            block of the placement the plan gives it (:func:`torchdistx_b200.parallel.tp_placements`:
            ``Shard(0)``, ``Shard(1)`` or ``Replicate()``) and comes back as a ``DTensor`` with the
            global shape and stride, so ``parallelize_module(module, device_mesh, plan)`` then keeps
            it as it is.  Other parameters and all buffers are built whole and stay plain tensors.
        rng: ``"fused"`` (default): random tensors on CUDA are drawn from the engine's own Philox
            layout -- the reference's distributions, other bits.  ``"aten"``: from ATen's own CUDA
            stream -- the bits an eager ``normal_``/``uniform_`` (and the reference's replay) gives
            after the same ``torch.manual_seed``, and the same generator offsets; draws the kernels
            cannot reproduce bit for bit (64-bit or non-contiguous iterators, other epilogue steps)
            are replayed through ATen in their place.  CPU-device tensors always take ATen's mt19937
            stream, whatever ``rng`` says.
    """
    if rng not in ("fused", "aten"):
        raise ValueError(f'materialize_module: rng must be "fused" or "aten", got {rng!r}')
    if parallelize_plan is not None:
        _materialize_tp(module, buffers_only, check_fn, device, shard, device_mesh, parallelize_plan, rng)
        return
    if device_mesh is not None:
        from . import parallel

        if device_mesh.ndim != 1:
            raise ValueError("materialize_module: `device_mesh` must be 1-D (pass the mesh dimension to shard over)")
        if shard is not None:
            raise ValueError("materialize_module: pass either `shard` or `device_mesh`")
        shard = (device_mesh.get_local_rank(), device_mesh.size())
        if device is None and device_mesh.device_type == "cuda":
            device = torch.device("cuda", torch.cuda.current_device())
        parallel.sync_rng(device if device is not None else torch.device(device_mesh.device_type),
                          group=device_mesh.get_group())
    elif as_dtensor:
        raise ValueError("materialize_module: `as_dtensor` needs a `device_mesh`")
    shapes = None
    if as_dtensor:
        shapes = {id(mod): {k: (tuple(p.shape), tuple(p.stride())) for k, p in mod._parameters.items()
                            if p is not None and _C.can_materialize(p)} for mod in module.modules()}
    # (a ValueError raised while a tensor is materialised comes back as the reference words it,
    # deferred_init.py:110-113: "'<key>' has already been materialized."; others pass unchanged)
    _C.materialize_module(module, buffers_only, check_fn, _device(device), shard, True, rng)
    if as_dtensor and not buffers_only:
        from torch.distributed.tensor import DTensor, Shard

        for mod in module.modules():
            for k, (shape, stride) in shapes.get(id(mod), {}).items():
                p = mod._parameters[k]
                if len(shape) == 0 or isinstance(p, DTensor) or _C.can_materialize(p):
                    continue  # 0-dim parameters are replicated; skipped modules (check_fn) are still fake
                dt = DTensor.from_local(p.detach(), device_mesh, [Shard(0)], run_check=False, shape=torch.Size(shape),
                                        stride=stride)
                mod._parameters[k] = torch.nn.Parameter(dt, requires_grad=p.requires_grad)


def _materialize_tp(module, buffers_only, check_fn, device, shard, device_mesh, plan, rng="fused") -> None:
    from torch.distributed.tensor import DTensor, Replicate, Shard

    from . import parallel

    if device_mesh is None or device_mesh.ndim != 1:
        raise ValueError(f"materialize_module({type(module).__name__}): `parallelize_plan` needs a 1-D `device_mesh`")
    if shard is not None:
        raise ValueError(f"materialize_module({type(module).__name__}): pass either `shard` or `parallelize_plan`")
    dims = parallel.tp_placements(module, plan)
    if device is None and device_mesh.device_type == "cuda":
        device = torch.device("cuda", torch.cuda.current_device())
    slots, unique, prepared = _tp_slots(module, dims, buffers_only, check_fn)
    parallel.sync_rng(device if device is not None else torch.device(device_mesh.device_type),
                      group=device_mesh.get_group())
    done = prepared(device, device_mesh.get_local_rank(), device_mesh.size(), rng)
    for i in unique:
        name, t = slots[i][2], slots[i][3]
        if name in dims:
            placement = Replicate() if dims[name] is None else Shard(dims[name])
            dt = DTensor.from_local(done[i].detach(), device_mesh, [placement], run_check=False,
                                    shape=t.shape, stride=t.stride())
            done[i] = torch.nn.Parameter(dt, requires_grad=t.requires_grad)
    first = {id(slots[i][3]): i for i in unique}
    for group, key, _, t in slots:
        group[key] = done[first[id(t)]]


def _tp_slots(module, dims, buffers_only=False, check_fn=None):
    """The tensors ``materialize_module(parallelize_plan=...)`` builds, in its traversal order (children
    first, each once, then own parameters, then buffers): ``(slots, unique, build)``.  ``slots`` are
    ``(dict, key, parameter name or "", fake tensor)``; ``unique`` the slots that build a tensor (a tied
    parameter is built once, with its names' one layout); ``build(device, rank, world)`` runs the one
    engine call and returns ``{slot: local tensor}``."""
    slots: List[Tuple[dict, str, str, Tensor]] = []

    def walk(mod: Module, prefix: str) -> None:
        seen = set()
        for cname, child in mod._modules.items():
            if child is not None and id(child) not in seen:
                seen.add(id(child))
                walk(child, f"{prefix}{cname}.")
        if check_fn is not None and not check_fn(mod):
            return
        groups = (mod._buffers,) if buffers_only else (mod._parameters, mod._buffers)
        for group in groups:
            for key, t in group.items():
                if t is not None and _C.can_materialize(t):
                    slots.append((group, key, prefix + key if group is mod._parameters else "", t))

    walk(module, "")
    first: Dict[int, int] = {}
    mask = []
    for i, (_, _, name, t) in enumerate(slots):
        dim = dims.get(name)
        if dim is not None and not t.is_contiguous():
            raise ValueError(f"materialize_module: '{name}' is not contiguous; a Shard({dim}) block needs a "
                             "row-major parameter")
        j = first.setdefault(id(t), i)
        other = slots[j][2]
        if j != i and name in dims and other in dims and dims[other] != dim:
            lay = lambda d: "Replicate()" if d is None else f"Shard({d})"
            raise ValueError(f"materialize_module: '{other}' and '{name}' are one tied parameter, but the plan "
                             f"gives them {lay(dims[other])} and {lay(dim)}")
        mask.append(0 if dim is None else 1 + dim)
    unique = sorted(set(first.values()))

    def build(device, rank, world, rng="fused"):
        return dict(zip(unique, _C.materialize_tensors([slots[i][3] for i in unique], _device(device), (rank, world),
                                                       True, [mask[i] for i in unique], rng)))

    return slots, unique, build


def materialize_flat_shard(
    params: Sequence[Tensor],
    rank: int,
    world_size: int,
    *,
    device: DeviceLike = None,
    align_numel: int = 0,
    out: Optional[Tensor] = None,
    rng: str = "fused",
) -> Tuple[Tensor, List[int]]:
    """FSDP1's layout: this rank's chunk of the ``FlatParameter`` the deferred ``params`` form.

    The parameters are (virtually) flattened and concatenated in order -- each start aligned to
    ``align_numel`` elements when > 1, as ``FlatParamHandle`` does under ``use_orig_params`` -- the
    flat vector is chunked ``world_size`` ways like ``torch.chunk`` and the last chunk right-padded
    with zeros ($TORCH/distributed/fsdp/_flat_param.py ``_get_shard``; alignment gaps are written as
    zeros too, where ``FlatParamHandle`` puts its debug value 42 -- elements nothing reads;
    tests/test_fsdp1_caller_gloo.py compares the layout with PyTorch's own functions).  Rank ``rank``'s chunk is
    written by the kernels straight into one 1-D tensor (``out`` if given, e.g. the handle's
    ``flat_param._local_shard``); neither the parameters nor the flat parameter exist unsharded at
    any time.  Returns ``(local_shard, offsets)``: ``offsets[i]`` is the start of ``params[i]`` in
    the flat parameter, ``offsets[-1]`` its unpadded total.

    ``out`` may be a CPU tensor, pinned or pageable: FSDP1's ``_local_shard`` under
    ``CPUOffload(offload_params=True)``.  The chunk is still built on the parameters' CUDA device and
    copied to host memory in passes through a bounded staging buffer (``tdx_init_submit_host``), with
    the bits a CUDA ``out`` gets; the call returns once ``out`` holds them.  ``last_materialize_stats()``
    counts the bytes and copies as ``host_bytes`` and ``host_copies``.

    The parameters stay deferred; all ranks must hold the same generator state
    (:func:`torchdistx_b200.parallel.sync_rng`) and pass the same list.  ``rng``: see
    :func:`materialize_module`.
    """
    shard, offsets = _C.materialize_flat_shard(list(params), rank, world_size, align_numel, _device(device), out, rng)
    return shard, list(offsets)


def plan_report(module: Module) -> Dict[str, Dict[str, object]]:
    """What the planner will do with every parameter / buffer of a deferred module, without
    allocating or launching anything (works on a machine without a GPU): per tensor name,
    ``{"fusible", "source" (uninit|const|uniform|normal|opaque|real|materialized), "dtype", "numel",
    "p0", "p1", "n_epilogue", "rng_ops", "first_unfusable_op"}``."""
    out: Dict[str, Dict[str, object]] = {}
    for name, t in list(module.named_parameters()) + list(module.named_buffers()):
        out[name] = dict(_C.plan_info(t))
    return out


def last_descriptors():
    """The `TdxInitDesc` table the last ``materialize_*`` call on this thread submitted to the
    kernels, as a ctypes array (see ``include/tdx_init.h``)."""
    from . import _cabi

    raw = _C.last_descriptors()
    n = len(raw) // 128
    return (_cabi.TdxInitDesc * n).from_buffer_copy(raw)


def last_materialize_stats() -> Dict[str, int]:
    """Counters of the last ``materialize_*`` call on this thread (fused tensors, generic ops
    replayed, dead RNG passes elided, kernel launches, bytes written)."""
    return dict(_C.last_stats())
