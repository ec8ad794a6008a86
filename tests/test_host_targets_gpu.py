"""Host targets on the H100: CPU-offloaded shards built by the kernels and copied to host memory in passes.

Every case compares raw bits with the same call into CUDA targets:
  * InitPlan.materialize(into=) with pinned and pageable CPU buffers -- small Llama and OPT in fp32 and
    bf16 and tests/submission_fuzz.py's mixed-precision module (A_log, causal mask, sinusoids, a host-built
    buffer, inv_freq, padding_idx); whole, shard=(r, W) for W = 2, 3, 8, tensor-parallel placements and
    (dp x tp) blocks; rng "fused" and "aten"; staging of 256 MiB, 1 MiB and a few KiB plus an odd size.
    Generator offsets are equal, and the launch count is the sum over passes of the kernel families each
    pass routes to (tests/submission_fuzz.py's restatement, over the cut the library exports);
  * device memory stays bounded by the staging buffer while a 2 GiB bf16 host shard is built;
  * Llama-3-8B bf16: rank 0 of shard=(0, 8) and rank 5 of its TP=8 plan, into pinned memory;
  * FSDP2 with CPUOffloadPolicy(pin_memory=True / False) on the fake backend's CUDA mesh, dp = 4 and
    (dp, tp) = (2, 4): init_sharded_module fills the CPU shards in place, FSDP2's padding untouched;
  * FSDP1: materialize_flat_shard(out=pinned CPU) with align_numel and a right pad.
"""
import os
import sys

import pytest
import torch
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import submission_fuzz as F  # noqa: E402
from test_fsdp_tp_cpu import MODELS, apply_steps, built, coordinates, fake_rank  # noqa: E402
from torchdistx_b200 import _cabi as C  # noqa: E402
from torchdistx_b200.deferred_init import deferred_init, materialize_module  # noqa: E402
from torchdistx_b200.parallel import tp_placements  # noqa: E402
from torchdistx_b200.plan import _DTYPES, InitPlan, host_staging_bytes, init_sharded_module, shard_range  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGINGS = [256 << 20, 1 << 20, 9001]


def raw(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8).cpu()


def targets(plan, device, pin, **layout):
    """One zeroed buffer per entry, sized for this rank's part: CUDA, or CPU (pinned or pageable)."""
    out = {}
    for e in plan.entries:
        if e.source == "alias":
            continue
        steps = plan._steps(e, layout.get("shard"), layout.get("placements"), layout.get("blocks"))
        n = shard_range(e, steps=steps)[1]
        t = torch.zeros(n, dtype=_DTYPES[e.dtype], device=device)
        out[e.name] = t.pin_memory() if pin else t
    return out


def host_launches(plan, into, staging, aten, **layout):
    """The launches the host submission of `plan` into `into` makes: the families of each pass of the cut."""
    table, _ = plan.descriptors(1, 0, gather_src=lambda g: 1 << 20, device_props=aten, **layout)
    descs = []
    for e, _, ds in table:
        if e.source in ("alias", "value") or into[e.name].device.type != "cpu":
            continue
        for d in ds:
            d.dst = (d.dst or 0) + into[e.name].data_ptr()
            descs.append(d)
    if not descs:
        return None  # (no host submission: the count is the last device submission's)
    pieces, passes = C.host_cut(descs, host_staging_bytes(descs, staging))
    per = [[] for _ in range(passes)]
    for p in pieces:
        per[p.pass_] += [F.spec_of(x) for x in C.piece_descs(descs[p.desc], p, 0)]
    return sum(F.launches(s) for s in per)


def check_plan(plan, pin, staging, **layout):
    aten = None
    if plan.rng == "aten":
        props = torch.cuda.get_device_properties(0)
        aten = (props.multi_processor_count, props.max_threads_per_multi_processor)
    torch.manual_seed(3)
    want = plan.materialize(into=targets(plan, "cuda", False, **layout), **layout)
    off_cuda = torch.cuda.default_generators[0].get_offset()
    into = targets(plan, "cpu", pin, **layout)
    torch.manual_seed(3)
    got = plan.materialize(into=into, staging_bytes=staging, **layout)
    launches = C.load().tdx_last_launch_count()
    assert torch.cuda.default_generators[0].get_offset() == off_cuda
    for k, t in want.items():
        assert got[k].device.type == "cpu" and (got[k].is_pinned() == pin or not got[k].numel()), k
        assert torch.equal(raw(got[k]), raw(t)), (k, layout, staging)
    expect = host_launches(plan, into, staging, aten, **layout)
    assert expect is None or launches == expect, (layout, staging, launches, expect)


def dp_tp_blocks(plan, placements, dp, tp, r):
    """Rank r's (dp x tp) block of each placed parameter: the tensor-parallel chunk, then FSDP2's dim-0 chunk."""
    blocks = {}
    for e in plan.entries:
        if e.kind != "param" or e.source == "alias" or not e.sizes:
            continue
        d = placements.get(e.name)
        steps = [] if d is None else [(d, r % tp, tp)]
        blocks[e.name] = steps + [(0, r // tp, dp)]
        try:
            shard_range(e, steps=blocks[e.name])
        except ValueError:
            blocks[e.name] = [(0, r // tp, dp)]
    return blocks


CASES = [("llama_v11_h12", torch.float32), ("llama_v11_h12", torch.bfloat16), ("opt_v11_h12", torch.float32),
         ("opt_v11_h12", torch.bfloat16), ("mixed", None)]


@pytest.mark.parametrize("case,dtype", CASES)
@pytest.mark.parametrize("rng", ["fused", "aten"])
@pytest.mark.parametrize("pin", [True, False])
def test_plan_into_host_buffers_is_bit_exact(case, dtype, rng, pin):
    if case == "mixed":
        cls = F.mixed_precision_model("cuda")
        build, tp_plan = cls, F.mixed_precision_plan
    else:
        fn, tp_plan_fn = MODELS[case]
        build = lambda: built(fn, dtype, "cuda")
        tp_plan = lambda m: tp_plan_fn()
    module = deferred_init(build)
    plan = InitPlan.from_module(module, rng=rng)
    placements = tp_placements(module, tp_plan(module))
    layouts = [dict(), dict(shard=(1, 2)), dict(shard=(2, 3)), dict(shard=(7, 8)),
               dict(placements=placements), dict(blocks=dp_tp_blocks(plan, placements, 2, 4, 5))]
    for i, layout in enumerate(layouts):
        for staging in STAGINGS if i in (0, 3, 5) else STAGINGS[1:]:
            check_plan(plan, pin, staging, **layout)


def test_device_memory_stays_bounded_by_the_staging_buffer():
    """A 2 GiB bf16 host shard through 64 MiB of staging: the device holds the staging buffer, nothing more."""
    build = lambda: torch.nn.Linear(32768, 32768, bias=False, dtype=torch.bfloat16, device="cuda")
    plan = InitPlan.from_module(deferred_init(build))
    host = torch.empty(32768 * 32768, dtype=torch.bfloat16).pin_memory()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    mem0 = torch.cuda.memory_allocated()
    torch.manual_seed(5)
    plan.materialize(into={"weight": host}, staging_bytes=64 << 20)
    peak = torch.cuda.max_memory_allocated() - mem0
    assert peak <= 64 << 20, peak
    torch.manual_seed(5)
    want = plan.materialize()["weight"]
    assert torch.equal(raw(host), raw(want))


def test_llama3_8b_shards_into_pinned_memory():
    from test_tp_shard_gpu import LLAMA3_8B_PLAN, llama3_8b

    module = deferred_init(llama3_8b)
    plan = InitPlan.from_module(module)
    check_plan(plan, True, 256 << 20, shard=(0, 8))
    placements = tp_placements(module, LLAMA3_8B_PLAN())
    blocks = {k: ([(d, 5, 8)] if d is not None else []) for k, d in placements.items()}
    check_plan(plan, True, 256 << 20, blocks=blocks)


# ------------------------------------------------------------------------- FSDP2 with CPU offload
def _fsdp2_worker(rank, shape, pin, outdir):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    torch.cuda.set_device(0)
    from torch.distributed.fsdp import CPUOffloadPolicy, fully_shard
    from torch.distributed.tensor.parallel import parallelize_module

    from torchdistx_b200.parallel import local_block

    def one(mesh):
        fn, tp_plan = MODELS["llama_v11_h12"]
        build = lambda: built(fn, torch.float32, "cuda")
        plan = InitPlan.from_module(deferred_init(build))
        with torch.device("meta"):
            m = fn()
        names = mesh.mesh_dim_names
        if len(names) > 1:
            parallelize_module(m, mesh["tp"], tp_plan())
        fully_shard(m, mesh=mesh["dp"] if len(names) > 1 else mesh, offload_policy=CPUOffloadPolicy(pin_memory=pin))
        m.to_empty(device="cpu")
        params = dict(m.named_parameters())
        pads = []  # FSDP2's padded shard storage past each local block: a sentinel must survive
        for fp in m._get_fsdp_state()._fsdp_param_group.fsdp_params:
            data, n = fp._sharded_param_data, fp.sharded_param.to_local().numel()
            data[n:].fill_(7)
            pads.append((data, n))
        blocks = {k: local_block(p, k) for k, p in params.items()}
        torch.manual_seed(1)
        init_sharded_module(m, plan)
        torch.manual_seed(1)
        full = deferred_init(build)
        materialize_module(full)
        whole = {k: v.detach() for k, v in list(full.named_parameters()) + list(full.named_buffers())}
        local = lambda p: p.to_local() if hasattr(p, "to_local") else p
        bad = [k for k, p in params.items() if not torch.equal(raw(local(p)), raw(apply_steps(whole[k], blocks[k])))]
        return dict(bad=bad, on_cpu=all(local(p).device.type == "cpu" for p in params.values()),
                    pinned=all(local(p).is_pinned() == pin for p in params.values() if local(p).numel()),
                    pads=all(bool((d[n:] == 7).all()) for d, n in pads))

    if len(shape) == 1:
        from torch.testing._internal.distributed.fake_pg import FakeStore
        import torch.distributed as dist
        from torch.distributed.device_mesh import init_device_mesh

        dist.init_process_group("fake", store=FakeStore(), rank=rank, world_size=shape[0])
        try:
            result = one(init_device_mesh("cuda", shape, mesh_dim_names=("dp",)))
        finally:
            dist.destroy_process_group()
    else:
        result = fake_rank(shape, rank, one, device_type="cuda")
    torch.save(result, os.path.join(outdir, f"rank{rank}.pt"))


@pytest.mark.parametrize("shape", [(4,), (2, 4)])
@pytest.mark.parametrize("pin", [True, False])
def test_fsdp2_cpu_offload_shards_are_filled_in_place(shape, pin, tmp_path):
    mp.spawn(_fsdp2_worker, args=(shape, pin, str(tmp_path)), nprocs=len(coordinates(shape)), join=True)
    for r in coordinates(shape):
        res = torch.load(str(tmp_path / f"rank{r}.pt"))
        assert not res["bad"] and res["on_cpu"] and res["pinned"] and res["pads"], (r, res)


# ------------------------------------------------------------------------------ FSDP1 offload_params
def test_fsdp1_flat_shard_into_pinned_memory():
    from torchdistx_b200.deferred_init import last_materialize_stats, materialize_flat_shard

    def build():
        fn, _ = MODELS["opt_v11_h12"]
        return built(fn, torch.bfloat16, "cuda")

    for world, rank in ((3, 2), (8, 7), (4, 1)):
        torch.manual_seed(9)
        m = deferred_init(build)
        params = [p for _, p in m.named_parameters()]
        want, offs = materialize_flat_shard(params, rank, world, align_numel=8)
        torch.manual_seed(9)
        m = deferred_init(build)
        params = [p for _, p in m.named_parameters()]
        out = torch.full((want.numel(),), 3.0, dtype=torch.bfloat16).pin_memory()
        got, offs2 = materialize_flat_shard(params, rank, world, align_numel=8, out=out)
        st = last_materialize_stats()
        assert got.data_ptr() == out.data_ptr() and offs == offs2
        assert torch.equal(raw(out), raw(want)), (world, rank)
        assert st["host_copies"] > 0 and st["host_bytes"] > 0, st
    with pytest.raises(ValueError, match="CPU `out`"):
        m = deferred_init(build)
        materialize_flat_shard([p for _, p in m.named_parameters()], 0, 2, out=torch.empty(3, dtype=torch.bfloat16))


# ------------------------------------------------------------------------------------- refusals
def test_host_refusals_before_any_launch():
    fn, _ = MODELS["llama_v11_h12"]
    plan = InitPlan.from_module(deferred_init(lambda: built(fn, torch.float32, "cuda")))
    e = next(x for x in plan.entries if x.kind == "param" and len(x.sizes) == 2 and x.source != "alias")
    n = shard_range(e)[1]
    for bad in (torch.zeros(n + 4)[::2][: n], torch.zeros(n - 1), torch.zeros(n, dtype=torch.float64)):
        with pytest.raises(ValueError, match="CPU `into` buffer"):
            plan.materialize(into={e.name: bad})
    lib = C.load()
    dev = torch.zeros(1024, device="cuda")
    staging = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    d = C.make_desc(dev.data_ptr(), dtype=C.TDX_F32, src=C.TDX_SRC_UNIFORM, elem_count=1024)
    arr = (C.TdxInitDesc * 1)(d)
    assert lib.tdx_init_submit_host(arr, 1, staging.data_ptr(), staging.numel(), None) == C.TDX_E_BADARG
    assert b"device memory" in lib.tdx_last_error()
    assert bool((dev == 0).all())
