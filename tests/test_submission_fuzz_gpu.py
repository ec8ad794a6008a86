"""Mixed submissions on the H100: a table launched whole equals its descriptors launched one at a time.

For every table tests/submission_fuzz.py draws (random mixes and the forced regimes of the scheduler):
  * arena A, filled with 0xFF, takes the whole table in one submission; arena B, filled with 0xFF, takes
    each descriptor alone, on its direct kernel where it has one (TDX_ALGO_NOLUT).  A must equal B byte
    for byte over the whole arena, gaps and guards included: the union is right, no descriptor writes
    into its neighbour's bytes (they share 16-byte lines across families), and the table kernel, the
    riders and the fallbacks give the direct kernels' bits;
  * the launch count equals the routing restated in submission_fuzz.py (one launch per family);
  * one uploaded plan, launched three times on a side stream with the arena refilled in between, and
    captured once in a CUDA graph and replayed twice, gives A's bytes every time (each kernel puts its
    work counter back to zero as it leaves).  Tables of more than 47 families go through
    tdx_init_launch three times instead: tdx_plan_upload takes one plan;
  * a sample of each table's descriptors is anchored to the CPU restatement (oracle/tdx_oracle.c, through
    submission_fuzz.oracle_bits; copies read the host copy of their source): bit for bit, ATen's stream
    for its unit uniform draws, the normals under the bars of tests/test_kernels_gpu.py, erfinv chains
    within 2 ulp and the state-space steps under the bar of tests/test_ssm_init_cpu.py.
"""
import ctypes
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import submission_fuzz as F  # noqa: E402
from torchdistx_b200 import _cabi as C  # noqa: E402

pytestmark = pytest.mark.gpu

SEEDS = 120  # (about a minute on one H100)
CHUNKS = 8
ANCHORS = 6  # descriptors per table held to the restatement (the first 4096 elements of each)
ANCHOR_ELEMS = 4096
NP_BITS = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def arena(nbytes):
    return torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")


def launch(descs, stream=None):
    """One submission (tdx_init_prepare + submit, as the engine drives it); returns its launch count."""
    stream = stream or torch.cuda.current_stream()
    need = C.prepare(descs)
    ws = torch.empty(max(need, 16), dtype=torch.uint8, device="cuda")
    n = C.submit(ws.data_ptr(), need, stream.cuda_stream)
    return n, ws


def first_diff(a, b):
    bad = (a != b).nonzero()
    return int(bad[0]) if bad.numel() else -1


def owner(t, byte):
    for i, s in enumerate(t.specs):
        if s.off <= byte < s.off + s.nbytes:
            return f"descriptor {i} {s.kw}"
    return "a gap or guard"


def expect_equal(t, got, want, what):
    if not torch.equal(got, want):
        at = first_diff(got, want)
        n = int((got != want).sum())
        raise AssertionError(f"{t.name}: {what}: {n} bytes differ, first at byte {at} ({owner(t, at)})")


def as_f64(bits, dtype):
    if dtype == C.TDX_F32:
        return bits.view(np.float32).astype(np.float64)
    if dtype == C.TDX_BF16:
        return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return bits.view(np.float16).astype(np.float64)


def check_anchor(t, spec, got, want):
    kw = spec.kw
    if F.epi_class(kw) == "ext" and kw["dtype"] != C.TDX_I64:
        # the state-space steps through libdevice against the C library (the bar of tests/test_ssm_init_cpu.py):
        # 4e-6 relative or 1e-5 absolute in fp32, 1 % in bf16 / fp16; NaN and infinities where the other has them
        g, w = as_f64(got, kw["dtype"]), as_f64(want, kw["dtype"])
        fin = np.isfinite(g) & np.isfinite(w)
        assert ((g == w) | (np.isnan(g) & np.isnan(w)) | fin).all(), (t.name, kw)
        g, w = g[fin], w[fin]
        tol = np.maximum(4e-6 * np.abs(w), 1e-5) if kw["dtype"] == C.TDX_F32 else 0.01 * np.abs(w) + 1e-5
        assert (np.abs(g - w) <= tol).all(), (t.name, kw, float(np.abs(g - w).max(initial=0)))
        return
    if any(st[0] == C.TDX_EPI_ERFINV for st in kw.get("epi", ())):
        # erfinvf (libdevice, as ATen's CUDA kernel: tests/test_epilogue_aten_gpu.py) against the restatement's
        # double ndtri: within 2 ulp of the result after the chain
        g, w = as_f64(got, kw["dtype"]), as_f64(want, kw["dtype"])
        ulp = np.abs(np.spacing(np.maximum(np.abs(g), np.abs(w)).astype(np.float32))).astype(np.float64)
        if kw["dtype"] == C.TDX_BF16:
            ulp *= 2.0 ** 16
        elif kw["dtype"] == C.TDX_F16:
            ulp = np.abs(np.spacing(np.maximum(np.abs(g), np.abs(w)).astype(np.float16))).astype(np.float64)
        assert (np.abs(g - w) <= 2 * ulp).all(), (t.name, kw, float(np.abs(g - w).max()))
        return
    if kw["src"] != F.N or F.is_aten(kw):
        same = got == want
        if kw.get("epi") and kw["dtype"] in F.FLOATS:  # (a NaN equals any NaN after a step: tests/test_epilogue_aten_gpu.py)
            same |= np.isnan(as_f64(got, kw["dtype"])) & np.isnan(as_f64(want, kw["dtype"]))
        bad = np.flatnonzero(~same)
        assert not bad.size, f"{t.name}: {kw}: {bad.size} elements off the restatement, first {bad[:4]}: " \
                             f"{got[bad[:4]]} vs {want[bad[:4]]}"
        return
    if kw.get("epi"):
        return  # (a normal through an epilogue: the steps carry the generator's ulp; held to ATen elsewhere)
    # the bars of tests/test_kernels_gpu.py: 16-bit inverse CDF within 1 ulp in <= 0.2 % of the elements;
    # Box-Muller within std * 1e-3 + 2 ulp
    if kw["dtype"] != C.TDX_F32 and F.resolve_algo(kw) == C.TDX_ALGO_ICDF16:
        diff = got.astype(np.int64) - want.astype(np.int64)
        assert np.abs(diff).max(initial=0) <= 1 and (diff != 0).sum() <= max(2, 0.002 * diff.size), (t.name, kw)
        return
    g, w = as_f64(got, kw["dtype"]), as_f64(want, kw["dtype"])
    if kw["dtype"] == C.TDX_BF16:
        ulp = np.abs(w) * 2.0 ** -7
    else:
        ulp = np.abs(np.spacing(w.astype(np.float32 if kw["dtype"] == C.TDX_F32 else np.float16))).astype(np.float64)
    bound = abs(kw["p1"]) * 1e-3 + 2 * ulp
    assert (np.abs(g - w) <= bound).all(), (t.name, kw, float(np.abs(g - w).max()))


def anchor(t, a, host_source, r):
    """Holds a sample of the table's descriptors to the restatement; copies read the host copy of their
    staged source."""
    picks = r.choice(len(t.specs), min(ANCHORS, len(t.specs)), replace=False)
    for i in picks:
        spec = t.specs[int(i)]
        n = min(spec.count, ANCHOR_ELEMS)
        if n == 0:
            continue
        d = spec.desc(0, host_source.ctypes.data, elem_count=n)
        want = F.oracle_bits(spec, d)
        if want is None:
            continue
        isz = F.ISZ[spec.kw["dtype"]]
        got = a[spec.off: spec.off + n * isz].cpu().numpy().view(NP_BITS[isz])
        check_anchor(t, spec, got, want)


def stage_source(t, r):
    """The copies' sources: random bytes (any bits: both arenas run the same copy kernel on them), on the
    host and staged on the device."""
    host = r.integers(0, 256, t.source_bytes, dtype=np.uint8)
    return host, torch.from_numpy(host).cuda()


def check_table(t, r, counts):
    host_source, source = stage_source(t, r)
    A = arena(t.arena_bytes)
    descs = t.descs(A.data_ptr(), source.data_ptr())
    n, ws = launch(descs)
    torch.cuda.synchronize()
    assert n == F.launches(t.specs), f"{t.name}: {n} launches, the routing says {F.launches(t.specs)}"
    B = arena(t.arena_bytes)
    for s in t.specs:
        k, _ = launch([F.alone(s).desc(B.data_ptr(), source.data_ptr())])
        assert k == (1 if s.count else 0), (t.name, s.kw)
    torch.cuda.synchronize()
    expect_equal(t, A, B, "whole table vs one descriptor at a time")
    del B
    # plan reuse, on a side stream
    side = torch.cuda.Stream()
    R = arena(t.arena_bytes)
    rdescs = t.descs(R.data_ptr(), source.data_ptr())
    lib = C.load()
    if F.groups(t.specs) <= F.MAX_GROUPS:
        arr = (C.TdxInitDesc * len(rdescs))(*rdescs)
        ws2 = torch.empty(lib.tdx_init_workspace_bytes(len(rdescs)), dtype=torch.uint8, device="cuda")
        plan = C.TdxPlan()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            C.check(lib.tdx_plan_upload(arr, len(rdescs), ws2.data_ptr(), ws2.numel(), side.cuda_stream,
                                        ctypes.byref(plan)))
            for it in range(3):
                R.fill_(0xFF)
                C.check(lib.tdx_plan_launch(ctypes.byref(plan), ws2.data_ptr(), side.cuda_stream))
                side.synchronize()
                expect_equal(t, R, A, f"plan launch {it}")
        if n:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                C.check(lib.tdx_plan_launch(ctypes.byref(plan), ws2.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))
            for it in range(2):
                R.fill_(0xFF)
                g.replay()
                torch.cuda.synchronize()
                expect_equal(t, R, A, f"graph replay {it}")
            counts["graphs"] = counts.get("graphs", 0) + 1
    else:
        for it in range(3):
            R.fill_(0xFF)
            side.wait_stream(torch.cuda.current_stream())
            n2, _ = launch(rdescs, side)
            side.synchronize()
            assert n2 == n
            expect_equal(t, R, A, f"submission {it} of a table of {F.groups(t.specs)} families")
    del R
    anchor(t, A, host_source, r)
    for tag in t.tags:
        counts[tag] = counts.get(tag, 0) + 1
    counts["tables"] = counts.get("tables", 0) + 1
    counts["descriptors"] = counts.get("descriptors", 0) + len(t.specs)


COUNTS = {}


@pytest.mark.parametrize("chunk", range(CHUNKS))
def test_tables_equal_their_descriptors_alone(chunk):
    per = SEEDS // CHUNKS
    t0 = time.time()
    for seed in range(chunk * per, (chunk + 1) * per):
        r = np.random.default_rng(10_000 + seed)
        # (the forced regimes in every other seed: they are the large tables)
        for t in F.tables(seed, sm=sm_count(), forced=seed % 2 == 0):
            check_table(t, r, COUNTS)
        torch.cuda.empty_cache()
    print(f"chunk {chunk}: {time.time() - t0:.1f} s, {COUNTS}")


def test_the_fuzz_reached_every_regime():
    """(after the chunks) every forced regime ran, and wide tables went through two plans"""
    if not COUNTS:
        pytest.skip("the chunks did not run in this process")
    for tag in ("random", "table-below", "table-at", "riders-at", "riders-above", "preassigned-below",
                "preassigned-at", "static-grabs", "one", "families-47", "wide", "every-row"):
        assert COUNTS.get(tag, 0) > 0, (tag, COUNTS)
    assert COUNTS.get("graphs", 0) > 0, COUNTS


def named_slots(m, dims):
    """The engine's slots of `m` under the layouts `dims`, each with its parameter or buffer name."""
    from torchdistx_b200.deferred_init import _tp_slots

    names = {}
    for n, t in list(m.named_buffers()) + list(m.named_parameters()):
        names.setdefault(id(t), n)
    slots, unique, make = _tp_slots(m, dims)
    return [names[id(slots[i][3])] for i in unique], unique, make


def each_tensor(build, rng):
    """{name: tensor} of every parameter and buffer, each built alone by materialize_tensor (one
    submission per tensor), from the recording of seed 1."""
    from torchdistx_b200.deferred_init import deferred_init, materialize_tensor

    torch.manual_seed(1)
    m = deferred_init(build)
    out = {}
    for n, t in list(m.named_parameters()) + list(m.named_buffers()):
        out.setdefault(n, materialize_tensor(t, rng=rng).detach())
    return out


def raw(t):
    return t.contiguous().view(torch.uint8).reshape(-1)


@pytest.mark.parametrize("rng", ["fused", "aten"])
def test_a_tensor_parallel_submission_of_more_than_47_families(rng):
    """Through the public API: a mixed-precision module whose Colwise/Rowwise blocks need 55 kernel families
    in one submission in the default stream (every direct generator family and every window family, the fp32
    draws cast with .to() among them), and the same module on ATen's stream.  Every rank's block of every
    parameter and buffer -- the engine's tensor-parallel call, and InitPlan -> JSON -> materialize(shard=,
    placements=) -- equals the same tensor built alone by materialize_tensor and sliced, bit for bit."""
    from test_tp_shard_cpu import block
    from torchdistx_b200.deferred_init import deferred_init, last_descriptors, last_materialize_stats
    from torchdistx_b200.parallel import tp_placements
    from torchdistx_b200.plan import InitPlan

    build = F.mixed_precision_model()
    alone = each_tensor(build, rng)
    assert {"mask", "sinus", "host", "inv_freq", "A_log", "emb.weight"} <= set(alone)
    assert any(n.endswith(".master") for n in alone)
    assert not alone["emb.weight"][0].view(torch.int16).any()
    world = 4
    for r in range(world):
        torch.manual_seed(1)
        m = deferred_init(build)
        dims = tp_placements(m, F.mixed_precision_plan(m))
        names, unique, make = named_slots(m, dims)
        done = make(torch.device("cuda"), r, world, rng=rng)
        got = dict(zip(names, (done[i] for i in unique)))
        st = last_materialize_stats()
        assert st["submissions"] == 1 and st["generic_ops"] == 0, st
        if rng == "fused":  # (one submission: its descriptors are last_descriptors())
            spans = F.groups([F.spec_of(d) for d in last_descriptors()])
            assert spans > F.MAX_GROUPS and st["kernel_launches"] == spans, (spans, st)
        torch.manual_seed(1)
        ip = InitPlan.from_module(deferred_init(build), rng=rng)
        path = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"tdx_mixed_plan_{os.getpid()}.json")
        ip.save(path)
        mine = InitPlan.load(path).materialize(shard=(r, world), placements=dims)
        os.remove(path)
        # (the engine leaves the host-built buffer alone: it is a real tensor already, not a recording)
        assert set(got) <= set(alone) and set(alone) - set(got) == {"host"} and set(alone) <= set(mine), \
            (set(alone) ^ set(got), set(alone) - set(mine))
        for k, t in alone.items():
            want = raw(block(t, world, r, dims.get(k)))
            if k in got:
                assert torch.equal(raw(got[k]), want), (k, r)
            assert torch.equal(raw(mine[k]), want), (k, r)

