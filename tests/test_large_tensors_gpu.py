"""Tensors past 2^31 elements and 4 GiB on the H100: every kernel family against its own small pieces.

A 32-bit product or a truncated division anywhere on the way from a descriptor to a store would give a
tensor whose first 2 GiB are right.  So every case of tests/test_large_tensors_cpu.py (one descriptor per
kernel family row, ATen's stream aside, each past 2^31 local elements and 2^32 bytes where its element
size allows, with an unaligned start and destination) is:
  * launched alone as one submission, into a buffer filled with 0xFF; the launch count equals
    tests/submission_fuzz.py's routing, and the bytes around the destination are untouched;
  * (a) regenerated in pieces of at most 2^27 elements at the same global elements -- each launched alone,
    on the direct kernel where the family has one (TDX_ALGO_NOLUT), into a scratch buffer at the same
    address mod 16 -- and every piece must equal its slice of the large buffer byte for byte.  A window's
    pieces are the host cut's own (tdx_init_host_piece_descs: a partial first run, whole runs windowed, a
    partial last run);
  * (b) held at local elements 0, 2^31 - 2048, the elements holding bytes 2^31 and 2^32, and the last 4096
    elements, to the C restatement under the bars of tests/test_submission_fuzz_gpu.py (check_anchor),
    and the 16-bit generators without an epilogue also to the float64 value of each element's Philox
    half-word (tests/generator_domain.py).
Then one mixed table of three descriptors past 2^31 elements and small riders, in one submission; ATen's
stream through materialize_module (a bf16 normal_ of 2^31 + 5 elements is replayed, a fused uniform_
follows); one large parameter against its shard=(r, 16) materialisations; FSDP1's flat shard of
Llama-3-70B against world-64 shards and into pinned memory; and InitPlan's offloaded shard of the same
model into pinned memory against the same call into HBM.

Every case checks free device (and, for pinned targets, host) memory first and skips, naming the bytes it
needs, when there is not enough.
"""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import generator_domain as G  # noqa: E402
import philox_torch as PT  # noqa: E402
import submission_fuzz as F  # noqa: E402
import test_large_tensors_cpu as L  # noqa: E402
from test_submission_fuzz_gpu import check_anchor  # noqa: E402
from torchdistx_b200 import _cabi as C  # noqa: E402

pytestmark = pytest.mark.gpu

PIECE = 1 << 27  # elements of a piece (at most)
SCRATCH = 256 << 20
ANCHOR = 4096
SLACK = 1 << 30  # device memory a case leaves free for the allocator, workspaces and the comparison
TORCH_DT = {C.TDX_BF16: torch.bfloat16, C.TDX_F16: torch.float16}


def need_device(nbytes):
    free = torch.cuda.mem_get_info()[0]
    if free < nbytes + SLACK:
        pytest.skip(f"needs {nbytes + SLACK} bytes of free device memory, {free} free")


def need_host(nbytes):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
    from offload_bench import host_bytes_available

    have = host_bytes_available()
    if have < nbytes + (4 << 30):
        pytest.skip(f"needs {nbytes + (4 << 30)} bytes of available host memory, {have} available")


@pytest.fixture(autouse=True)
def _release():
    yield
    torch.cuda.synchronize()
    print(f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    torch.cuda.reset_peak_memory_stats()
    torch.cuda.empty_cache()


def submit(descs):
    need = C.prepare(descs)
    ws = torch.empty(max(need, 16), dtype=torch.uint8, device="cuda")
    n = C.submit(ws.data_ptr(), need, torch.cuda.current_stream().cuda_stream)
    return n, ws


class Anchored:
    """What check_anchor reads of a table: its name."""

    def __init__(self, name):
        self.name = name


def anchors(count, head, isz):
    at = {0, (1 << 31) - 2048, ((1 << 31) - head) // isz, ((1 << 32) - head) // isz, count - ANCHOR}
    return sorted({min(max(0, a), max(0, count - ANCHOR)) for a in at if a < count})


def piece_descs(case, d, a, n, scratch):
    """The descriptors that write local elements [a, a + n) of `d` into `scratch` at the same address mod 16
    (a window's: the host cut's own pieces), each on the direct kernel where the family has one."""
    isz = case.isz
    shift = (d.dst + a * isz) % 16
    p = C.TdxHostPiece(0, 0, a, n, shift)
    parts = C.piece_descs(d, p, scratch)
    for x in parts:
        if x.src in (F.U, F.N) and not F.is_aten(dict(algo=int(x.algo))):
            x.algo |= C.TDX_ALGO_NOLUT
    return parts, shift


def check_pieces(case, d, big, base_off, scratch, name):
    """Reference (a): every local element of `d` (at byte base_off of `big`) equals its small piece."""
    isz, count = case.isz, int(d.elem_count)
    per = min(PIECE, SCRATCH // isz - 16)
    for a in range(0, count, per):
        n = min(per, count - a)
        scratch.fill_(0)
        parts, shift = piece_descs(case, d, a, n, scratch.data_ptr())
        submit(parts)
        got = big[base_off + a * isz: base_off + (a + n) * isz]
        want = scratch[shift: shift + n * isz]
        if not torch.equal(got, want):
            bad = int((got != want).nonzero()[0])
            raise AssertionError(f"{name}: local elements [{a}, {a + n}) differ from their piece, first at "
                                 f"element {a + bad // isz} (byte {bad % isz} of it), "
                                 f"{int((got != want).sum())} bytes in all")


def generator_f64(case, kw, d, x, got):
    """16-bit generators without an epilogue: every anchor element against the float64 value of its Philox
    half-word, under the T1' float64 bar of tests/generator_domain.py."""
    dt = TORCH_DT[kw["dtype"]]
    if kw.get("epi") or F.resolve_algo(kw) not in (0, C.TDX_ALGO_ICDF16):
        return
    i = torch.arange(x, x + got.size, dtype=torch.int64)
    if kw.get("flags", 0) & C.TDX_FLAG_WINDOW:
        w, p = kw["window_width"], kw["window_pitch"]
        g = int(d.elem_begin) + (i // w) * p + i % w
    else:
        g = int(d.elem_begin) + i
    k = PT.halfwords(int(d.philox_seed), int(d.philox_offset), g).numpy()
    v = G.as_f64(got, dt)
    lo, hi = kw["p0"], kw["p1"]
    if kw["src"] == F.U:
        ref = lo + k * (hi - lo) / 65536.0
        V, _ = G._grid(dt)
        cap = V[V < float(torch.tensor(hi, dtype=dt))].max() if lo != hi else None  # (below `to`, as ATen)
        G.near(v, ref, 4 * G.EPS32 * (abs(lo) + abs(hi) + np.abs(ref)), dt, cap=cap, ulp1=False)
        return
    mean, std = lo, hi
    body = k != 0
    ref = G.normal_ref(k[body].astype(np.float64), mean, std)
    z = np.abs(ref - mean) / std if std else np.zeros_like(ref)
    G.near(v[body], ref, G.ICDF_REL_ERR * std * z + 8 * G.EPS32 * (abs(mean) + std * z) + 1e-300, dt, ulp1=False)
    if (~body).any():
        from scipy.special import ndtri

        w = PT.tail_words(int(d.philox_seed), int(d.philox_offset), g[torch.from_numpy(~body)]).numpy().astype(np.int64)
        pr = ((w & 0x7FFFFFFF).astype(np.float64) + 0.5) * 2.0 ** -31 * 2.0 ** -17
        tref = mean + std * np.where(w & 0x80000000, 1.0, -1.0) * -ndtri(pr)
        G.near(v[~body], tref, 8 * G.EPS32 * np.abs(tref) + 1e-300, dt, ulp1=False)


def check_anchors(case, d, big, base_off, host_source, name):
    """Reference (b): the C restatement at the anchors."""
    isz, count, kw = case.isz, int(d.elem_count), case.spec.kw
    for x in anchors(count, base_off % 16, isz):
        k = min(ANCHOR, count - x)
        sub, skip = L.sub_desc(d, x, k)
        if sub.src == C.TDX_SRC_GATHER:
            sub.fill_bits[0] = host_source.ctypes.data
        want = F.oracle_bits(case.spec, sub)
        got = big[base_off + x * isz: base_off + (x + k) * isz].cpu().numpy().view(NP_BITS[isz])
        if want is not None:
            check_anchor(Anchored(f"{name} at local element {x}"), case.spec, got, want[skip:])
        if isz == 2 and kw["src"] in (F.U, F.N):
            generator_f64(case, kw, d, x, got)


NP_BITS = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def run_case(case):
    isz, nbytes = case.isz, case.nbytes
    need_device(nbytes + 64 + SCRATCH)
    big = torch.full((nbytes + 64,), 0xFF, dtype=torch.uint8, device="cuda")
    host_source, source = None, None
    if case.source_elems:
        r = np.random.default_rng(7)
        host_source = r.integers(0, 256, case.source_elems * isz, dtype=np.uint8)
        source = torch.from_numpy(host_source).cuda()
    d = case.desc(big.data_ptr(), source.data_ptr() if source is not None else 0)
    n, ws = submit([d])
    torch.cuda.synchronize()
    assert n == F.launches([case.spec]) == 1, (case, n)
    del ws
    # the bytes around the destination are untouched
    assert bool((big[: case.head] == 0xFF).all()) and bool((big[case.head + nbytes:] == 0xFF).all()), case
    scratch = torch.empty(SCRATCH, dtype=torch.uint8, device="cuda")
    check_pieces(case, d, big, case.head, scratch, case.name)
    check_anchors(case, d, big, case.head, host_source, case.name)


@pytest.mark.parametrize("case", L.family_cases(), ids=repr)
def test_a_large_descriptor_equals_its_pieces(case):
    run_case(case)


@pytest.mark.parametrize("case", L.large_i64_cases(), ids=repr)
def test_past_2_to_31_eight_byte_elements(case):
    run_case(case)


@pytest.mark.parametrize("case", L.window_cases(), ids=repr)
def test_a_large_window_equals_the_host_cut_pieces(case):
    run_case(case)


def test_a_window_block_past_2_to_31_vectors():
    run_case(L.huge_window_case())


def test_a_mixed_table_of_large_descriptors():
    specs, arena_bytes = L.mixed_table()
    need_device(arena_bytes + SCRATCH)
    big = torch.full((arena_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    descs = [s.desc(big.data_ptr()) for s in specs]
    n, ws = submit(descs)
    torch.cuda.synchronize()
    assert n == F.launches(specs), (n, F.launches(specs))
    del ws
    scratch = torch.empty(SCRATCH, dtype=torch.uint8, device="cuda")
    ends = [0] + [x for s in specs for x in (s.off, s.off + s.nbytes)] + [arena_bytes]
    for a, b in zip(ends[::2], ends[1::2]):  # gaps and guards untouched
        assert bool((big[a:b] == 0xFF).all()), (a, b)
    for i, (s, d) in enumerate(zip(specs, descs)):
        case = L.Case(f"mixed descriptor {i}", s, F.family(s.kw), head=s.off)
        check_pieces(case, d, big, s.off, scratch, case.name)
        check_anchors(case, d, big, s.off, None, case.name)


# ---- the public API at these sizes -----------------------------------------------------------------

def raw(t):
    return t.detach().reshape(-1).view(torch.uint8)


def test_aten_stream_past_2_to_31_elements():
    """rng="aten": a bf16 normal_ of 2^31 + 5 elements (ATen splits its iterator: the engine replays it)
    and a fused uniform_ after it equal eager CUDA after the same seed, with the same generator offset."""
    from torch import nn

    from torchdistx_b200.deferred_init import deferred_init, last_materialize_stats, materialize_module

    n = (1 << 31) + 5
    need_device(2 * 2 * n + 2 * (1 << 24) * 2)

    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.big = nn.Parameter(torch.empty(n, dtype=torch.bfloat16, device="cuda"))
            self.small = nn.Parameter(torch.empty(1 << 24, dtype=torch.bfloat16, device="cuda"))
            nn.init.normal_(self.big, 0.0, 0.02)
            nn.init.uniform_(self.small, -0.1, 0.1)

    gen = torch.cuda.default_generators[0]
    torch.manual_seed(11)
    m = deferred_init(M)
    materialize_module(m, rng="aten")
    off = gen.get_offset()
    st = last_materialize_stats()
    assert st["fused_tensors"] >= 1 and st["generic_ops"] >= 1, st  # (the uniform_ fused, the normal_ replayed)
    big, small = m.big.detach(), m.small.detach()
    del m
    torch.manual_seed(11)
    e_small = torch.empty(1 << 24, dtype=torch.bfloat16, device="cuda")
    e_big = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    e_big.normal_(0.0, 0.02)
    e_small.uniform_(-0.1, 0.1)
    assert gen.get_offset() == off, (gen.get_offset(), off)
    assert torch.equal(raw(small), raw(e_small))
    step = 1 << 30
    for a in range(0, n, step):
        assert torch.equal(raw(big[a: a + step]), raw(e_big[a: a + step])), a


def test_one_large_parameter_equals_its_shards():
    """materialize_module of a 2^31 + 2^20 + 3-element bf16 normal_(0, 0.02) and an fp32 trunc_normal_ of
    2^31 + 17 elements: each equals the concatenation of its shard=(r, 16) materialisations, slice by slice,
    and is fused whole."""
    from torch import nn

    from torchdistx_b200.deferred_init import deferred_init, last_materialize_stats, materialize_module

    nb, nf = (1 << 31) + (1 << 20) + 3, (1 << 31) + 17
    free = torch.cuda.mem_get_info()[0]
    with_f32 = free >= 2 * nb + 4 * nf + 2 * (4 * nf // 16) + SLACK
    need_device(2 * nb + 2 * (2 * nb // 16))

    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.w = nn.Parameter(torch.empty(nb, dtype=torch.bfloat16, device="cuda"))
            nn.init.normal_(self.w, 0.0, 0.02)
            if with_f32:
                self.t = nn.Parameter(torch.empty(nf, dtype=torch.float32, device="cuda"))
                nn.init.trunc_normal_(self.t, std=0.02)

    torch.manual_seed(21)
    m = deferred_init(M)
    materialize_module(m)
    st = last_materialize_stats()
    assert st["fused_tensors"] == (2 if with_f32 else 1) and st["generic_ops"] == 0, st
    whole = {k: v.detach() for k, v in m.named_parameters()}
    del m
    for r in range(16):
        torch.manual_seed(21)
        s = deferred_init(M)
        materialize_module(s, shard=(r, 16))
        assert last_materialize_stats()["generic_ops"] == 0
        for k, v in s.named_parameters():
            per = -(-whole[k].numel() // 16)
            assert torch.equal(raw(v), raw(whole[k][r * per: (r + 1) * per])), (k, r)
        del s
    if not with_f32:
        pytest.skip(f"ran the bf16 parameter only: the fp32 one needs {2 * nb + 4 * nf + SLACK} bytes of free "
                    f"device memory, {free} free")


def llama3_70b():
    import transformers as T

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
    from offload_bench import LLAMA3_70B

    cfg = T.LlamaConfig(**LLAMA3_70B)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            return T.LlamaForCausalLM(cfg)
    finally:
        torch.set_default_dtype(prev)


def test_fsdp1_flat_shard_of_llama3_70b():
    """materialize_flat_shard(align_numel=8) of Llama-3-70B bf16, ranks 0 and 7 of 8 (17.6 GB each), in HBM:
    every flat element equals the same element of the world-64 shards; rank 0 into pinned host memory
    equals the HBM shard byte for byte."""
    from torchdistx_b200.deferred_init import deferred_init, materialize_flat_shard

    def params():
        torch.manual_seed(4)
        return [p for _, p in deferred_init(llama3_70b).named_parameters()]

    ps = params()
    total = sum(p.numel() for p in ps) + 8 * len(ps)
    per8 = -(-total // 8)
    need_device(2 * per8 + 2 * (-(-total // 64)))
    fine = params()
    for rank in (0, 7):
        ps = params()
        shard, offs = materialize_flat_shard(ps, rank, 8, align_numel=8)
        per8 = shard.numel()
        lo8 = rank * per8
        per64 = None
        for r64 in range(rank * 8, min(64, rank * 8 + 9)):  # (and the next rank's first, if any)
            torch.manual_seed(4)
            small, offs64 = materialize_flat_shard(fine, r64, 64, align_numel=8)
            assert offs64 == offs
            per64 = small.numel()
            lo, hi = max(lo8, r64 * per64), min(lo8 + per8, (r64 + 1) * per64)
            if lo < hi:
                assert torch.equal(raw(shard[lo - lo8: hi - lo8]), raw(small[lo - r64 * per64: hi - r64 * per64])), \
                    (rank, r64)
            del small
        if rank == 0:
            need_host(2 * per8)
            out = torch.empty(per8, dtype=torch.bfloat16).pin_memory()
            torch.manual_seed(4)
            got, _ = materialize_flat_shard(params(), 0, 8, align_numel=8, out=out)
            assert got.data_ptr() == out.data_ptr()
            step = 1 << 29
            for a in range(0, per8, step):
                assert torch.equal(raw(out[a: a + step].cuda()), raw(shard[a: a + step])), a
            del out, got
        del shard


def test_offloaded_plan_shard_of_llama3_70b():
    """InitPlan.materialize(shard=(0, 8), into=pinned host) of Llama-3-70B bf16 equals the same call into a
    CUDA buffer, compared in 1 GiB slices."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "benchmarks"))
    from offload_bench import carve, shard_bytes

    from torchdistx_b200.deferred_init import deferred_init
    from torchdistx_b200.plan import InitPlan

    plan = InitPlan.from_module(deferred_init(llama3_70b))
    shard = (0, 8)
    nbytes = shard_bytes(plan, shard)
    need_device(nbytes + (256 << 20))
    need_host(nbytes)
    hbm = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    torch.manual_seed(6)
    plan.materialize(shard=shard, into=carve(plan, shard, hbm)[0])
    off = torch.cuda.default_generators[0].get_offset()
    pinned = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    torch.manual_seed(6)
    plan.materialize(shard=shard, into=carve(plan, shard, pinned)[0])
    assert torch.cuda.default_generators[0].get_offset() == off
    step = 1 << 30
    for a in range(0, nbytes, step):
        assert torch.equal(pinned[a: a + step].cuda(), hbm[a: a + step]), a
