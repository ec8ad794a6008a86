"""The generator KERNELS at edge parameters, bit for bit against the exact references of
tests/generator_edges.py (zero spreads, collapsed ranges, signed zeros, fp16 overflow and subnormals).

Every case runs through every kernel family that can take it, each proven by its launch count: the direct
16-bit kernels (TDX_ALGO_NOLUT), the table kernel (a 2^25-element descriptor and a small one in one launch:
two kernels; mean +0 is its mirrored build) and its any-seed form (two seeds in one launch), the fp32
generators, the wide (fp32 stream) 16-bit forms, and the window kernels on their whole-vector path (aligned
W, P, start and destination) and their element path -- each without an epilogue, with a basic one and with
the superset epilogue (steps that change no bit, or the case's own program).  Then the ATen-stream kernels
(rng="aten": plain, fp32-then-cast and windowed) against eager ATen after the same seed, generator offset
included.  Last, a Llama-shaped bf16 model whose largest weight is drawn with normal_(0.0, 0.0)."""
import pytest
import torch
from torch import nn

import generator_edges as E
from torchdistx_b200 import _C
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, last_descriptors, last_materialize_stats, \
    materialize_module, materialize_tensor

pytestmark = pytest.mark.gpu

SEEDS, OFFSET = (0xC0FFEE_1234, 0x51), 0x2_0000_0100
# (the table kernel takes a launch of >= 2^25 normal or >= 2^26 uniform 16-bit elements)
SMALL, BIG, PROBE = 1 << 22, {E.N: 1 << 25, E.U: 1 << 26}, 4099
# window geometry: rows, pitch P, first column, width W, destination offset in elements
WINDOWS = {"window-vec": (4096, 2048, 512, 1024, 0), "window-elem": (4194, 1999, 7, 1000, 1)}


def launch(descs):
    need = C.prepare(descs)
    ws = torch.empty(max(need, 16), dtype=torch.uint8, device="cuda")
    n = C.submit(ws.data_ptr(), need)
    torch.cuda.synchronize()
    return n


def families(dtype, case):
    """(family, wide, epilogue variants) that can run the case."""
    if dtype == torch.float32:
        rows = [("direct", False), ("window-vec", False), ("window-elem", False)]
    else:
        rows = [(f, False) for f in ("direct", "table", "two-seeds", "window-vec", "window-elem")]
        if case.kind != "range":  # (its references are functions of the 16-bit stream)
            rows += [(f, True) for f in ("direct", "window-vec", "window-elem")]
    out = []
    for fam, wide in rows:
        epis = {"table": ("none", "basic"), "two-seeds": ("none",)}.get(fam, ("none", "basic", "ext"))
        out.append((fam, wide, case.variants(epis)))
    return out


_streams = {}


def stream(seed, key, g):
    """Decoded streams, shared by every case of the module (the geometry `key` fixes g)."""
    if (seed, key) not in _streams:
        _streams[(seed, key)] = E.Stream(seed, OFFSET, g())
    return _streams[(seed, key)]


def run(dtype, case, fam, wide, steps, p0, p1):
    """[(bits, stream)] of the family's outputs; asserts the launch count that proves the family."""
    native16 = dtype != torch.float32 and not wide
    if wide:
        algo = C.TDX_ALGO_WIDE32
    else:
        algo = (C.TDX_ALGO_ICDF16 if native16 else C.TDX_ALGO_BM32) if case.src == E.N else 0
    kw = dict(dtype=E.TDX[dtype], src=case.src, offset=OFFSET, p0=p0, p1=p1)
    # a small descriptor of the plain direct family: one more kernel unless the case runs in that family
    probe_t = torch.empty(PROBE, dtype=dtype, device="cuda")
    probe = C.make_desc(probe_t.data_ptr(), elem_count=PROBE, seed=SEEDS[0],
                        algo=algo | (C.TDX_ALGO_NOLUT if native16 else 0), **kw)
    if fam == "direct":
        t = torch.empty(SMALL, dtype=dtype, device="cuda")
        d = C.make_desc(t.data_ptr(), elem_count=SMALL, seed=SEEDS[0], epi=steps,
                        algo=algo | (C.TDX_ALGO_NOLUT if native16 else 0), **kw)
        assert launch([d, probe]) == (2 if steps else 1), (fam, steps)
        g = lambda: torch.arange(SMALL, dtype=torch.int64, device="cuda")  # noqa: E731
        return [(t.view(E.INT[dtype]), stream(SEEDS[0], "small", g))]
    if fam in ("table", "two-seeds"):
        seeds = SEEDS if fam == "two-seeds" else SEEDS[:1]
        big = BIG[case.src]
        outs = [torch.empty(big, dtype=dtype, device="cuda") for _ in seeds]
        descs = [C.make_desc(t.data_ptr(), elem_count=big, seed=s, algo=algo, epi=steps, **kw)
                 for t, s in zip(outs, seeds)]
        # a small descriptor (below the table kernel's 2^18) runs in the direct kernel, and is the head of the
        # first large one: two kernels prove that the large ones took the table kernel (with two seeds its
        # form that reads the Philox keys from each descriptor)
        small = torch.empty(PROBE, dtype=dtype, device="cuda")
        descs.append(C.make_desc(small.data_ptr(), elem_count=PROBE, seed=SEEDS[0], algo=algo, epi=steps, **kw))
        assert launch(descs) == 2, (fam, steps)
        E.assert_bits(outs[0][:PROBE].view(E.INT[dtype]), small.view(E.INT[dtype]), "table head vs direct")
        g = lambda: torch.arange(big, dtype=torch.int64, device="cuda")  # noqa: E731
        return [(t.view(E.INT[dtype]), stream(s, big, g)) for t, s in zip(outs, seeds)]
    rows, pitch, c0, w, off = WINDOWS[fam]
    n = rows * w
    buf = torch.empty(n + off, dtype=dtype, device="cuda")
    d = C.make_desc(buf.data_ptr() + off * buf.element_size(), elem_begin=c0, elem_count=n, seed=SEEDS[0], algo=algo,
                    epi=steps, flags=C.TDX_FLAG_WINDOW, **kw)
    d.fill_bits[0], d.fill_bits[1] = w, pitch
    assert launch([d, probe]) == 2, (fam, steps)

    def g():
        i = torch.arange(n, dtype=torch.int64, device="cuda")
        return (i // w) * pitch + c0 + i % w

    return [(buf[off:].view(E.INT[dtype]), stream(SEEDS[0], fam, g))]


PARAMS = [(dt, c) for dt in E.DTYPES for c in E.cases(dt)]


@pytest.mark.parametrize("dtype,case", PARAMS, ids=[f"{str(dt)[6:]}-{c.id}" for dt, c in PARAMS])
def test_kernels_give_the_exact_answer(dtype, case):
    """Every family, every epilogue variant; all failures of a case are reported together."""
    failures, tables = [], {}
    for fam, wide, variants in families(dtype, case):
        for epi, steps in variants:
            what = f"{dtype} {case.id} {fam}{' wide' if wide else ''} {epi}"
            try:
                outs = run(dtype, case, fam, wide, steps, case.p0, case.p1)
            except AssertionError as e:
                failures.append(f"{what}: {str(e).splitlines()[0]}")
                continue
            for j, (bits, st) in enumerate(outs):
                raw = lambda p0, p1, j=j: run(dtype, case, fam, wide, [], p0, p1)[j][0]  # noqa: E731
                try:
                    table = E.check(case, dtype, wide, bits, st, raw, what)
                except AssertionError as e:
                    failures.append(str(e).splitlines()[0])
                    continue
                if table is not None:
                    tables[(fam, epi, j)] = table
    if tables:  # the table kernel (and its mirrored build) == the direct kernel, bit for bit
        ref = tables.pop(("direct", "none", 0))
        for k, t in tables.items():
            if not (t[1:] == ref[1:]).all():
                failures.append(f"{case.id} {k}: {int((t[1:] != ref[1:]).sum())} k differ from the direct kernel's")
    assert not failures, "\n".join(failures)


# Descriptors whose parameters are equal as numbers but not as bit patterns, in one table launch.  A CTA
# reuses the table it holds for the next descriptor only if their parameters are the same bits: +0 and -0
# give tables of opposite signed zeros.  (source, (p0, p1, steps) of each)
PAIRS = {
    "normal(+0,0)|normal(-0,0)": (E.N, (0.0, 0.0, []), (-0.0, 0.0, [])),
    "normal(-0,+0)|normal(-0,-0)": (E.N, (-0.0, 0.0, []), (-0.0, -0.0, [])),
    "uniform(-0,-0)|uniform(-0,+0)": (E.U, (-0.0, -0.0, []), (-0.0, 0.0, [])),
    "mul_(0)|mul_(-0)": (E.N, (0.0, 1.0, E.TIMES0), (0.0, 1.0, E.NEG_TIMES0)),
}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("pair", list(PAIRS))
@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_table_is_not_shared_across_signed_zeros(dtype, pair, order):
    """Both large descriptors of a pair in one table launch (a small one in the direct kernel: two
    kernels), each bit for bit the direct kernel's output for its own parameters -- which
    test_kernels_give_the_exact_answer holds to the exact references."""
    src, *params = PAIRS[pair]
    if order == "reverse":
        params = params[::-1]
    big = BIG[src]
    kw = dict(dtype=E.TDX[dtype], src=src, seed=SEEDS[0], offset=OFFSET)
    algo = C.TDX_ALGO_ICDF16 if src == E.N else 0
    outs, descs = [], []
    for p0, p1, steps in params:
        outs.append(torch.empty(big, dtype=dtype, device="cuda"))
        descs.append(C.make_desc(outs[-1].data_ptr(), elem_count=big, p0=p0, p1=p1, epi=steps, algo=algo, **kw))
    small = torch.empty(PROBE, dtype=dtype, device="cuda")
    p0, p1, steps = params[0]
    descs.append(C.make_desc(small.data_ptr(), elem_count=PROBE, p0=p0, p1=p1, epi=steps, algo=algo, **kw))
    assert launch(descs) == 2
    ref = torch.empty(big, dtype=dtype, device="cuda")
    for t, (p0, p1, steps) in zip(outs, params):
        d = C.make_desc(ref.data_ptr(), elem_count=big, p0=p0, p1=p1, epi=steps, algo=algo | C.TDX_ALGO_NOLUT, **kw)
        assert launch([d]) == 1
        E.assert_bits(t.view(E.INT[dtype]), ref.view(E.INT[dtype]), f"{pair} {order}: ({p0!r}, {p1!r}, {steps})")


# ---- the ATen stream ------------------------------------------------------------------------------
def program(case, dtype, shape, wide):
    """The eager program of a case on a CUDA tensor of `shape` (wide: drawn in fp32, then cast)."""
    def fn():
        t = torch.empty(shape, device="cuda", dtype=torch.float32 if wide else dtype)
        if case.src == E.N:
            t.normal_(case.p0, case.p1)
        else:
            t.uniform_(case.p0, case.p1)
        if case.steps is E.TRUNC0:
            t.erfinv_().mul_(0.0).add_(0.0).clamp_(-2.0, 2.0)
        elif case.kind == "times0":
            t.mul_(case.steps[0][1])
        return t.to(dtype) if wide else t
    return fn


ATEN = [(dt, c, form) for dt in E.DTYPES for c in E.cases(dt)
        for form in (("plain", "window") if dt == torch.float32 else ("plain", "wide", "window"))]


@pytest.mark.parametrize("dtype,case,form", ATEN, ids=[f"{str(dt)[6:]}-{c.id}-{f}" for dt, c, f in ATEN])
def test_aten_stream_gives_eager_bits(dtype, case, form):
    if form == "window":
        rows, cols, world = 2048, 2048, 4
        torch.manual_seed(3)
        whole = program(case, dtype, (rows, cols), False)()
        for r in (0, world - 1):
            torch.manual_seed(3)
            t = deferred_init(program(case, dtype, (rows, cols), False))
            got = _C.materialize_tensors([t], None, (r, world), True, [2], rng="aten")[0]  # (Shard(1))
            assert any(d.reserved & C.TDX_FLAG_WINDOW for d in last_descriptors())
            want = torch.chunk(whole, world, 1)[r].contiguous()
            E.assert_bits(got.contiguous().view(E.INT[dtype]), want.view(E.INT[dtype]), f"{case.id} window rank {r}")
        return
    fn = program(case, dtype, SMALL + 3, form == "wide")
    torch.manual_seed(7)
    want = fn()
    want_off = torch.cuda.default_generators[0].get_offset()
    torch.manual_seed(7)
    got = materialize_tensor(deferred_init(fn), rng="aten")
    st = last_materialize_stats()
    assert st["aten_stream_tensors"] == 1 and st["generic_ops"] == 0, st
    algos = {d.algo & 0x0F for d in last_descriptors()}
    assert algos == {C.TDX_ALGO_ATEN_WIDE if form == "wide" else C.TDX_ALGO_ATEN}, algos
    E.assert_bits(got.view(E.INT[dtype]), want.view(E.INT[dtype]), f"{case.id} {form}")
    assert torch.cuda.default_generators[0].get_offset() == want_off
    if case.kind == "const":  # eager itself gives the exact answer
        E.assert_bits(want.view(E.INT[dtype]), E.full_bits(E.const_value(case), dtype, want.numel(), "cuda"), "eager")


# ---- end to end -----------------------------------------------------------------------------------
class ZeroEmbeddingLlama(nn.Module):
    """Llama-shaped, bf16: embedding, attention and MLP projections, RMSNorm weights, an untied head;
    _init_weights draws the embedding with normal_(0.0, 0.0) and the rest with normal_(0.0, 0.02).  With
    262M-element embedding and head, even an eighth of the model is a table-kernel launch."""

    def __init__(self, vocab=128256, hidden=2048, inter=8192, layers=2):
        super().__init__()
        kw = dict(dtype=torch.bfloat16, device="cuda")
        lin = lambda i, o: nn.Linear(i, o, bias=False, **kw)  # noqa: E731
        self.embed_tokens = nn.Embedding(vocab, hidden, **kw)
        self.layers = nn.ModuleList(nn.ModuleDict(dict(
            q_proj=lin(hidden, hidden), k_proj=lin(hidden, hidden // 4), v_proj=lin(hidden, hidden // 4),
            o_proj=lin(hidden, hidden), gate_proj=lin(hidden, inter), up_proj=lin(hidden, inter),
            down_proj=lin(inter, hidden))) for _ in range(layers))
        self.norm_weight = nn.Parameter(torch.ones(hidden, **kw))
        self.lm_head = lin(hidden, vocab)
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if m is self.embed_tokens:
            nn.init.normal_(m.weight, 0.0, 0.0)
        elif isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, 0.0, 0.02)


def assert_table_takes_the_embedding(descs, what):
    """The host's rule (tdx_init_host.cu): a 16-bit normal of >= 2^18 elements, not windowed, takes the table
    kernel when its launch holds >= 2^25 such elements.  Holds the test to the kernel it exists for."""
    lut = [d for d in descs if d.src == C.TDX_SRC_NORMAL and d.dtype == C.TDX_BF16 and d.elem_count >= 1 << 18
           and not d.reserved & C.TDX_FLAG_WINDOW and not d.algo & C.TDX_ALGO_NOLUT]
    assert sum(d.elem_count for d in lut) >= 1 << 25, what
    assert any(d.p0 == 0.0 and d.p1 == 0.0 for d in lut), what


def assert_zero(t, what):
    E.assert_bits(t.contiguous().view(torch.int16), torch.zeros(t.shape, dtype=torch.int16, device=t.device), what)


def test_zero_std_embedding_is_positive_zero_end_to_end(tmp_path):
    from torch.distributed.tensor.parallel import ColwiseParallel

    from test_tp_shard_gpu import tp_local
    from torchdistx_b200.plan import InitPlan

    torch.manual_seed(0)
    m = deferred_init(ZeroEmbeddingLlama)
    materialize_module(m)
    assert_table_takes_the_embedding(last_descriptors(), "materialize_module")
    assert_zero(m.embed_tokens.weight, "materialize_module")
    assert float(m.lm_head.weight.float().std()) > 0.019
    del m
    for r in range(8):
        torch.manual_seed(0)
        m = deferred_init(ZeroEmbeddingLlama)
        materialize_module(m, shard=(r, 8))
        assert_table_takes_the_embedding(last_descriptors(), f"shard=({r}, 8)")
        assert m.embed_tokens.weight.shape[0] == 128256 // 8
        assert_zero(m.embed_tokens.weight, f"shard=({r}, 8)")
        del m
    for r in (0, 3):
        got, dims = tp_local(ZeroEmbeddingLlama, {"embed_tokens": ColwiseParallel(), "lm_head": ColwiseParallel()}, r, 4,
                             seed=0)
        assert dims["embed_tokens.weight"] == 1
        assert any(d.reserved & C.TDX_FLAG_WINDOW for d in last_descriptors())
        assert_zero(got["embed_tokens.weight"], f"Shard(1) rank {r}")
        del got
    torch.manual_seed(0)
    InitPlan.from_module(deferred_init(ZeroEmbeddingLlama)).save(str(tmp_path / "p.json"))
    plan = InitPlan.load(str(tmp_path / "p.json"))
    assert_table_takes_the_embedding([d for _, _, ds in plan.descriptors(0, 0)[0] for d in ds], "InitPlan")
    got = plan.materialize(device="cuda")
    assert_zero(got["embed_tokens.weight"], "InitPlan")
    del got
    torch.manual_seed(0)
    m = deferred_init(ZeroEmbeddingLlama)
    materialize_module(m, rng="aten")
    assert last_materialize_stats()["aten_stream_tensors"] > 0
    assert_zero(m.embed_tokens.weight, 'rng="aten"')
