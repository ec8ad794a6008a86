"""`rng="aten"` on the H100: every fused draw is bit for bit what ATen's own CUDA kernels give -- against
eager ATen after the same seed, against the op-by-op ATen replay of the reference's semantics
(`fused=False`), whole and in partitions -- and the default stream is untouched."""
import hashlib
import math

import pytest
import torch

from oracle import cases
from torchdistx_b200 import _C
from torchdistx_b200.deferred_init import deferred_init, last_descriptors, last_materialize_stats, \
    materialize_flat_shard, materialize_module, materialize_tensor

from test_tp_shard_gpu import LLAMA3_8B, llama3_8b

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def grid_stride():
    p = torch.cuda.get_device_properties(0)
    return 256 * p.multi_processor_count * (p.max_threads_per_multi_processor // 256)


def same_bits(a, b):
    """Equal dtypes, shapes and raw bits: -0 is not +0, and a NaN equals only the same NaN pattern."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype.is_floating_point:
        iv = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
        a, b = a.contiguous().view(iv), b.contiguous().view(iv)
    return torch.equal(a, b)


def same_as_eager(fn, seed=11):
    """fn() on CUDA eagerly, and recorded then materialised with rng="aten": equal bits and equal
    generator offsets afterwards."""
    torch.manual_seed(seed)
    want = fn()
    want_offset = torch.cuda.default_generators[0].get_offset()
    torch.manual_seed(seed)
    t = deferred_init(fn)
    got = materialize_tensor(t, rng="aten")
    assert got.dtype == want.dtype and got.shape == want.shape
    assert same_bits(got, want)
    assert torch.cuda.default_generators[0].get_offset() == want_offset


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("op", ["normal", "uniform"])
def test_draws_equal_eager(dtype, op):
    S = grid_stride()
    for n in (1, 255, S - 1, 4 * S + 3, 10**7 + 7):
        if op == "normal":
            same_as_eager(lambda: torch.empty(n, device="cuda", dtype=dtype).normal_(0.5, 2.0))
        else:
            same_as_eager(lambda: torch.empty(n, device="cuda", dtype=dtype).uniform_(-3.0, 0.7))
        assert last_materialize_stats()["aten_stream_tensors"] == 1 and last_materialize_stats()["generic_ops"] == 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_initialisers_equal_eager(dtype):
    kw = dict(device="cuda", dtype=dtype)
    programs = {
        "randn": lambda: torch.randn(3000, 77, **kw),
        "rand": lambda: torch.rand(5, 1000, 3, **kw),
        "kaiming_uniform_": lambda: torch.nn.init.kaiming_uniform_(torch.empty(512, 300, **kw), a=math.sqrt(5)),
        "xavier_normal_": lambda: torch.nn.init.xavier_normal_(torch.empty(700, 129, **kw)),
        "trunc_normal_": lambda: torch.nn.init.trunc_normal_(torch.empty(1000, 333, **kw), std=0.02),
        "randn_s_m": lambda: torch.randn(4099, 17, **kw) * 0.02 + 0.5,
        "dt_exp": lambda: torch.exp(torch.rand(1536, **kw) * (math.log(0.1) - math.log(0.001)) + math.log(0.001)),
    }
    for name, fn in programs.items():
        same_as_eager(fn)
        assert last_materialize_stats()["generic_ops"] == 0, name


def test_reverse_bound_branch_fires_in_bf16():
    """uniform_(1, 1.0078125) in bf16: the two bounds are adjacent bf16 values, so about half the draws
    round to `to` and are reversed to `from`."""
    fn = lambda: torch.empty(100003, device="cuda", dtype=torch.bfloat16).uniform_(1.0, 1.0078125)
    same_as_eager(fn)
    torch.manual_seed(11)
    assert (fn() == 1.0).float().mean() > 0.3


def test_explicit_generator():
    def fn(g):
        return torch.empty(12345, device="cuda").normal_(generator=g), torch.rand(999, device="cuda", generator=g)

    g = torch.Generator(device="cuda")
    g.manual_seed(77)
    want = fn(g)
    end = g.get_offset()
    g.manual_seed(77)
    a, b = deferred_init(lambda: fn(g))
    assert torch.equal(materialize_tensor(a, rng="aten"), want[0])
    assert torch.equal(materialize_tensor(b, rng="aten"), want[1])
    assert g.get_offset() == end


def replay_vs_aten(build, default_dtype=torch.float32):
    """materialize_module(rng="aten") against _C.materialize_module(fused=False) of the same recording.
    The replay runs under the default dtype the recording was made with: a factory op recorded without
    a dtype takes the one current when ATen runs it."""
    out = {}
    for mode in ("aten", "replay"):
        torch.manual_seed(5)
        m = deferred_init(build)
        if mode == "aten":
            materialize_module(m, rng="aten")
            stats = last_materialize_stats()
        else:
            prev = torch.get_default_dtype()
            torch.set_default_dtype(default_dtype)
            try:
                _C.materialize_module(m, False, None, None, None, False)
            finally:
                torch.set_default_dtype(prev)
        out[mode] = (m.state_dict(), torch.cuda.default_generators[0].get_offset())
    (a, oa), (b, ob) = out["aten"], out["replay"]
    assert oa == ob
    for k in b:
        assert same_bits(a[k], b[k]), k
    return stats


@pytest.mark.parametrize("case", ["family_bert", "family_opt", "family_t5", "family_vit", "family_conv_bn",
                                  "tiny_llama", "tiny_gpt2", "padded_embeddings", "clones", "cast_variant"])
def test_model_zoo_equals_replay(case):
    replay_vs_aten(lambda: cases.build(case, "fp32", "cuda"))


def test_llama3_8b_bf16_equals_replay():
    stats = replay_vs_aten(llama3_8b, torch.bfloat16)
    m = deferred_init(llama3_8b)
    draws = sum(1 for t in m.parameters() if _C.plan_info(t)["source"] in ("uniform", "normal"))
    assert stats["aten_stream_tensors"] == draws and stats["generic_ops"] == 0


def test_llama_built_fp32_then_cast_equals_replay():
    import transformers as T

    cfg = dict(LLAMA3_8B, num_hidden_layers=2, vocab_size=32000)

    def build():
        with torch.device("cuda"):
            return T.LlamaForCausalLM(T.LlamaConfig(**cfg)).to(torch.bfloat16)

    replay_vs_aten(build)


def test_gpt2_xl_fp32_equals_replay():
    import transformers as T

    def build():
        with torch.device("cuda"):
            return T.GPT2LMHeadModel(T.GPT2Config(n_embd=1600, n_layer=48, n_head=25))

    replay_vs_aten(build)


def whole_tensor(build):
    torch.manual_seed(9)
    m = deferred_init(build)
    materialize_module(m, rng="aten")
    return m


def tiny():
    with torch.device("cuda"):
        return torch.nn.Sequential(torch.nn.Linear(1000, 777), torch.nn.Embedding(5003, 96, padding_idx=1))


@pytest.mark.parametrize("world", [2, 3, 8])
def test_shards_are_slices(world):
    whole = whole_tensor(tiny).state_dict()
    for r in range(world):
        torch.manual_seed(9)
        m = deferred_init(tiny)
        materialize_module(m, shard=(r, world), rng="aten")
        for k, v in m.state_dict().items():
            want = torch.chunk(whole[k], world, 0)[r] if whole[k].dim() else whole[k]
            assert torch.equal(v, want), (k, r, world)


def test_fsdp1_flat_chunks_are_slices():
    whole = whole_tensor(tiny)
    flat = torch.cat([p.detach().reshape(-1) for p in whole.parameters()])
    world = 3
    for r in range(world):
        torch.manual_seed(9)
        m = deferred_init(tiny)
        shard, offsets = materialize_flat_shard(list(m.parameters()), r, world, device="cuda", rng="aten")
        chunk = (flat.numel() + world - 1) // world
        want = flat[r * chunk:(r + 1) * chunk]
        assert torch.equal(shard[:want.numel()], want), r


def test_windowed_shard1_blocks_are_slices():
    whole = whole_tensor(tiny).state_dict()
    world = 3
    for r in range(world):
        torch.manual_seed(9)
        m = deferred_init(tiny)
        ts = [m[0].weight, m[0].bias, m[1].weight]  # (in materialize_module's order: it sets the offsets)
        got = _C.materialize_tensors(ts, None, (r, world), True, [2, 0, 2], rng="aten")
        for k, v in zip(("0.weight", "0.bias", "1.weight"), got):
            want = whole[k] if k == "0.bias" else torch.chunk(whole[k], world, 1)[r]
            assert torch.equal(v, want), (k, r)


def test_boundaries():
    """2^30 bf16 elements take the kernels; 2^30 + 1 (a 64-bit iterator: 1 + N * 2 > 2^31 - 1) and a
    draw through a non-contiguous view are replayed through ATen.  All three equal eager."""
    same_as_eager(lambda: torch.empty(2**30, device="cuda", dtype=torch.bfloat16).normal_())
    assert last_materialize_stats()["aten_stream_tensors"] == 1
    same_as_eager(lambda: torch.empty(2**30 + 1, device="cuda", dtype=torch.bfloat16).normal_())
    assert last_materialize_stats()["aten_stream_tensors"] == 0 and last_materialize_stats()["generic_ops"] > 0
    same_as_eager(lambda: torch.empty(300, 200, device="cuda").t().normal_().t())
    assert last_materialize_stats()["aten_stream_tensors"] == 0


# sha256 of last_descriptors() of the default-stream Llama-3-8B bf16 call at seed 0, with the output
# addresses zeroed: the parent release's table
DEFAULT_LLAMA_DIGEST = "440164b243ab090b555920da31a2c40618f553625d77384fab5dee41714081dc"


def test_default_stream_is_untouched():
    import numpy as np

    torch.manual_seed(0)
    m = deferred_init(llama3_8b)
    materialize_module(m)
    raw = bytearray(last_descriptors())
    a = np.frombuffer(raw, dtype=np.uint64).reshape(-1, 16).copy()
    a[:, 0] = 0  # (dst)
    digest = hashlib.sha256(a.tobytes()).hexdigest()
    assert last_materialize_stats()["aten_stream_tensors"] == 0
    assert digest == DEFAULT_LLAMA_DIGEST
