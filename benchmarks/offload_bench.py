"""Host-memory targets on one GPU: how close InitPlan.materialize(into=CPU) comes to the host link.

One command, one GPU, one JSON line:
  * rank 0's shard=(0, 8) of Llama-3-70B bf16 (Llama-3-8B when host memory is short: the line says which)
    into one pinned host buffer through InitPlan.materialize(into=...): wall time ending in a synchronise,
    pinned allocation outside the timed region;
  * alternating with it, a plain device-to-host cudaMemcpyAsync of the same bytes from HBM into the same
    pinned buffer: the link's measured rate, and the ratio of the two;
  * the same shard built into HBM: CUDA events around the call (its host planning included);
  * the same shard into a pageable host buffer;
  * one decoder layer of the same model initialised eagerly on the host CPU (its own constructor's init),
    per layer, not extrapolated.
The GPU's name and power limit and the host's core count are printed beside the numbers.

    python benchmarks/offload_bench.py [--model 70b|8b] [--reps 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

LLAMA3_70B = dict(vocab_size=128256, hidden_size=8192, intermediate_size=28672, num_hidden_layers=80,
                  num_attention_heads=64, num_key_value_heads=8, max_position_embeddings=8192, rope_theta=500000.0,
                  tie_word_embeddings=False)
LLAMA3_8B = dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                 num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=8192, rope_theta=500000.0,
                 tie_word_embeddings=False)


def gpu_context():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, _, limit = (q.stdout.strip().splitlines() or ["?, ?"])[0].partition(",")
    return dict(gpu=name.strip() or torch.cuda.get_device_name(0), power_limit=limit.strip(), host_cores=os.cpu_count())


def host_bytes_available() -> int:
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def config(name):
    import transformers as T

    return T.LlamaConfig(**(LLAMA3_70B if name == "70b" else LLAMA3_8B))


def carve(plan, shard, buf):
    """One target per entry of this rank's part, 16-byte aligned views into the flat byte buffer `buf`."""
    from torchdistx_b200.plan import _DTYPES, shard_range

    out, off = {}, 0
    for e in plan.entries:
        if e.source == "alias":
            continue
        dt = _DTYPES[e.dtype]
        n = shard_range(e, steps=plan._steps(e, shard, None, None))[1]
        nbytes = n * torch.empty((), dtype=dt).element_size()
        out[e.name] = buf[off: off + nbytes].view(dt)
        off = (off + nbytes + 15) & ~15
    return out, off


def shard_bytes(plan, shard):
    from torchdistx_b200.plan import _DTYPES, shard_range

    total = 0
    for e in plan.entries:
        if e.source != "alias":
            n = shard_range(e, steps=plan._steps(e, shard, None, None))[1]
            total = ((total + n * torch.empty((), dtype=_DTYPES[e.dtype]).element_size()) + 15) & ~15
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["70b", "8b"], default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("offload_bench.py measures on a CUDA device; there is none")
    import transformers as T

    from torchdistx_b200.deferred_init import deferred_init
    from torchdistx_b200.plan import InitPlan

    shard = (0, 8)
    model = args.model
    plans = {}
    for name in ([model] if model else ["70b", "8b"]):
        cfg = config(name)

        def build(cfg=cfg):
            prev = torch.get_default_dtype()
            torch.set_default_dtype(torch.bfloat16)
            try:
                with torch.device("cuda"):
                    return T.LlamaForCausalLM(cfg)
            finally:
                torch.set_default_dtype(prev)

        plan = InitPlan.from_module(deferred_init(build))
        need = shard_bytes(plan, shard)
        # the pinned and the pageable buffer, the eager layer and some slack
        if model or host_bytes_available() > 2 * need + (16 << 30):
            model, plans[name] = name, (plan, need)
            break
    plan, nbytes = plans[model]
    ctx = gpu_context()
    ctx.update(model=f"llama3-{model}", shard=list(shard), shard_bytes=nbytes)

    pinned = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    into, _ = carve(plan, shard, pinned)
    hbm = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dev_into, _ = carve(plan, shard, hbm)
    # warm-up: every kernel family, the staging allocation, the copy path
    torch.manual_seed(0)
    plan.materialize(shard=shard, into=into)
    pinned.copy_(hbm, non_blocking=True)
    torch.cuda.synchronize()

    build_s, copy_s = [], []
    for _ in range(args.reps):  # alternating: the host build, then the plain copy of the same bytes
        torch.manual_seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        plan.materialize(shard=shard, into=into)
        torch.cuda.synchronize()
        build_s.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        pinned.copy_(hbm, non_blocking=True)
        torch.cuda.synchronize()
        copy_s.append(time.perf_counter() - t0)

    hbm_ms = []
    for _ in range(args.reps):
        torch.manual_seed(0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        plan.materialize(shard=shard, into=dev_into)
        b.record()
        torch.cuda.synchronize()
        hbm_ms.append(a.elapsed_time(b))
    del hbm, dev_into
    torch.cuda.empty_cache()

    del into
    pinned = None
    pageable = torch.empty(nbytes, dtype=torch.uint8)
    pageable.fill_(0)  # (touched: first-touch page faults are not the library's time)
    p_into, _ = carve(plan, shard, pageable)
    pageable_s = []
    for _ in range(max(1, args.reps - 1)):
        torch.manual_seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        plan.materialize(shard=shard, into=p_into)
        torch.cuda.synchronize()
        pageable_s.append(time.perf_counter() - t0)
    del p_into, pageable

    cfg = config(model)
    from transformers.models.llama.modeling_llama import LlamaDecoderLayer

    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        t0 = time.perf_counter()
        layer = LlamaDecoderLayer(cfg, 0)
        for m in layer.modules():  # (what init_weights() does to a decoder layer: HF's _init_weights)
            if isinstance(m, torch.nn.Linear):
                m.weight.data.normal_(0.0, cfg.initializer_range)
        layer_s = time.perf_counter() - t0
    finally:
        torch.set_default_dtype(prev)
    layer_params = sum(p.numel() for p in layer.parameters())

    gb = nbytes / 1e9
    res = dict(ctx, host_pinned_s=min(build_s), host_pinned_gbps=gb / min(build_s), link_copy_s=min(copy_s),
               link_gbps=gb / min(copy_s), ratio_to_link=min(copy_s) / min(build_s), hbm_kernel_ms=min(hbm_ms),
               hbm_gbps=gb / (min(hbm_ms) / 1e3), host_pageable_s=min(pageable_s),
               host_pageable_gbps=gb / min(pageable_s), cpu_eager_layer_s=layer_s, cpu_eager_layer_params=layer_params,
               all_host_pinned_s=build_s, all_link_copy_s=copy_s, all_hbm_kernel_ms=hbm_ms,
               all_host_pageable_s=pageable_s)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
