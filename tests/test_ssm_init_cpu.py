"""State-space and linear-attention initialisers (Mamba / Mamba-2 A_log and dt bias, Qwen3-Next's
random A_log) on the fused path, without a GPU: planner verdicts, the compacted descriptors, and the
host chain InitPlan -> JSON -> descriptors -> CPU restatement of the kernels (oracle/tdx_oracle.c)."""
import json
import math

import numpy as np
import pytest
import torch
from scipy import stats
from torch import nn

import ssm_replicas as R
from oracle import tdx_oracle as O
from torchdistx_b200 import _cabi as C
from torchdistx_b200.deferred_init import deferred_init, plan_report
from torchdistx_b200.plan import FORMAT, FORMAT_SSM, InitPlan, offset_increment

SSM = {C.TDX_EPI_EXP, C.TDX_EPI_LOG, C.TDX_EPI_EXPM1, C.TDX_EPI_INV_SOFTPLUS, C.TDX_EPI_MULADD}


def ops(info):
    return [int(e[0]) & 0xFF for e in info["epilogue"]]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_mamba2_idioms_fold(dtype):
    r = plan_report(deferred_init(R.Mamba2Mixer, 24, dtype))
    a = r["A_log"]
    assert (a["source"], a["fusible"], ops(a)) == ("iota", True, [C.TDX_EPI_LOG]) and (a["p0"], a["p1"]) == (1.0, 1.0)
    dt = r["dt_bias"]
    assert dt["source"] == "uniform" and dt["fusible"]
    assert dt["dtype"] == {torch.float32: "Float", torch.bfloat16: "BFloat16"}[dtype]
    # [MUL, ADD, EXP, CLAMP, INV_SOFTPLUS] compacted to 4 steps
    assert ops(dt) == [C.TDX_EPI_MULADD, C.TDX_EPI_EXP, C.TDX_EPI_CLAMP, C.TDX_EPI_INV_SOFTPLUS]
    assert dt["n_epilogue"] <= 4 and dt["rng_ops"] == 1
    assert r["D"]["source"] == "const"


def test_int64_arange_is_promoted_by_log():
    a = plan_report(deferred_init(R.Mamba2Mixer, 24, int_arange=True))["A_log"]
    assert (a["source"], a["fusible"], ops(a)) == ("iota", True, [C.TDX_EPI_LOG])


def test_mamba_broadcast_arange_is_a_periodic_iota():
    r = plan_report(deferred_init(R.MambaMixer, 64, 16))
    a = r["A_log"]
    assert (a["source"], a["fusible"], ops(a)) == ("iota", True, [C.TDX_EPI_LOG])
    (seg,) = a["segments"]
    assert (seg["iota_period"], seg["iota_repeat"]) == (16, 0)
    b = r["dt_proj.bias"]  # Linear's kaiming uniform_ is overwritten: a dead pass
    assert b["source"] == "uniform" and b["fusible"] and b["rng_ops"] == 2 and len(b["epilogue"]) == 4
    rb = plan_report(deferred_init(R.Buffers, 12, 5))
    assert [(s["iota_period"], s["iota_repeat"]) for s in rb["cols"]["segments"]] == [(12, 5)]
    assert [(s["iota_period"], s["iota_repeat"]) for s in rb["rep"]["segments"]] == [(12, 0)]
    assert rb["cols"]["fusible"] and rb["rep"]["fusible"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_qwen3_next_random_a_log_folds(dtype):
    a = plan_report(deferred_init(R.GatedDeltaNet, 32, dtype))["A_log"]
    assert (a["source"], a["fusible"], ops(a), a["rng_ops"]) == ("uniform", True, [C.TDX_EPI_LOG], 2)
    assert (a["p0"], a["p1"]) == (0.0, 16.0)


class Negatives(nn.Module):
    def __init__(self):
        super().__init__()
        x = torch.rand(16)
        y = torch.rand(16)
        self.register_buffer("unrelated", x + torch.log(-torch.expm1(-y)))
        self.register_buffer("alpha", torch.add(x, torch.log(-torch.expm1(-x)), alpha=2))
        self.register_buffer("five", ((torch.randn(16) * 2 + 1) * 3 + 4) * 5)  # five steps, none new
        self.register_buffer("mask", torch.tril(torch.ones(8, 8)))


def test_negatives_stay_opaque():
    r = plan_report(deferred_init(Negatives))
    for name in ("unrelated", "alpha", "five", "mask"):
        assert r[name]["source"] == "opaque" and not r[name]["fusible"], (name, r[name])


class Model(nn.Module):
    def __init__(self, heads=4096):
        super().__init__()
        self.mamba2 = R.Mamba2Mixer(heads)
        self.mamba = R.MambaMixer(96, 16)
        self.qwen = R.GatedDeltaNet(heads)


def test_plan_round_trip_and_cpu_restatement(tmp_path):
    torch.manual_seed(0)
    plan = InitPlan.from_module(deferred_init(Model))
    p = tmp_path / "ssm.json"
    plan.save(str(p))
    assert json.load(open(p))["format"] == FORMAT_SSM
    plan = InitPlan.load(str(p))
    seed, off0 = 1234, 8
    got, end, _ = O.evaluate_plan(plan, seed, off0)
    # generator: Mamba-2's dt draw, Mamba's dead kaiming pass (dt_proj.weight's, then the bias's) and
    # its dt draw, Qwen's dead constructor draw and live _init_weights draw
    n_weight = 96 * 8
    assert end == off0 + offset_increment(4096) + offset_increment(n_weight) + offset_increment(96) * 2 + \
        2 * offset_increment(4096)
    # A_log: deterministic, within 1 ulp of ATen on the CPU (C libm vs ATen's vectorised log)
    ref2 = torch.log(torch.arange(1, 4097, dtype=torch.float32))
    assert (got["mamba2.A_log"].view(torch.int32) - ref2.view(torch.int32)).abs().max() <= 1
    ref1 = torch.log(torch.arange(1, 17, dtype=torch.float32))[None, :].expand(96, -1)
    assert (got["mamba.A_log"].view(torch.int32) - ref1.view(torch.int32)).abs().max() <= 1
    # RNG tensors: hard ranges, and T1 against an eager sample of the same program
    lo, hi = R.inv_softplus(R.T_MIN), R.inv_softplus(R.T_MAX)
    dt = got["mamba2.dt_bias"].double()
    assert dt.min() >= lo - 1e-5 and dt.max() <= hi + 1e-5 and not torch.isnan(dt).any()
    torch.manual_seed(1)
    ks = stats.ks_2samp(dt.numpy(), R.dt_program(4096, torch.float32, None).double().numpy())
    assert ks.pvalue > 1e-4, ks
    qa = got["qwen.A_log"].double()
    assert not torch.isnan(qa).any() and qa.max() <= math.log(16)
    ks = stats.ks_2samp(qa[torch.isfinite(qa)].numpy(), torch.empty(4096).uniform_(0, 16).log().double().numpy())
    assert ks.pvalue > 1e-4, ks
    # shards are torch.chunk of the whole
    for world in (2, 3, 8):
        parts = [O.evaluate_plan(plan, seed, off0, shard=(r, world))[0] for r in range(world)]
        for name in ("mamba2.A_log", "mamba2.dt_bias", "mamba.A_log", "qwen.A_log", "mamba.dt_proj.bias"):
            whole = torch.cat([p[name] for p in parts if p[name].numel()])
            assert torch.equal(whole.view(-1), got[name].view(-1)), (world, name)


def test_plans_without_the_extension_stay_version_2(tmp_path):
    plan = InitPlan.from_module(deferred_init(nn.Linear, 8, 8))
    plan.save(str(tmp_path / "p.json"))
    assert json.load(open(tmp_path / "p.json"))["format"] == FORMAT and not plan.uses_ssm()


def test_from_module_accepts_the_replicas():
    for cls in (R.Mamba2Mixer, R.GatedDeltaNet, R.MambaMixer):
        plan = InitPlan.from_module(deferred_init(cls))
        assert all(e.source != "value" for e in plan.entries), [(e.name, e.source) for e in plan.entries]


def test_make_desc_writes_the_broadcast_geometry():
    d = C.make_desc(0, dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_count=10, p0=1, p1=1, iota_period=5, iota_repeat=2)
    assert list(d.fill_bits) == [5, 2]
    assert list(C.make_desc(0, dtype=C.TDX_F32, src=C.TDX_SRC_IOTA, elem_count=10).fill_bits) == [0, 0]
    bits = O.generate(d).view(np.float32)
    assert bits.tolist() == [1, 1, 2, 2, 3, 3, 4, 4, 5, 5]
