"""Small replicas of the state-space / linear-attention initialisers of transformers 5.5 (the
classes themselves are not instantiated: their constructors load kernels from the hub)."""
import math

import numpy as np
import torch
from torch import nn

T_MIN, T_MAX, FLOOR = 0.001, 0.1, 1e-4


def dt_program(n, dtype, device):
    """models/mamba2/modeling_mamba2.py:228-235 (and mamba/modeling_mamba.py:135-141)."""
    dt = torch.exp(
        torch.rand(n, device=device, dtype=dtype) * (math.log(T_MAX) - math.log(T_MIN)) + math.log(T_MIN)
    ).clamp(min=FLOOR)
    return dt + torch.log(-torch.expm1(-dt))


class Mamba2Mixer(nn.Module):
    """models/mamba2/modeling_mamba2.py:174-178 (parameters), 222-236 (init_mamba2_weights)."""

    def __init__(self, heads=24, dtype=torch.float32, device=None, int_arange=False):
        super().__init__()
        self.dt_bias = nn.Parameter(torch.empty(heads, dtype=dtype, device=device))
        self.A_log = nn.Parameter(torch.empty(heads, device=device))
        self.D = nn.Parameter(torch.empty(heads, device=device))
        with torch.no_grad():
            if int_arange:  # Bamba / Falcon-H1 / Granite-hybrid: an int64 arange promoted by log
                A = torch.arange(1, heads + 1, device=device)
            else:
                A = torch.arange(1, heads + 1, device=device, dtype=torch.float32)
            self.A_log.copy_(torch.log(A))
            self.D.fill_(1.0)
            self.dt_bias.copy_(dt_program(heads, dtype, device))


class MambaMixer(nn.Module):
    """models/mamba/modeling_mamba.py:100 (A_log), 122-142 (init_mamba_weights)."""

    def __init__(self, inner=64, state=16, rank=8, device=None):
        super().__init__()
        self.A_log = nn.Parameter(torch.empty(inner, state, device=device))
        self.dt_proj = nn.Linear(rank, inner, bias=True, device=device)
        with torch.no_grad():
            A = torch.arange(1, state + 1, dtype=torch.float32, device=device)[None, :]
            A = A.expand(inner, -1).contiguous()
            self.A_log.copy_(torch.log(A))
            self.dt_proj.bias.copy_(dt_program(inner, torch.float32, device))


class GatedDeltaNet(nn.Module):
    """models/qwen3_next/modeling_qwen3_next.py:532-535 (constructor), 890-892 (_init_weights)."""

    def __init__(self, heads=32, dtype=torch.float32, device=None):
        super().__init__()
        self.dt_bias = nn.Parameter(torch.ones(heads, dtype=dtype, device=device))
        A = torch.empty(heads, dtype=dtype, device=device).uniform_(0, 16)
        self.A_log = nn.Parameter(torch.log(A))
        with torch.no_grad():
            self.dt_bias.fill_(1.0)
            self.A_log.copy_(torch.empty_like(self.A_log).uniform_(0, 16).log_())


class Buffers(nn.Module):
    """Other broadcast index programs: a column broadcast and `repeat`."""

    def __init__(self, n=12, m=5, device=None):
        super().__init__()
        self.register_buffer("cols", torch.log(torch.arange(1, n + 1, dtype=torch.float32, device=device)[:, None]
                                               .expand(-1, m).contiguous()))
        self.register_buffer("rep", torch.log(torch.arange(1, n + 1, dtype=torch.float32, device=device).repeat(m, 1)))


def inv_softplus(x: float) -> float:
    return x + math.log(-math.expm1(-x))


def as_tensor(bits: np.ndarray, dtype: torch.dtype) -> torch.Tensor:
    view = {torch.float32: np.int32, torch.bfloat16: np.int16, torch.float16: np.int16, torch.int64: np.int64}[dtype]
    return torch.from_numpy(bits.view(view).copy()).view(dtype)
