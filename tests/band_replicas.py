"""Replicas of the causal-mask builders of transformers 5.5 (GPT-BigCode, GPT-Neo, ImageGPT / Bark /
CLVP, OpenAI GPT) and of the additive `full(-inf).triu(1)` mask, each as its module records it (the
constructor's buffer and `_init_weights`' `copy_` over it)."""
import numpy as np
import torch
from torch import nn


def causal_bool(n: int) -> torch.Tensor:
    """GPT-BigCode's `bias`: tril(ones(n, n, bool))."""
    return torch.tril(torch.ones((n, n), dtype=torch.bool))


def neo_bias(n: int, window: int = 0) -> torch.Tensor:
    """GPT-Neo's `bias` ([1, 1, n, n]); a local layer keeps only the last `window` diagonals."""
    bias = torch.tril(torch.ones((n, n), dtype=bool)).view(1, 1, n, n)
    if window:
        bias = torch.bitwise_xor(bias, torch.tril(bias, -window))
    return bias


def openai_bias(n: int) -> torch.Tensor:
    """OpenAI GPT's fp32 `bias`: tril(ones(n, n)).view(1, 1, n, n)."""
    return torch.tril(torch.ones(n, n)).view(1, 1, n, n)


def additive_mask(n: int, dtype=torch.float32) -> torch.Tensor:
    """The additive causal mask (nn.Transformer.generate_square_subsequent_mask): -inf above the diagonal."""
    return torch.triu(torch.full((n, n), float("-inf"), dtype=dtype), diagonal=1)


class BigCodeMask(nn.Module):
    def __init__(self, n):
        super().__init__()
        self.register_buffer("bias", causal_bool(n), persistent=False)
        with torch.no_grad():
            self.bias.copy_(causal_bool(n))


class NeoAttentionMask(nn.Module):
    def __init__(self, n, window=0):
        super().__init__()
        self.register_buffer("bias", neo_bias(n, window), persistent=False)
        with torch.no_grad():
            self.bias.copy_(neo_bias(n, window))


class OpenAIMask(nn.Module):
    def __init__(self, n):
        super().__init__()
        self.register_buffer("bias", openai_bias(n), persistent=False)
        with torch.no_grad():
            self.bias.copy_(openai_bias(n))


class AdditiveMask(nn.Module):
    def __init__(self, n, dtype=torch.float32):
        super().__init__()
        self.register_buffer("mask", additive_mask(n, dtype))


class NeoStack(nn.Module):
    """The masks of a GPT-Neo stack: alternating global and local layers."""

    def __init__(self, layers=24, n=2048, window=256):
        super().__init__()
        self.h = nn.ModuleList(NeoAttentionMask(n, window if i % 2 else 0) for i in range(layers))


def as_tensor(raw: np.ndarray, dtype: torch.dtype) -> torch.Tensor:
    return torch.from_numpy(raw.copy()).view(dtype)
