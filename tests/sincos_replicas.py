"""Small replicas of the sinusoidal position tables of transformers 5.5 (the four builders verbatim,
and the modules that register and re-initialise them)."""
import math

import numpy as np
import torch
from torch import nn


def sinusoids(length: int, channels: int, max_timescale: float = 10000) -> torch.Tensor:
    """models/whisper/modeling_whisper.py:55-64."""
    if channels % 2 != 0:
        raise ValueError(
            f"Number of channels has to be divisible by 2 for sinusoidal positional embeddings, got {channels} channels."
        )
    log_timescale_increment = math.log(max_timescale) / (channels // 2 - 1)
    inv_timescales = torch.exp(-log_timescale_increment * torch.arange(channels // 2))
    scaled_time = torch.arange(length).view(-1, 1) * inv_timescales.view(1, -1)
    return torch.cat([scaled_time.sin(), scaled_time.cos()], dim=1)


def m2m100_embedding(num_embeddings: int, embedding_dim: int, padding_idx=None):
    """models/m2m_100/modeling_m2m_100.py:100-118 (M2M100SinusoidalPositionalEmbedding.get_embedding)."""
    half_dim = embedding_dim // 2
    emb = math.log(10000) / (half_dim - 1)
    emb = torch.exp(torch.arange(half_dim, dtype=torch.int64).float() * -emb)
    emb = torch.arange(num_embeddings, dtype=torch.int64).float().unsqueeze(1) * emb.unsqueeze(0)
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=1).view(num_embeddings, -1)
    if embedding_dim % 2 == 1:
        # zero pad
        emb = torch.cat([emb, torch.zeros(num_embeddings, 1)], dim=1)
    if padding_idx is not None:
        emb[padding_idx, :] = 0

    return emb.to(torch.get_default_dtype())


def musicgen_embedding(num_embeddings: int, embedding_dim: int):
    """models/musicgen/modeling_musicgen.py:124-137 (MusicgenSinusoidalPositionalEmbedding.get_embedding)."""
    half_dim = embedding_dim // 2
    emb = math.log(10000) / (half_dim - 1)
    emb = torch.exp(torch.arange(half_dim, dtype=torch.int64).float() * -emb)
    emb = torch.arange(num_embeddings, dtype=torch.int64).float().unsqueeze(1) * emb.unsqueeze(0)
    emb = torch.cat([torch.cos(emb), torch.sin(emb)], dim=1).view(num_embeddings, -1)
    if embedding_dim % 2 == 1:
        # zero pad
        emb = torch.cat([emb, torch.zeros(num_embeddings, 1)], dim=1)
    return emb.to(torch.get_default_dtype())


def create_sinusoidal_positions(num_pos: int, dim: int) -> torch.Tensor:
    """models/gptj/modeling_gptj.py:47-50 (CodeGen's is the same)."""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dim, 2, dtype=torch.int64) / dim))
    sinusoid_inp = torch.einsum("i , j -> i j", torch.arange(num_pos, dtype=torch.int64).float(), inv_freq).float()
    return torch.cat((torch.sin(sinusoid_inp), torch.cos(sinusoid_inp)), dim=1)


class WhisperPositions(nn.Module):
    """WhisperEncoder.embed_positions (modeling_whisper.py:570-571) and its _init_weights (:527):
    nn.Embedding's own normal_, the normal_ of _init_weights' nn.Embedding branch, then the copy of
    the table."""

    def __init__(self, length=1500, channels=1280):
        super().__init__()
        self.embed_positions = nn.Embedding(length, channels)
        self.embed_positions.requires_grad_(False)
        with torch.no_grad():
            self.embed_positions.weight.normal_(mean=0.0, std=0.02)
            self.embed_positions.weight.copy_(sinusoids(*self.embed_positions.weight.shape))


class M2M100Positions(nn.Module):
    """M2M100SinusoidalPositionalEmbedding (modeling_m2m_100.py:82-99) and its _init_weights (:493-498)."""

    def __init__(self, num_positions=1024, embedding_dim=1024, padding_idx=1):
        super().__init__()
        self.offset = 2
        self.num_positions = num_positions
        self.embedding_dim = embedding_dim
        self.padding_idx = padding_idx
        self.make_weights(num_positions + self.offset, embedding_dim, padding_idx)
        with torch.no_grad():
            self.weights.copy_(m2m100_embedding(num_positions + self.offset, embedding_dim, padding_idx))

    def make_weights(self, num_embeddings, embedding_dim, padding_idx=None):
        emb_weights = m2m100_embedding(num_embeddings, embedding_dim, padding_idx)
        if hasattr(self, "weights"):
            emb_weights = emb_weights.to(dtype=self.weights.dtype, device=self.weights.device)
        self.register_buffer("weights", emb_weights, persistent=False)


class MusicgenPositions(nn.Module):
    """MusicgenSinusoidalPositionalEmbedding (modeling_musicgen.py:108-121) and its _init_weights (:412-414)."""

    def __init__(self, num_positions=2048, embedding_dim=1024):
        super().__init__()
        self.embedding_dim = embedding_dim
        self.register_buffer("weights", musicgen_embedding(num_positions, embedding_dim), persistent=False)
        with torch.no_grad():
            self.weights.copy_(musicgen_embedding(num_positions, embedding_dim))


class GPTJAttentionPositions(nn.Module):
    """GPTJAttention.embed_positions (modeling_gptj.py:104-106) and its _init_weights (:429)."""

    def __init__(self, max_positions=2048, pos_embd_dim=64):
        super().__init__()
        self.register_buffer("embed_positions", create_sinusoidal_positions(max_positions, pos_embd_dim),
                             persistent=False)
        with torch.no_grad():
            self.embed_positions.copy_(create_sinusoidal_positions(max_positions, pos_embd_dim))


def as_tensor(bits: np.ndarray, dtype: torch.dtype) -> torch.Tensor:
    view = {torch.float32: np.int32, torch.bfloat16: np.int16, torch.float16: np.int16, torch.int64: np.int64}[dtype]
    return torch.from_numpy(bits.view(view).copy()).view(dtype)
