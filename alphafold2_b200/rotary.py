"""Mirror of alphafold2_pytorch/rotary.py (dead code at the reference HEAD, named in the north star).
``apply_rotary_pos_emb`` runs the sm_90a kernel; the sin/cos table builders are host-side setup."""
import torch
from torch import nn

from . import ops


def rotate_every_two(x):
    """rotary.py:9-13 — (x0, x1) -> (-x1, x0) on interleaved pairs; expressed through the kernel with sin=1, cos=0."""
    shp = x.shape
    x4 = x.reshape(1, 1, -1, shp[-1]).float().contiguous()
    n = x4.shape[2]
    one = torch.ones(1, n, shp[-1], device=x.device)
    return ops.apply_rotary_pos_emb(x4, (one, torch.zeros_like(one))).reshape(shp).to(x.dtype)


def apply_rotary_pos_emb(x, sinu_pos):
    """rotary.py:15-20 — x [b, h, n, dh]; sinu_pos = (sin, cos), each [1 or b, n, rot]; channels >= rot pass through."""
    return ops.apply_rotary_pos_emb(x.float().contiguous(), sinu_pos).to(x.dtype)


class FixedPositionalEmbedding(nn.Module):
    """rotary.py:35-45."""

    def __init__(self, dim):
        super().__init__()
        self.register_buffer('inv_freq', 1. / (10000 ** (torch.arange(0, dim, 2).float() / dim)))

    def forward(self, n, device):
        seq = torch.arange(n, device=device).type_as(self.inv_freq)
        freqs = (seq[:, None] * self.inv_freq[None, :]).repeat_interleave(2, dim=-1)[None]
        return [freqs.sin(), freqs.cos()]


class AxialRotaryEmbedding(nn.Module):
    """rotary.py:47-67."""

    def __init__(self, dim, max_freq=10):
        super().__init__()
        self.dim = dim // 2
        self.register_buffer('inv_freq', 1. / (10000 ** (torch.arange(0, self.dim, 2).float() / self.dim)))

    def forward(self, n, device):
        seq = torch.arange(n, device=device).type_as(self.inv_freq)
        f = seq[:, None] * self.inv_freq[None, :]                       # [n, dim/4]
        xs = f[:, None, :].expand(n, n, -1)
        ys = f[None, :, :].expand(n, n, -1)
        sin = torch.cat((xs.sin(), ys.sin()), dim=-1)
        cos = torch.cat((xs.cos(), ys.cos()), dim=-1)
        sin, cos = (t.reshape(1, n * n, -1).repeat_interleave(2, dim=-1) for t in (sin, cos))
        return [sin, cos]
