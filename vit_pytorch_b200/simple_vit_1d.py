"""Drop-in `SimpleViT` of `vit_pytorch.simple_vit_1d` (reference simple_vit_1d.py:9-112): SimpleViT over a series
`(B, C, L)` cut into `L / patch_size` patches of `patch_size * C` values, 1-D sin-cos positions built from the token
matrix on every call, mean pool, linear head.

Same constructor keywords, parameter names / registration order (=> identical `state_dict`, identical init under one
seed).  The encoder blocks are simple_vit's; on the fused sm_90a path the series is handed to the patch kernels as a
`(B, C, 1, L)` image with a `1 x patch_size` patch box -- `'b c (n p) -> b n (p c)'` (reference :84) is the 2-D
`(p1 p2 c)` order with `p1 = 1` -- so no new kernel is involved.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import FusedWeightsMixin, HeadEngine, fused_mean_pooled_features, hooks_inside, on_device, why_not_fused
from .simple_vit import Attention, FeedForward, Transformer  # noqa: F401  (same block classes, reference :23-76)


def posemb_sincos_1d(patches: torch.Tensor, temperature: int = 10000, dtype: torch.dtype = torch.float32
                     ) -> torch.Tensor:
    """Reference simple_vit_1d.py:9-19 (the `dtype` argument is shadowed by the token dtype there too)."""
    n, dim = patches.shape[1], patches.shape[2]
    return sincos_table_1d(n, dim, temperature, patches.device).type(patches.dtype)


def sincos_table_1d(n: int, dim: int, temperature: int = 10000, device=None) -> torch.Tensor:
    assert (dim % 2) == 0, 'feature dimension must be multiple of 2 for sincos emb'
    omega = torch.arange(dim // 2, device=device) / (dim // 2 - 1)
    omega = 1. / (temperature ** omega)
    t = torch.arange(n, device=device)[:, None] * omega[None, :]
    return torch.cat((t.sin(), t.cos()), dim=1)


class SeriesPatchify(nn.Module):
    """`Rearrange('b c (n p) -> b n (p c)', p = patch_size)` (reference :84); parameter-free."""

    def __init__(self, p: int) -> None:
        super().__init__()
        self.p = p

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, c, length = x.shape
        return x.reshape(b, c, length // self.p, self.p).permute(0, 2, 3, 1).reshape(b, length // self.p, self.p * c)


class SimpleViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, seq_len, patch_size, num_classes, dim, depth, heads, mlp_dim, channels=3, dim_head=64
                 ) -> None:
        super().__init__()
        assert seq_len % patch_size == 0
        patch_dim = channels * patch_size
        self.to_patch_embedding = nn.Sequential(
            SeriesPatchify(patch_size),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim)
        self.to_latent = nn.Identity()
        self.linear_head = nn.Linear(dim, num_classes)
        self.fused_patch_box: Tuple[int, int] = (1, patch_size)
        self._channels = channels
        self._patch_engine = None
        self._head_engine: Optional[HeadEngine] = None
        self._pos_cache: Dict[Tuple[int, str], torch.Tensor] = {}

    def fused_reason(self, series: torch.Tensor) -> Optional[str]:
        if series.dim() != 3:
            return "input is not (B, C, L)"
        p = self.fused_patch_box[1]
        if series.shape[1] != self._channels:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        if series.shape[2] % p or series.shape[2] == 0:
            return "series length not divisible by the patch size"
        if len(self.transformer.layers) == 0:
            return "depth == 0"
        r = why_not_fused(list(self.parameters()), series, training=self.training, dropout_p=0.0)
        if r is None and hooks_inside(self, skip=(self.to_latent, self.transformer)):
            r = "forward hooks registered inside the model"
        if r is None:
            r = self.transformer.engine().unsupported_reason(series.shape[2] // p)
        return r

    def forward(self, series: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(series) is None:
            with on_device(series):
                return self.forward_fused(series)
        return self.forward_eager(series)

    def forward_eager(self, series: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(series)
        x = x + posemb_sincos_1d(x)
        x = self.transformer(x)
        x = x.mean(dim=1)
        return self.linear_head(self.to_latent(x))

    def forward_fused(self, series: torch.Tensor) -> torch.Tensor:
        b, c, length = series.shape
        n = length // self.fused_patch_box[1]
        dim = self.linear_head.in_features
        key = (n, str(series.device))
        if key not in self._pos_cache:
            self._pos_cache[key] = sincos_table_1d(n, dim, device=series.device).contiguous()
        pm = fused_mean_pooled_features(self, series.contiguous().view(b, c, 1, length), patch=self.fused_patch_box,
                                        pos=self._pos_cache[key])
        pooled = torch.empty(pm.shape, device=series.device, dtype=torch.bfloat16)
        _lib.cast_f32_bf16(pm, pooled)
        pooled = self.to_latent(pooled)
        if self._head_engine is None:
            self._head_engine = HeadEngine(self.linear_head)
        return self._head_engine.run(pooled)
