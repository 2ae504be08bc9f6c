"""Drop-in `SimpleViT` of `vit_pytorch.simple_vit_with_qk_norm` (reference simple_vit_with_qk_norm.py:29-141): SimpleViT
whose attention RMS-normalises queries and keys per head (learned `gamma[h, 1, d]`, initialised to 1/sqrt(d)) and uses
softmax scale 1.

Mirrored as the reference defines it, including its quirk that `linear_head` is `nn.LayerNorm(dim)` -- the model
returns (B, dim) normalised features and `num_classes` is unused (simple_vit_with_qk_norm.py:128,141).

Fused sm_90a path: the q / k normalisation runs right after the QKV GEMM
(`b200vit_gemm_headnorm_bf16`, built for NaViT), attention runs with scale 1, everything else is simple_vit's schedule.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from .engine import (FusedWeightsMixin, TransformerEngine, fused_mean_pooled_features, hooks_inside, on_device,
                     why_not_fused)
from .simple_vit import FeedForward, posemb_sincos_2d
from .vit import Patchify, pair


class RMSNorm(nn.Module):
    def __init__(self, heads: int, dim: int) -> None:
        super().__init__()
        self.scale = dim ** 0.5
        self.gamma = nn.Parameter(torch.ones(heads, 1, dim) / self.scale)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return F.normalize(x, dim=-1) * self.scale * self.gamma


class Attention(nn.Module):
    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.dim, self.dim_head = dim, dim_head
        self.project_out = True
        self.heads = heads
        self.softmax_scale = 1.0            # no dim_head ** -0.5: q and k are normalised (reference :75)
        self.scale = 1.0
        self.norm = nn.LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.q_norm = RMSNorm(heads, dim_head)
        self.k_norm = RMSNorm(heads, dim_head)
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        self.to_out = nn.Linear(inner_dim, dim, bias=False)

    def out_linear(self) -> nn.Linear:
        return self.to_out

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, n, _ = x.shape
        qkv = self.to_qkv(self.norm(x)).reshape(b, n, 3, self.heads, -1).permute(2, 0, 3, 1, 4)
        q, k, v = self.q_norm(qkv[0]), self.k_norm(qkv[1]), qkv[2]
        attn = self.attend(torch.matmul(q, k.transpose(-1, -2)))
        out = torch.matmul(attn, v).permute(0, 2, 1, 3).reshape(b, n, -1)
        return self.to_out(out)


class Transformer(FusedWeightsMixin, nn.Module):
    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int) -> None:
        super().__init__()
        self.dropout_p = 0.0
        self.norm = nn.LayerNorm(dim)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([Attention(dim, heads=heads, dim_head=dim_head), FeedForward(dim, mlp_dim)]))
        self._engine: Optional[TransformerEngine] = None

    def engine(self) -> TransformerEngine:
        if self._engine is None:
            self._engine = TransformerEngine(self)
        return self._engine

    def fused_reason(self, x: torch.Tensor) -> Optional[str]:
        if len(self.layers) == 0:
            return "depth == 0"
        r = why_not_fused(list(self.parameters()), x, training=self.training, dropout_p=0.0)
        if r is None and hooks_inside(self):
            r = "forward hooks registered inside the transformer"
        if r is None and x.dim() != 3:
            r = "input is not (B, N, D)"
        if r is None:
            r = self.engine().unsupported_reason(x.shape[1])
        return r

    def forward_eager(self, x: torch.Tensor) -> torch.Tensor:
        for attn, ff in self.layers:
            x = attn(x) + x
            x = ff(x) + x
        return self.norm(x)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(x) is None:
            return self.engine().forward_tokens(x)
        return self.forward_eager(x)


class SimpleViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, channels=3,
                 dim_head=64) -> None:
        super().__init__()
        image_height, image_width = pair(image_size)
        self.patch_size = patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, \
            'Image dimensions must be divisible by the patch size.'
        patch_dim = channels * patch_height * patch_width
        self.to_patch_embedding = nn.Sequential(
            Patchify(patch_height, patch_width),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.pos_embedding = posemb_sincos_2d(h=image_height // patch_height, w=image_width // patch_width, dim=dim)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim)
        self.pool = "mean"
        self.to_latent = nn.Identity()
        self.linear_head = nn.LayerNorm(dim)          # sic (reference :128): features, not logits
        self._patch_engine = None

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        if img.shape[1] * self.patch_size[0] * self.patch_size[1] != self.to_patch_embedding[1].normalized_shape[0]:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        if len(self.transformer.layers) == 0:
            return "depth == 0"
        r = why_not_fused(list(self.parameters()), img, training=self.training, dropout_p=0.0)
        if r is None and hooks_inside(self, skip=(self.to_latent, self.transformer)):
            r = "forward hooks registered inside the model"
        if r is None:
            ph, pw = self.patch_size
            if img.shape[2] % ph or img.shape[3] % pw:
                return "image not divisible by the patch size"
            n = (img.shape[2] // ph) * (img.shape[3] // pw)
            if n != self.pos_embedding.shape[0]:
                return "input resolution differs from image_size (the reference's add raises)"
            r = self.transformer.engine().unsupported_reason(n)
        return r

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    def forward_eager(self, img: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(img)
        x = x + self.pos_embedding.to(img.device, dtype=x.dtype)
        x = self.transformer(x).mean(dim=1)
        return self.linear_head(self.to_latent(x))

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        pm = fused_mean_pooled_features(self, img)
        pooled = torch.empty(pm.shape, device=img.device, dtype=torch.bfloat16)
        _lib.cast_f32_bf16(pm, pooled)
        lat = self.to_latent(pooled)                  # stays a called module (Dino / LeJEPA hook it)
        if lat is not pooled:
            pm = lat.float().contiguous()
        out = torch.empty(pm.shape, device=img.device, dtype=torch.bfloat16)
        h = self.linear_head
        _lib.layernorm(pm, h.weight.detach().float().contiguous(), h.bias.detach().float().contiguous(),
                       out_bf16=out, eps=h.eps)
        return out
