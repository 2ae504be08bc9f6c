"""Drop-in `SimpleViT` for `vit_pytorch.SimpleViT` (reference simple_vit.py:80-120) with a fused sm_90a forward.

Differences from vit.ViT that the reference defines and this mirrors: no cls token and no dropout modules, a fixed
2-D sin-cos positional table kept as a plain tensor attribute (not a parameter / buffer, so it is absent from
`state_dict` and is cast per call, simple_vit.py:97-101,114), bias-free `to_out` Linear (simple_vit.py:48),
FeedForward Sequential indices 0..3 (simple_vit.py:28-33), mean pooling and a head called `linear_head`.
Dispatch rules are those of vit.ViT.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from . import _lib
from .engine import (FusedWeightsMixin, HeadEngine, PatchEmbedEngine, TransformerEngine, fused_mean_pooled_features,
                     hooks_inside, ln_mode, on_device, transformer_is_hooked, why_not_fused)
from .vit import Patchify, pair


def posemb_sincos_2d(h: int, w: int, dim: int, temperature: int = 10000, dtype=torch.float32) -> torch.Tensor:
    """[h*w, dim] table: concat(sin(x w_i), cos(x w_i), sin(y w_i), cos(y w_i)), w_i = T^(-i/(dim/4-1)),
    token index = y*w + x (reference simple_vit.py:12-21)."""
    assert (dim % 4) == 0, "feature dimension must be multiple of 4 for sincos emb"
    quarter = dim // 4
    omega = 1.0 / (temperature ** (torch.arange(quarter) / (quarter - 1)))
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    ya = yy.reshape(-1, 1) * omega.reshape(1, -1)
    xa = xx.reshape(-1, 1) * omega.reshape(1, -1)
    return torch.cat((xa.sin(), xa.cos(), ya.sin(), ya.cos()), dim=1).type(dtype)


class FeedForward(nn.Module):
    def __init__(self, dim: int, hidden_dim: int) -> None:
        super().__init__()
        self.dim, self.hidden_dim = dim, hidden_dim
        self.net = nn.Sequential(
            nn.LayerNorm(dim),
            nn.Linear(dim, hidden_dim),
            nn.GELU(),
            nn.Linear(hidden_dim, dim),
        )

    def parts(self):
        return self.net[0], self.net[1], self.net[3]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.net(x)


class Attention(nn.Module):
    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.dim, self.dim_head = dim, dim_head
        self.project_out = True
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.norm = nn.LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        self.to_out = nn.Linear(inner_dim, dim, bias=False)

    def out_linear(self) -> nn.Linear:
        return self.to_out

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, n, _ = x.shape
        qkv = self.to_qkv(self.norm(x)).reshape(b, n, 3, self.heads, -1).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        attn = self.attend(torch.matmul(q, k.transpose(-1, -2)) * self.scale)
        out = torch.matmul(attn, v).permute(0, 2, 1, 3).reshape(b, n, -1)
        return self.to_out(out)


class Transformer(FusedWeightsMixin, nn.Module):
    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int) -> None:
        super().__init__()
        self.dropout_p = 0.0
        self.norm = nn.LayerNorm(dim)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head),
                FeedForward(dim, mlp_dim),
            ]))
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
        self.pos_embedding = posemb_sincos_2d(
            h=image_height // patch_height,
            w=image_width // patch_width,
            dim=dim,
        )
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim)
        self.pool = "mean"
        self.to_latent = nn.Identity()
        self.linear_head = nn.Linear(dim, num_classes)

        self._patch_engine: Optional[PatchEmbedEngine] = None
        self._head_engine: Optional[HeadEngine] = None

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
                return "input resolution differs from image_size (the reference's add at simple_vit.py:114 raises)"
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
        x = self.transformer(x)
        x = x.mean(dim=1)
        return self.linear_head(self.to_latent(x))

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        if self._patch_engine is None:
            self._patch_engine = PatchEmbedEngine(self)
        eng = self.transformer.engine()
        dev = img.device
        if transformer_is_hooked(self):                # Extractor-style hook on .transformer: tokens through the module
            pm = fused_mean_pooled_features(self, img)
            B, D = pm.shape
        else:
            B, N = self._patch_engine.geometry(img)
            primed = ln_mode() == "fold"
            ws = eng.workspace(B * N, img.device) if primed else None
            x, B, N = self._patch_engine.run(img, xb=ws["xn"] if primed else None,
                                             stats=ws["stats_in"] if primed else None)
            D = x.shape[1]
            eng.run_blocks(x, B, N, primed=primed)
            xf = torch.empty_like(x)
            eng.final_norm(x, out_f32=xf)
            pm = torch.empty(B, D, device=dev, dtype=torch.float32)
            _lib.mean_pool(xf, pm, B, N, D)
        pooled = torch.empty(B, D, device=dev, dtype=torch.bfloat16)
        _lib.cast_f32_bf16(pm, pooled)
        pooled = self.to_latent(pooled)
        if self._head_engine is None:
            self._head_engine = HeadEngine(self.linear_head)
        return self._head_engine.run(pooled)
