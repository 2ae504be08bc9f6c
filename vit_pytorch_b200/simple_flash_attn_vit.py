"""Drop-in `SimpleViT` of `vit_pytorch.simple_flash_attn_vit` (reference simple_flash_attn_vit.py:25-176): the SimpleViT
twin whose attention calls `F.scaled_dot_product_attention` (`use_flash=True`, the default) or the explicit
softmax(q k^T) v (`use_flash=False`), whose Transformer has NO final LayerNorm, and whose head is
`Sequential(LayerNorm, Linear)`; the sin-cos table is built from the input's own patch grid on every call.

Both `use_flash` settings compute the same function; on the fused sm_90a path both are this repo's own attention
kernel (the flag only selects the PyTorch operator of the eager graph, exactly as in the reference).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from .engine import (FusedWeightsMixin, HeadEngine, TransformerEngine, fused_mean_pooled_features, hooks_inside,
                     on_device, why_not_fused)
from .simple_vit import FeedForward, posemb_sincos_2d
from .simple_vit_with_patch_dropout import GridPatchify
from .vit import pair


class Attend(nn.Module):
    def __init__(self, use_flash: bool = False) -> None:
        super().__init__()
        self.use_flash = use_flash

    def forward(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
        if self.use_flash:
            return F.scaled_dot_product_attention(q, k, v)
        sim = torch.matmul(q, k.transpose(-1, -2)) * q.shape[-1] ** -0.5
        return torch.matmul(sim.softmax(dim=-1), v)


class Attention(nn.Module):
    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, use_flash: bool = True) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.dim, self.dim_head = dim, dim_head
        self.project_out = True
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.norm = nn.LayerNorm(dim)
        self.attend = Attend(use_flash=use_flash)
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        self.to_out = nn.Linear(inner_dim, dim, bias=False)

    def out_linear(self) -> nn.Linear:
        return self.to_out

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, n, _ = x.shape
        qkv = self.to_qkv(self.norm(x)).reshape(b, n, 3, self.heads, -1).permute(2, 0, 3, 1, 4)
        out = self.attend(qkv[0], qkv[1], qkv[2])
        return self.to_out(out.permute(0, 2, 1, 3).reshape(b, n, -1))


class Transformer(FusedWeightsMixin, nn.Module):
    """No final LayerNorm (reference :117-131)."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, use_flash: bool) -> None:
        super().__init__()
        self.dropout_p = 0.0
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, use_flash=use_flash),
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
        return x

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(x) is None:
            return self.engine().forward_tokens(x)
        return self.forward_eager(x)


class SimpleViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, channels=3, dim_head=64,
                 use_flash=True) -> None:
        super().__init__()
        image_height, image_width = pair(image_size)
        self.patch_size = patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, \
            'Image dimensions must be divisible by the patch size.'
        patch_dim = channels * patch_height * patch_width
        self.to_patch_embedding = nn.Sequential(
            GridPatchify(patch_height, patch_width),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim, use_flash)
        self.to_latent = nn.Identity()
        self.linear_head = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, num_classes))
        self._dim = dim
        self._patch_engine = None
        self._head_engine: Optional[HeadEngine] = None

    def fused_pos_table(self, gh: int, gw: int) -> torch.Tensor:
        return posemb_sincos_2d(gh, gw, self._dim)

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
            r = self.transformer.engine().unsupported_reason((img.shape[2] // ph) * (img.shape[3] // pw))
        return r

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    def forward_eager(self, img: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(img)
        b, gh, gw, d = x.shape
        pe = posemb_sincos_2d(gh, gw, d).to(device=x.device, dtype=x.dtype)
        x = self.transformer(x.reshape(b, gh * gw, d) + pe).mean(dim=1)
        return self.linear_head(self.to_latent(x))

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        pm = fused_mean_pooled_features(self, img)              # fp32 mean of the un-normalised tokens
        pooled = torch.empty(pm.shape, device=img.device, dtype=torch.bfloat16)
        _lib.cast_f32_bf16(pm, pooled)
        lat = self.to_latent(pooled)
        if lat is not pooled:
            pm = lat.float().contiguous()
        ln, lin = self.linear_head[0], self.linear_head[1]
        normed = torch.empty(pm.shape, device=img.device, dtype=torch.bfloat16)
        _lib.layernorm(pm, ln.weight.detach().float().contiguous(), ln.bias.detach().float().contiguous(),
                       out_bf16=normed, eps=ln.eps)
        if self._head_engine is None:
            self._head_engine = HeadEngine(lin)
        return self._head_engine.run(normed)
