"""Drop-in `SimpleViT` of `vit_pytorch.simple_vit_with_register_tokens` (reference
simple_vit_with_register_tokens.py:85-134): SimpleViT plus `num_register_tokens` learned tokens appended to every
image's sequence (no positional embedding on them), dropped again before the mean pool.

Same constructor keywords, parameter names / registration order (=> identical `state_dict` and identical init under one
seed) as the reference.  The encoder blocks are exactly simple_vit's, so the fused sm_90a path is the same kernel
schedule on N = patches + registers tokens; the registers are written by the token-assembly kernel
(`b200vit_embed_tokens`, tail rows) and the pooling kernel averages only the patch tokens.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from . import _lib
from .engine import FusedWeightsMixin, HeadEngine, fused_mean_pooled_features, hooks_inside, on_device, why_not_fused
from .simple_vit import Attention, FeedForward, Transformer, posemb_sincos_2d  # noqa: F401  (same block classes)
from .vit import Patchify, pair


class SimpleViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, num_register_tokens=4,
                 channels=3, dim_head=64) -> None:
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
        self.register_tokens = nn.Parameter(torch.randn(num_register_tokens, dim))
        self.pos_embedding = posemb_sincos_2d(h=image_height // patch_height, w=image_width // patch_width, dim=dim)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim)
        self.pool = "mean"
        self.to_latent = nn.Identity()
        self.linear_head = nn.Linear(dim, num_classes)
        self._patch_engine = None
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
                return "input resolution differs from image_size (the reference's add raises)"
            r = self.transformer.engine().unsupported_reason(n + self.register_tokens.shape[0])
        return r

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    def forward_eager(self, img: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(img)
        x = x + self.pos_embedding.to(img.device, dtype=x.dtype)
        n = x.shape[1]
        r = self.register_tokens.unsqueeze(0).expand(x.shape[0], -1, -1)
        x = self.transformer(torch.cat((x, r), dim=1))
        x = x[:, :n].mean(dim=1)
        return self.linear_head(self.to_latent(x))

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        n = self.pos_embedding.shape[0]
        pm = fused_mean_pooled_features(self, img, pool_tokens=n)     # mean over the patch tokens only
        pooled = torch.empty(pm.shape, device=img.device, dtype=torch.bfloat16)
        _lib.cast_f32_bf16(pm, pooled)
        pooled = self.to_latent(pooled)
        if self._head_engine is None:
            self._head_engine = HeadEngine(self.linear_head)
        return self._head_engine.run(pooled)
