"""Drop-in `SimpleViT` of `vit_pytorch.simple_vit_with_patch_dropout` (reference
simple_vit_with_patch_dropout.py:27-141): SimpleViT that, IN TRAINING, keeps a random subset of the patch tokens
(`PatchDropout`), and builds its sin-cos positional table from the input's own patch grid on every call (so any
resolution divisible by the patch size is accepted).

In eval mode `PatchDropout` is the identity (reference :34-35) and the fused sm_90a path is simple_vit's schedule;
in training with prob > 0 the PyTorch graph runs (random token subsets are a training-time feature, the fused path
is forward only).
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from .engine import FusedWeightsMixin, classify, common_reason, fused_mean_pooled_features, on_device
from .simple_vit import Transformer, posemb_sincos_2d
from .vit import Patchify, pair


class PatchDropout(nn.Module):
    def __init__(self, prob: float) -> None:
        super().__init__()
        assert 0 <= prob < 1.
        self.prob = prob

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not self.training or self.prob == 0.:
            return x
        b, n, _ = x.shape
        keep = max(1, int(n * (1 - self.prob)))
        idx = torch.randn(b, n, device=x.device).topk(keep, dim=-1).indices
        return x[torch.arange(b, device=x.device)[:, None], idx]


class GridPatchify(Patchify):
    """'b c (h p1) (w p2) -> b h w (p1 p2 c)': patch vectors with the grid kept (reference :114)."""

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        b = img.shape[0]
        gh, gw = img.shape[2] // self.patch_height, img.shape[3] // self.patch_width
        return super().forward(img).reshape(b, gh, gw, -1)


class SimpleViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, channels=3, dim_head=64,
                 patch_dropout=0.5) -> None:
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
        self.patch_dropout = PatchDropout(patch_dropout)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim)
        self.to_latent = nn.Identity()
        self.linear_head = nn.Linear(dim, num_classes)
        self._dim = dim

    def fused_pos_table(self, gh: int, gw: int) -> torch.Tensor:
        return posemb_sincos_2d(gh, gw, self._dim)

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        if img.shape[1] * self.patch_size[0] * self.patch_size[1] != self.to_patch_embedding[1].normalized_shape[0]:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        if len(self.transformer.layers) == 0:
            return "depth == 0"
        if self.training and self.patch_dropout.prob > 0.:
            return "patch dropout is active (training)"
        r = common_reason(self, img, skip=(self.to_latent, self.transformer))
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
        x = x.reshape(b, gh * gw, d) + pe
        x = self.patch_dropout(x)
        x = self.transformer(x).mean(dim=1)
        return self.linear_head(self.to_latent(x))

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        _, pooled = fused_mean_pooled_features(self, img)
        return classify(self, self.linear_head, pooled)
