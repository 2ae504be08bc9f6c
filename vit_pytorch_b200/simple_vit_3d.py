"""Drop-in `SimpleViT` of `vit_pytorch.simple_vit_3d` (reference simple_vit_3d.py:12-128): SimpleViT over a video
`(B, C, F, H, W)` cut into `frame_patch_size x p1 x p2` boxes, 3-D sin-cos positions built from the patch grid on every
call, mean pool, linear head.

Same constructor keywords, parameter names / registration order (=> identical `state_dict`, identical init under one
seed).  The encoder blocks are simple_vit's.  On the fused sm_90a path the video is handed to the 2-D patch kernels
as a `(B, C, F' * H, W)` image: with `frame_patch_size == 1` that is the video's own memory (a view; 16 x 16 boxes then
go through the TMA patch embedding), otherwise one device-side permute first puts the `pf` frames of a box under each
other so that `(pf p1)` becomes the box height -- `'(pf p1 p2 c)'` (reference :97) is the 2-D `(p1' p2 c)` order with
`p1' = pf * p1`.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from .engine import FusedWeightsMixin, HeadEngine, fused_mean_pooled_features, hooks_inside, on_device, why_not_fused
from .simple_vit import Attention, FeedForward, Transformer  # noqa: F401  (same block classes, reference :36-88)
from .vit import pair


def sincos_table_3d(f: int, h: int, w: int, dim: int, temperature: int = 10000, device=None) -> torch.Tensor:
    """fp32 table [(f h w), dim] of reference simple_vit_3d.py:12-34."""
    z, y, x = torch.meshgrid(torch.arange(f, device=device), torch.arange(h, device=device),
                             torch.arange(w, device=device), indexing='ij')
    fourier_dim = dim // 6
    omega = torch.arange(fourier_dim, device=device) / (fourier_dim - 1)
    omega = 1. / (temperature ** omega)
    z = z.flatten()[:, None] * omega[None, :]
    y = y.flatten()[:, None] * omega[None, :]
    x = x.flatten()[:, None] * omega[None, :]
    pe = torch.cat((x.sin(), x.cos(), y.sin(), y.cos(), z.sin(), z.cos()), dim=1)
    return F.pad(pe, (0, dim - (fourier_dim * 6)))       # pad if the feature dimension is not divisible by 6


def posemb_sincos_3d(patches: torch.Tensor, temperature: int = 10000, dtype: torch.dtype = torch.float32
                     ) -> torch.Tensor:
    _, f, h, w, dim = patches.shape
    return sincos_table_3d(f, h, w, dim, temperature, patches.device).type(patches.dtype)


class VideoPatchify(nn.Module):
    """`Rearrange('b c (f pf) (h p1) (w p2) -> b f h w (pf p1 p2 c)')` (reference :97); parameter-free."""

    def __init__(self, pf: int, p1: int, p2: int) -> None:
        super().__init__()
        self.pf, self.p1, self.p2 = pf, p1, p2

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, c, ft, ht, wt = x.shape
        f, h, w = ft // self.pf, ht // self.p1, wt // self.p2
        x = x.reshape(b, c, f, self.pf, h, self.p1, w, self.p2).permute(0, 2, 4, 6, 3, 5, 7, 1)
        return x.reshape(b, f, h, w, self.pf * self.p1 * self.p2 * c)


class SimpleViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, image_patch_size, frames, frame_patch_size, num_classes, dim, depth, heads,
                 mlp_dim, channels=3, dim_head=64) -> None:
        super().__init__()
        image_height, image_width = pair(image_size)
        self.patch_size = patch_height, patch_width = pair(image_patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, \
            'Image dimensions must be divisible by the patch size.'
        assert frames % frame_patch_size == 0, 'Frames must be divisible by the frame patch size'
        patch_dim = channels * patch_height * patch_width * frame_patch_size
        self.to_patch_embedding = nn.Sequential(
            VideoPatchify(frame_patch_size, patch_height, patch_width),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim)
        self.to_latent = nn.Identity()
        self.linear_head = nn.Linear(dim, num_classes)
        self.fused_patch_box: Tuple[int, int] = (frame_patch_size * patch_height, patch_width)
        self._pf = frame_patch_size
        self._channels = channels
        self._patch_engine = None
        self._head_engine: Optional[HeadEngine] = None
        self._pos_cache: Dict[Tuple[int, int, int, str], torch.Tensor] = {}

    def _grid(self, video: torch.Tensor) -> Tuple[int, int, int]:
        return video.shape[2] // self._pf, video.shape[3] // self.patch_size[0], video.shape[4] // self.patch_size[1]

    def fused_reason(self, video: torch.Tensor) -> Optional[str]:
        if video.dim() != 5:
            return "input is not (B, C, F, H, W)"
        if video.shape[1] != self._channels:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        if video.shape[2] % self._pf or video.shape[3] % self.patch_size[0] or video.shape[4] % self.patch_size[1]:
            return "video not divisible by the patch box"
        if len(self.transformer.layers) == 0:
            return "depth == 0"
        r = why_not_fused(list(self.parameters()), video, training=self.training, dropout_p=0.0)
        if r is None and hooks_inside(self, skip=(self.to_latent, self.transformer)):
            r = "forward hooks registered inside the model"
        if r is None:
            f, h, w = self._grid(video)
            if f * h * w == 0:
                return "empty patch grid"
            if self.fused_patch_box[0] * video.shape[4] * video.shape[1] * 2 > 200 * 1024:
                return "one row of patch boxes exceeds the patch kernel's shared-memory slab"
            r = self.transformer.engine().unsupported_reason(f * h * w)
        return r

    def forward(self, video: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(video) is None:
            with on_device(video):
                return self.forward_fused(video)
        return self.forward_eager(video)

    def forward_eager(self, video: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(video)
        pe = posemb_sincos_3d(x)
        x = x.flatten(1, 3) + pe
        x = self.transformer(x)
        x = x.mean(dim=1)
        return self.linear_head(self.to_latent(x))

    def forward_fused(self, video: torch.Tensor) -> torch.Tensor:
        b, c, ft, ht, wt = video.shape
        f, h, w = self._grid(video)
        p1 = self.patch_size[0]
        if self._pf == 1:
            img = video.contiguous().view(b, c, ft * ht, wt)
        else:
            # (f pf) (h p1) -> (f h pf p1): the pf frames of one box under each other; token order (f h w) unchanged
            img = video.reshape(b, c, f, self._pf, h, p1, wt).permute(0, 1, 2, 4, 3, 5, 6).reshape(b, c, ft * ht, wt)
        dim = self.linear_head.in_features
        key = (f, h, w, str(video.device))
        if key not in self._pos_cache:
            self._pos_cache[key] = sincos_table_3d(f, h, w, dim, device=video.device).contiguous()
        pm = fused_mean_pooled_features(self, img, patch=self.fused_patch_box, pos=self._pos_cache[key])
        pooled = torch.empty(pm.shape, device=video.device, dtype=torch.bfloat16)
        _lib.cast_f32_bf16(pm, pooled)
        pooled = self.to_latent(pooled)
        if self._head_engine is None:
            self._head_engine = HeadEngine(self.linear_head)
        return self._head_engine.run(pooled)
