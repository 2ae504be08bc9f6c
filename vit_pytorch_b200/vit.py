"""Drop-in `ViT` for lucidrains/vit-pytorch's `vit_pytorch.ViT` with a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed) and the same attribute surface the reference's wrappers reach into
(`to_patch_embedding[0..3]`, `cls_token`, `pos_embedding`, `dropout`, `transformer`, `pool`, `to_latent`, `mlp_head`,
`patch_size`; reference vit.py:85-138, users: mae.py:25-31, simmim.py:19-25, recorder.py:26-28, extractor.py:46-59).

forward() dispatch:
  * CUDA sm_90 + bf16 parameters and input + no autograd recording + dropout inactive + no forward hooks inside the
    model  ->  hand-written kernels of libb200vit.so through the C ABI (engine.py).  If the library is missing or a
    kernel call fails this RAISES; there is no silent fallback for an eligible call.
  * anything else (CPU, fp32, training with dropout, Recorder/Extractor hooks) -> the plain PyTorch graph below, which
    keeps the module tree observable exactly like the reference's.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import (FusedWeightsMixin, HeadEngine, PatchEmbedEngine, TransformerEngine, hooked_transformer_tokens,
                     hooks_inside, ln_mode, on_device, transformer_is_hooked, why_not_fused)


def pair(t):
    return t if isinstance(t, tuple) else (t, t)


class Patchify(nn.Module):
    """'b c (h p1) (w p2) -> b (h w) (p1 p2 c)' (the Rearrange at reference vit.py:100), without einops."""

    def __init__(self, patch_height: int, patch_width: int) -> None:
        super().__init__()
        self.patch_height, self.patch_width = patch_height, patch_width

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        b, c, hh, ww = img.shape
        ph, pw = self.patch_height, self.patch_width
        gh, gw = hh // ph, ww // pw
        t = img.reshape(b, c, gh, ph, gw, pw).permute(0, 2, 4, 3, 5, 1)
        return t.reshape(b, gh * gw, ph * pw * c)

    def extra_repr(self) -> str:
        return f"p1={self.patch_height}, p2={self.patch_width}"


class FeedForward(nn.Module):
    """LayerNorm -> Linear -> GELU(erf) -> Dropout -> Linear -> Dropout (reference vit.py:15-28)."""

    def __init__(self, dim: int, hidden_dim: int, dropout: float = 0.) -> None:
        super().__init__()
        self.dim, self.hidden_dim = dim, hidden_dim
        self.net = nn.Sequential(
            nn.LayerNorm(dim),
            nn.Linear(dim, hidden_dim),
            nn.GELU(),
            nn.Dropout(dropout),
            nn.Linear(hidden_dim, dim),
            nn.Dropout(dropout),
        )

    def parts(self):
        return self.net[0], self.net[1], self.net[4]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.net(x)


class Attention(nn.Module):
    """Pre-LN multi-head self attention (reference vit.py:30-64)."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, dropout: float = 0.) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.dim, self.dim_head = dim, dim_head
        self.project_out = not (heads == 1 and dim_head == dim)
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.norm = nn.LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout)) if self.project_out \
            else nn.Identity()

    def out_linear(self) -> nn.Linear:
        return self.to_out[0]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, n, _ = x.shape
        h = self.heads
        qkv = self.to_qkv(self.norm(x)).reshape(b, n, 3, h, -1).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        dots = torch.matmul(q, k.transpose(-1, -2)) * self.scale
        attn = self.dropout(self.attend(dots))
        out = torch.matmul(attn, v).permute(0, 2, 1, 3).reshape(b, n, -1)
        return self.to_out(out)


class Transformer(FusedWeightsMixin, nn.Module):
    """depth x (attention, feed-forward) residual blocks + final LayerNorm (reference vit.py:66-83).

    Callable on arbitrary (B, N, D) tokens, as the reference's MAE / SimMIM / distillation wrappers do.
    """

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.) -> None:
        super().__init__()
        self.dropout_p = float(dropout)
        self.norm = nn.LayerNorm(dim)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))
        self._engine: Optional[TransformerEngine] = None

    def engine(self) -> TransformerEngine:
        if self._engine is None:
            self._engine = TransformerEngine(self)
        return self._engine

    def fused_reason(self, x: torch.Tensor) -> Optional[str]:
        """None if forward(x) will run the fused kernels, else why not."""
        if len(self.layers) == 0:
            return "depth == 0"
        r = why_not_fused(list(self.parameters()), x, training=self.training, dropout_p=self.dropout_p)
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


class ViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, pool='cls', channels=3,
                 dim_head=64, dropout=0., emb_dropout=0.) -> None:
        super().__init__()
        image_height, image_width = pair(image_size)
        self.patch_size = patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, \
            'Image dimensions must be divisible by the patch size.'
        num_patches = (image_height // patch_height) * (image_width // patch_width)
        patch_dim = channels * patch_height * patch_width
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        num_cls_tokens = 1 if pool == 'cls' else 0

        self.to_patch_embedding = nn.Sequential(
            Patchify(patch_height, patch_width),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.cls_token = nn.Parameter(torch.randn(num_cls_tokens, dim))
        self.pos_embedding = nn.Parameter(torch.randn(num_patches + num_cls_tokens, dim))
        self.dropout = nn.Dropout(emb_dropout)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim, dropout)
        self.pool = pool
        self.to_latent = nn.Identity()
        self.mlp_head = nn.Linear(dim, num_classes) if num_classes > 0 else None

        self._emb_dropout_p = float(emb_dropout)
        self._patch_engine: Optional[PatchEmbedEngine] = None
        self._head_engine: Optional[HeadEngine] = None

    # ---------------------------------------------------------------------------------------------- dispatch
    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        if img.shape[1] * self.patch_size[0] * self.patch_size[1] != self.to_patch_embedding[1].normalized_shape[0]:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        if len(self.transformer.layers) == 0:
            return "depth == 0"
        p_drop = max(self._emb_dropout_p, self.transformer.dropout_p)
        r = why_not_fused(list(self.parameters()), img, training=self.training, dropout_p=p_drop)
        if r is None and hooks_inside(self, skip=(self.to_latent, self.transformer)):
            r = "forward hooks registered inside the model"
        if r is None:
            ph, pw = self.patch_size
            if img.shape[2] % ph or img.shape[3] % pw:
                return "image not divisible by the patch size"
            n = (img.shape[2] // ph) * (img.shape[3] // pw) + self.cls_token.shape[0]
            r = self.transformer.engine().unsupported_reason(n)
        return r

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, img: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(img)
        cls = self.cls_token.unsqueeze(0).expand(x.shape[0], -1, -1)
        x = torch.cat((cls, x), dim=1)
        x = self.dropout(x + self.pos_embedding[: x.shape[1]])
        x = self.transformer(x)
        if self.mlp_head is None:
            return x
        x = x.mean(dim=1) if self.pool == 'mean' else x[:, 0]
        return self.mlp_head(self.to_latent(x))

    # ---------------------------------------------------------------------------------------------- fused kernels
    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        if self._patch_engine is None:
            self._patch_engine = PatchEmbedEngine(self)
        eng = self.transformer.engine()
        if transformer_is_hooked(self):                # Extractor (reference extractor.py:50-59): hook on .transformer
            x, B, N = self._patch_engine.run(img)
            out = hooked_transformer_tokens(self, x, B, N)
            if self.mlp_head is None:
                return out
            pooled = (out.mean(dim=1) if self.pool == 'mean' else out[:, 0]).contiguous()
            pooled = self.to_latent(pooled)
            if self._head_engine is None:
                self._head_engine = HeadEngine(self.mlp_head)
            return self._head_engine.run(pooled)
        B, N = self._patch_engine.geometry(img)
        primed = ln_mode() == "fold"
        ws = eng.workspace(B * N, img.device) if primed else None
        x, B, N = self._patch_engine.run(img, xb=ws["xn"] if primed else None,
                                         stats=ws["stats_in"] if primed else None)   # fp32 residual stream [B*N, D]
        D = x.shape[1]
        eng.run_blocks(x, B, N, primed=primed)
        dev = img.device
        if self.mlp_head is None:                      # reference vit.py:132-133: return the normalised tokens
            out = torch.empty(B * N, D, device=dev, dtype=torch.bfloat16)
            eng.final_norm(x, out_bf16=out)
            return out.view(B, N, D)
        pooled = torch.empty(B, D, device=dev, dtype=torch.bfloat16)
        if self.pool == 'mean':
            xf = torch.empty_like(x)
            eng.final_norm(x, out_f32=xf)
            pm = torch.empty(B, D, device=dev, dtype=torch.float32)
            _lib.mean_pool(xf, pm, B, N, D)
            _lib.cast_f32_bf16(pm, pooled)
        else:                                          # LayerNorm is per token: normalise only the cls rows
            rows = torch.arange(0, B * N, N, device=dev, dtype=torch.int32)
            eng.final_norm(x, out_bf16=pooled, row_index=rows)
        pooled = self.to_latent(pooled)                # stays a called module: Dino / LeJEPA hook it
        if self._head_engine is None:
            self._head_engine = HeadEngine(self.mlp_head)
        return self._head_engine.run(pooled)
