"""Drop-in `ViTND` for lucidrains/vit-pytorch's `vit_pytorch.vit_nd.ViTND` (inputs of any rank 1..7: signals, images,
video, volumes) with a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed), including the 3-D `cls_token` (1, 1, dim) and `pos_embedding` (1, n + 1, dim)
(reference vit_nd.py:89-170).  The Transformer is vit.Transformer, whose module tree is the reference's
(vit_nd.py:23-87).

Fused forward (engine.py): b200vit_patchify_nd -> patch GEMM + bias -> b200vit_embed_tokens (LayerNorm(dim), cls, pos;
primes the LN-folded layer chain) -> encoder blocks -> final LayerNorm -> cls row, or the mean over the patch tokens
x[:, 1:] (vit_nd.py:167) -> head GEMM.  Anything the fused path does not cover runs the PyTorch graph below, which
mirrors the reference module for module (Recorder / Extractor hooks keep working there).
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import torch
from torch import nn

from . import _lib
from .engine import FusedWeightsMixin, _Prepared, _bf16_rows, _f32, classify, common_reason, on_device
from .vit import Transformer

MAX_FUSED_PATCH_DIM = 16384      # b200vit_patchify_nd stages at least one whole patch in shared memory


def ensure_tuple(t, length: int) -> tuple:
    if isinstance(t, (tuple, list)):
        assert len(t) == length, f'Expected tuple of length {length}, got {len(t)}'
        return tuple(t)
    return (t,) * length


class PatchifyND(nn.Module):
    """'b c (f p0) (g p1) ... -> b (f g ...) (p0 p1 ... c)' (the Rearrange at reference vit_nd.py:130-142), without
    einops.  flatten=False keeps the patch grid: 'b c (f p0) ... -> b f g ... (p0 p1 ... c)' (vit_nd_rotary.py:222)."""

    def __init__(self, patch_size: Sequence[int], flatten: bool = True) -> None:
        super().__init__()
        self.patch_size, self.flatten = tuple(patch_size), flatten

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, c, *shape = x.shape
        r = len(self.patch_size)
        if len(shape) != r:
            raise ValueError(f"expected an input of rank {r} after (batch, channels), got shape {tuple(x.shape)}")
        split = []
        for s, p in zip(shape, self.patch_size):
            if s % p:
                raise ValueError(f"input extent {s} is not divisible by the patch size {p}")
            split += [s // p, p]
        t = x.reshape(b, c, *split)
        # (b, c, g0, p0, g1, p1, ...) -> (b, g0, g1, ..., p0, p1, ..., c)
        t = t.permute(0, *range(2, 2 + 2 * r, 2), *range(3, 3 + 2 * r, 2), 1)
        grid = [s // p for s, p in zip(shape, self.patch_size)]
        return t.reshape(b, math.prod(grid), -1) if self.flatten else t.reshape(b, *grid, -1)

    def extra_repr(self) -> str:
        return f"patch_size={self.patch_size}"


class NdPatchEngine:
    """Fused N-d patch embedding + token assembly of ViTND and the rotary ViTND: b200vit_patchify_nd -> patch GEMM
    (+ bias) -> b200vit_embed_tokens (LayerNorm(dim), then the cls row and the positional table when the model has
    them)."""

    def __init__(self, owner: nn.Module, patch_size: Tuple[int, ...]) -> None:
        self.owner, self.patch_size = owner, patch_size
        self.prep = _Prepared()

    def params(self) -> List[torch.Tensor]:
        o = self.owner
        ps = list(o.to_patch_embedding.parameters())
        for name in ("cls_token", "pos_embedding"):
            v = getattr(o, name, None)
            if isinstance(v, nn.Parameter):
                ps.append(v)
        return ps

    def prepared(self, device: torch.device) -> dict:
        return self.prep.get(self.params(), self._build, str(device))

    def _build(self) -> dict:
        o = self.owner
        lin, ln = o.to_patch_embedding[1], o.to_patch_embedding[2]
        D, pd = lin.weight.shape
        cls, pos = getattr(o, "cls_token", None), getattr(o, "pos_embedding", None)
        return {"w": _bf16_rows(lin.weight, (pd + 63) // 64 * 64), "b": _f32(lin.bias),
                "ln.w": _f32(ln.weight), "ln.b": _f32(ln.bias),
                "cls": None if cls is None else _f32(cls.reshape(-1, D)),
                "pos": None if pos is None else _f32(pos.reshape(-1, D))}

    def tokens(self, img: torch.Tensor) -> Tuple[int, int]:
        """(patches per input, tokens per input)."""
        n = math.prod(s // p for s, p in zip(img.shape[2:], self.patch_size))
        return n, n + (0 if getattr(self.owner, "cls_token", None) is None else 1)

    def run(self, img: torch.Tensor, xb: Optional[torch.Tensor] = None,
            stats: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, int, int]:
        """img [B, C, S_0 .. S_{r-1}] bf16 -> (x fp32 [B*N, D], B, N); optionally also the bf16 copy of x and its row
        sums (the entry statistics of the LN-folded layer chain)."""
        t = self.prepared(img.device)
        B = img.shape[0]
        n, N = self.tokens(img)
        D = t["w"].shape[0]
        dev = img.device
        a = torch.empty(B * n, t["w"].shape[1], device=dev, dtype=torch.bfloat16)
        _lib.patchify_nd(img.contiguous(), a, self.patch_size)
        y = torch.empty(B * n, D, device=dev, dtype=torch.float32)
        _lib.gemm(a, t["w"], out_f32=y, bias=t["b"])
        x = torch.empty(B * N, D, device=dev, dtype=torch.float32)
        _lib.embed_tokens(y, t["ln.w"], t["ln.b"], t["cls"], t["pos"], x, B, n, N - n, xb=xb, stats=stats,
                          eps=self.owner.to_patch_embedding[2].eps)
        return x, B, N


def nd_fused_reason(owner: nn.Module, img: torch.Tensor, patch_size: Tuple[int, ...], dropout_p: float
                    ) -> Optional[str]:
    """The dispatch rules both ViTNDs share (those of vit.ViT, plus the input's rank and divisibility)."""
    r = len(patch_size)
    if img.dim() != 2 + r:
        return f"input is not (B, C) + {r} spatial dims"
    lin = owner.to_patch_embedding[1]
    if img.shape[1] * math.prod(patch_size) != lin.in_features:
        return "channel count differs from the constructor's (the reference's Linear raises)"
    if any(s % p for s, p in zip(img.shape[2:], patch_size)):
        return "input not divisible by the patch size"
    reason = common_reason(owner, img, encoders=(owner.transformer,), dropout_p=dropout_p, skip=(owner.to_latent,))
    if reason is None and lin.in_features > MAX_FUSED_PATCH_DIM:
        reason = f"patch_dim {lin.in_features} > {MAX_FUSED_PATCH_DIM}"
    return reason


def nd_encode(owner: nn.Module, pe: NdPatchEngine, img: torch.Tensor,
              rope: Optional[Tuple[torch.Tensor, int]] = None) -> Tuple[torch.Tensor, int, int]:
    """Patch embedding -> encoder blocks: (x fp32 [B*N, D] before the final LayerNorm, B, N).  In fold mode the token
    assembly also writes the engine's bf16 copy of x and its row statistics.  Must run inside on_device(img)."""
    eng = owner.transformer.engine()
    xb, stats = eng.entry_buffers(img.shape[0] * pe.tokens(img)[1], img.device)
    x, B, N = pe.run(img, xb=xb, stats=stats)
    eng.run_blocks(x, B, N, primed=xb is not None, rope=rope)
    return x, B, N


class ViTND(FusedWeightsMixin, nn.Module):
    def __init__(self, *, ndim: int, input_shape, patch_size, num_classes: int, dim: int, depth: int, heads: int,
                 mlp_dim: int, pool: str = 'cls', channels: int = 3, dim_head: int = 64, dropout: float = 0.,
                 emb_dropout: float = 0.) -> None:
        super().__init__()
        assert 1 <= ndim <= 7, 'ndim must be between 1 and 7'
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        self.ndim = ndim
        self.pool = pool
        input_shape = ensure_tuple(input_shape, ndim)
        patch_size = ensure_tuple(patch_size, ndim)
        for i, (s, p) in enumerate(zip(input_shape, patch_size)):
            assert s % p == 0, f'Input dimension {i} ({s}) must be divisible by patch size ({p})'
        num_patches = math.prod(s // p for s, p in zip(input_shape, patch_size))
        patch_dim = channels * math.prod(patch_size)

        self.to_patch_embedding = nn.Sequential(
            PatchifyND(patch_size),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.pos_embedding = nn.Parameter(torch.randn(1, num_patches + 1, dim))
        self.cls_token = nn.Parameter(torch.randn(1, 1, dim))
        self.dropout = nn.Dropout(emb_dropout)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim, dropout)
        self.to_latent = nn.Identity()
        self.mlp_head = nn.Linear(dim, num_classes)

        self._nd_patch = tuple(patch_size)
        self._emb_dropout_p = float(emb_dropout)
        self._nd_engine = NdPatchEngine(self, self._nd_patch)

    # ---------------------------------------------------------------------------------------------- dispatch
    def fused_reason(self, x: torch.Tensor) -> Optional[str]:
        """None if forward(x) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        r = nd_fused_reason(self, x, self._nd_patch, max(self._emb_dropout_p, self.transformer.dropout_p))
        if r is None:
            N = self._nd_engine.tokens(x)[1]
            if N > self.pos_embedding.shape[1]:
                return f"{N} tokens exceed the positional table ({self.pos_embedding.shape[1]}; the reference raises)"
            r = self.transformer.engine().unsupported_reason(N)
        return r

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(x) is None:
            with on_device(x):
                return self.forward_fused(x)
        return self.forward_eager(x)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, x: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(x)
        b, n, _ = x.shape
        cls_tokens = self.cls_token.expand(b, -1, -1)
        x = torch.cat((cls_tokens, x), dim=1)
        x += self.pos_embedding[:, :(n + 1)]
        x = self.dropout(x)
        x = self.transformer(x)
        x = x[:, 1:].mean(dim=1) if self.pool == 'mean' else x[:, 0]
        x = self.to_latent(x)
        return self.mlp_head(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        x, B, N = nd_encode(self, self._nd_engine, img)
        eng = self.transformer.engine()
        if self.pool == 'mean':                        # mean over the patch tokens x[:, 1:], N - 1 rows per input
            pooled = eng.pool(x, B, N, mean=True, skip=1, n_pool=N - 1)
        else:
            pooled = eng.pool(x, B, N, mean=False)
        return classify(self, self.mlp_head, pooled)
