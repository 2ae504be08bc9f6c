"""Drop-in `PiT` for lucidrains/vit-pytorch's `vit_pytorch.pit.PiT` (pooling-based vision transformer), with `Pool`,
`DepthWiseConv2d`, `Transformer`, `Attention` and `FeedForward` of the same file, and a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed): `to_patch_embedding.2` the patch Linear (index 0 is the Unfold, 1 the transpose),
`pos_embedding` (1, num_patches + 1, dim), `cls_token` (1, 1, dim), `layers` one nn.Sequential alternating
`Transformer` and `Pool`, `mlp_head.{0,1}` (reference pit.py:117-182).  The PyTorch graph below mirrors the reference
module for module, including Pool's `int(sqrt(n))` grid rule, so hooks on any submodule keep working there.

Fused forward:
  * patch embedding: b200vit_unfold_patches (overlapping p x p patches at stride p // 2, bit copies), the patch GEMM,
    then b200vit_embed_tokens without a LayerNorm (cls row, positional rows :n + 1) writing the first stage's stream
    and, in fold mode, its bf16 copy and row statistics (pit.py:172-178);
  * per stage, the stage Transformer's TransformerEngine.run_blocks (plain pre-LN ViT layers without a final
    LayerNorm, pit.py:69-82) on that stage's fp32 residual stream [B*(1 + n), D];
  * between stages (Pool, pit.py:98-113): b200vit_pit_pool (depthwise 3 x 3 stride-2 convolution with channel
    multiplier 2 -> bf16 A operand, cls slots zeroed, and the bf16 cls rows), the 1 x 1 convolution as one GEMM over
    all B*(1 + n') rows writing the next stage's stream [B*(1 + n'), 2D], the cls_ff GEMM over the B cls rows
    (row stride (1 + n')*2D) overwriting its cls rows, and in fold mode b200vit_rowstats_cast into the next stage's
    entry buffers;
  * head: LayerNorm of the last stage's cls rows, then the head GEMM (pit.py:166-182).
Every stage's grid follows the reference: n tokens are read as int(sqrt(n)) x n // int(sqrt(n)), which is not the
geometric grid of a non-square image (a 4 x 16 unfold grid is pooled as 8 x 8).
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import (FusedWeightsMixin, _bf16_rows, _f32, cached, cls_row_index, common_reason, head_engine,
                     head_norm, head_width_reason, on_device)
from .vit import Attention, FeedForward, FusedTransformer

__all__ = ["Attention", "DepthWiseConv2d", "FeedForward", "PiT", "Pool", "Transformer", "cast_tuple",
           "conv_output_size", "pool_grid", "pool_weights"]


def cast_tuple(val, num):
    return val if isinstance(val, tuple) else (val,) * num


def conv_output_size(image_size, kernel_size, stride, padding=0):
    return int(((image_size - kernel_size + (2 * padding)) / stride) + 1)


def pool_grid(n: int) -> Optional[Tuple[int, int]]:
    """The (h, w) grid Pool reads n tokens as (pit.py:109: h = int(sqrt(n)), w inferred by einops), or None where
    einops raises (n not divisible by h)."""
    h = int(math.sqrt(n))
    if h == 0 or n % h:
        return None
    return h, n // h


class Transformer(FusedTransformer):
    """depth x (Attention, FeedForward) residual blocks without a final LayerNorm (reference pit.py:69-82).  Callable
    on (B, N, D) tokens; runs fused when eligible."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.) -> None:
        super().__init__()
        self.dropout_p = float(dropout)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))


class DepthWiseConv2d(nn.Module):
    """Depthwise k x k convolution (groups = dim_in) followed by a 1 x 1 convolution (reference pit.py:86-94)."""

    def __init__(self, dim_in, dim_out, kernel_size, padding, stride, bias=True) -> None:
        super().__init__()
        self.net = nn.Sequential(
            nn.Conv2d(dim_in, dim_out, kernel_size=kernel_size, padding=padding, groups=dim_in, stride=stride,
                      bias=bias),
            nn.Conv2d(dim_out, dim_out, kernel_size=1, bias=bias),
        )

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.net(x)


class Pool(nn.Module):
    """cls row through a Linear(dim, 2 dim); the token grid through DepthWiseConv2d(dim, 2 dim, 3, stride 2, pad 1)
    (reference pit.py:98-113)."""

    def __init__(self, dim: int) -> None:
        super().__init__()
        self.downsample = DepthWiseConv2d(dim, dim * 2, kernel_size=3, stride=2, padding=1)
        self.cls_ff = nn.Linear(dim, dim * 2)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        cls_token, tokens = x[:, :1], x[:, 1:]
        cls_token = self.cls_ff(cls_token)
        b, n, c = tokens.shape
        h = int(math.sqrt(n))
        if h == 0 or n % h:
            # what einops raises for 'b (h w) c -> b c h w' with an h that does not divide n
            raise RuntimeError(f"Pool: {n} tokens cannot be read as a grid of {h} rows (pit.py:109)")
        tokens = tokens.reshape(b, h, n // h, c).permute(0, 3, 1, 2)
        tokens = self.downsample(tokens)
        tokens = tokens.flatten(2).transpose(1, 2)
        return torch.cat((cls_token, tokens), dim=1)


def pool_weights(pool: Pool) -> dict:
    """The prepared weights of b200vit_pit_pool and the two GEMMs after it: 'w9' fp32 [9, 2D] (the depthwise weights
    tap major), 'b9' fp32 [2D], 'w1' bf16 [2D, 2D] and 'b1' fp32 (the 1 x 1 convolution), 'wc' bf16 [2D, D] and 'bc'
    fp32 (cls_ff)."""
    dw, pw = pool.downsample.net
    o = dw.weight.shape[0]
    zeros = torch.zeros(o, device=dw.weight.device, dtype=torch.float32)
    return {"w9": dw.weight.detach().float().reshape(o, 9).t().contiguous(),
            "b9": _f32(dw.bias) if dw.bias is not None else zeros,
            "w1": _bf16_rows(pw.weight.reshape(o, o)), "b1": _f32(pw.bias),
            "wc": _bf16_rows(pool.cls_ff.weight), "bc": _f32(pool.cls_ff.bias)}


class _Transpose(nn.Module):
    """Rearrange('b c n -> b n c') (reference pit.py:142), without einops."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x.transpose(1, 2)


class PiT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, dim_head=64, dropout=0.,
                 emb_dropout=0., channels=3) -> None:
        super().__init__()
        assert image_size % patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        assert isinstance(depth, tuple), \
            'depth must be a tuple of integers, specifying the number of blocks before each downsizing'
        heads = cast_tuple(heads, len(depth))
        patch_dim = channels * patch_size ** 2
        self.patch_size = patch_size

        self.to_patch_embedding = nn.Sequential(
            nn.Unfold(kernel_size=patch_size, stride=patch_size // 2),
            _Transpose(),
            nn.Linear(patch_dim, dim),
        )
        output_size = conv_output_size(image_size, patch_size, patch_size // 2)
        num_patches = output_size ** 2
        self.pos_embedding = nn.Parameter(torch.randn(1, num_patches + 1, dim))
        self.cls_token = nn.Parameter(torch.randn(1, 1, dim))
        self.dropout = nn.Dropout(emb_dropout)

        layers = []
        for ind, (layer_depth, layer_heads) in enumerate(zip(depth, heads)):
            not_last = ind < (len(depth) - 1)
            layers.append(Transformer(dim, layer_depth, layer_heads, dim_head, mlp_dim, dropout))
            if not_last:
                layers.append(Pool(dim))
                dim *= 2
        self.layers = nn.Sequential(*layers)
        self.mlp_head = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, num_classes))

        self._emb_dropout_p = float(emb_dropout)
        self._rows: dict = {}

    def stages(self) -> List[Transformer]:
        return [m for m in self.layers if isinstance(m, Transformer)]

    def pools(self) -> List[Pool]:
        return [m for m in self.layers if isinstance(m, Pool)]

    # ---------------------------------------------------------------------------------------------- dispatch
    def stage_grids(self, H: int, W: int) -> Optional[List[Tuple[int, int]]]:
        """The (h, w) token grid every Pool reads for an H x W image, in order; None where the reference's Pool
        raises (a token count the int(sqrt(n)) rule cannot reshape)."""
        p, s = self.patch_size, self.patch_size // 2
        n = ((H - p) // s + 1) * ((W - p) // s + 1)
        grids = []
        for _ in self.pools():
            g = pool_grid(n)
            if g is None:
                return None
            grids.append(g)
            n = ((g[0] + 1) // 2) * ((g[1] + 1) // 2)
        return grids

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        p = self.patch_size
        if img.shape[1] * p * p != self.to_patch_embedding[2].in_features:
            return "channel count differs from the constructor's (the reference's Linear raises)"
        if p < 2:
            return f"patch_size={p} (the reference's Unfold gets stride {p // 2})"
        stages = self.stages()
        r = common_reason(self, img, encoders=stages,
                          dropout_p=max([self._emb_dropout_p] + [t.dropout_p for t in stages]))
        if r is not None:
            return r
        H, W = img.shape[2], img.shape[3]
        if H < p or W < p:
            return f"image {H} x {W} smaller than one {p} x {p} patch"
        s = p // 2
        n = ((H - p) // s + 1) * ((W - p) // s + 1)
        if n + 1 > self.pos_embedding.shape[1]:
            return f"{n + 1} tokens exceed the positional table ({self.pos_embedding.shape[1]})"
        grids = self.stage_grids(H, W)
        if grids is None:
            return "a stage's token count cannot be read as a grid by the reference's int(sqrt(n)) rule"
        r = head_width_reason(stages[0].layers[0][0].dim_head)
        if r is not None:
            return r
        tokens = [n] + [((h + 1) // 2) * ((w + 1) // 2) for h, w in grids]
        for t, nt in zip(stages, tokens):
            r = t.engine().unsupported_reason(nt + 1)
            if r is not None:
                return r
        return None

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, img: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(img)
        b, n, _ = x.shape
        cls_tokens = self.cls_token.expand(b, -1, -1)
        x = torch.cat((cls_tokens, x), dim=1)
        x += self.pos_embedding[:, :n + 1]
        x = self.dropout(x)
        x = self.layers(x)
        return self.mlp_head(x[:, 0])

    # ---------------------------------------------------------------------------------------------- fused kernels
    def _patch_weights(self) -> dict:
        lin = self.to_patch_embedding[2]
        params = [lin.weight, lin.bias, self.pos_embedding, self.cls_token]
        kp = (lin.in_features + 63) // 64 * 64

        def build():
            D = lin.out_features
            return {"w": _bf16_rows(lin.weight, kp), "b": _f32(lin.bias), "kp": kp,
                    "pos": self.pos_embedding.detach().float().reshape(-1, D).contiguous(),
                    "cls": self.cls_token.detach().float().reshape(1, D).contiguous()}
        return cached(self, "_patch", params, build)

    def _pool_weights(self, i: int, pool: Pool) -> dict:
        return cached(self, f"_pool{i}", list(pool.parameters()), lambda: pool_weights(pool))

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev, bf = img.device, dict(device=img.device, dtype=torch.bfloat16)
        B, C, H, W = img.shape
        p = self.patch_size
        s = p // 2
        n = ((H - p) // s + 1) * ((W - p) // s + 1)
        stages, pools = self.stages(), self.pools()
        grids = self.stage_grids(H, W)
        # patch embedding: unfold -> patch GEMM -> cls row and positions
        t = self._patch_weights()
        D = t["w"].shape[0]
        a0 = torch.empty(B * n, t["kp"], **bf)
        _lib.unfold_patches(img.contiguous(), a0, p, s)
        y = torch.empty(B * n, D, device=dev, dtype=torch.float32)
        _lib.gemm(a0, t["w"], out_f32=y, bias=t["b"])
        N = n + 1
        eng = stages[0].engine()
        xb, stats = eng.entry_buffers(B * N, dev)
        x = torch.empty(B * N, D, device=dev, dtype=torch.float32)
        _lib.embed_tokens(y, None, None, t["cls"], t["pos"], x, B, n, 1, xb=xb, stats=stats)
        primed = xb is not None
        for i, stage in enumerate(stages):
            eng = stage.engine()
            eng.run_blocks(x, B, N, primed=primed)
            if i == len(pools):
                break
            # Pool: depthwise stride-2 convolution -> 1 x 1 convolution GEMM over every row -> cls_ff on the cls rows
            (h, w), pw = grids[i], self._pool_weights(i, pools[i])
            N2, D2 = ((h + 1) // 2) * ((w + 1) // 2) + 1, 2 * D
            a = torch.empty(B * N2, D2, **bf)
            cls = torch.empty(B, D, **bf)
            _lib.pit_pool(x, B, h, w, pw["w9"], pw["b9"], a, cls)
            x2 = torch.empty(B * N2, D2, device=dev, dtype=torch.float32)
            _lib.gemm(a, pw["w1"], out_f32=x2, bias=pw["b1"])
            _lib.gemm(cls, pw["wc"], out_f32=x2.view(B, N2, D2)[:, 0], bias=pw["bc"])
            x, N, D = x2, N2, D2
            xb, stats = stages[i + 1].engine().entry_buffers(B * N, dev)
            primed = xb is not None
            if primed:
                _lib.rowstats_cast(x, xb, stats)
        # head: LayerNorm of the cls rows, then the classifier GEMM
        ln = self.mlp_head[0]
        g, bt = head_norm(self, ln)
        pooled = torch.empty(B, D, **bf)
        _lib.layernorm(x, g, bt, out_bf16=pooled, row_index=cls_row_index(self._rows, B, N, dev), eps=ln.eps)
        return head_engine(self, self.mlp_head[1]).run(pooled)
