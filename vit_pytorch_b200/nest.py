"""Drop-in `NesT` for lucidrains/vit-pytorch's `vit_pytorch.nest.NesT` (hierarchical attention inside local blocks of
the map, aggregated by a convolution and a max-pool between hierarchies), with `LayerNorm`, `FeedForward`,
`Attention`, `Aggregate`, `Transformer` and `cast_tuple` of the same file, and a fused sm_90a forward.

Same constructor keywords and defaults, parameter names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed).  As in the reference, `dim_head` is accepted and ignored: every head is
dim // heads wide.  The PyTorch graph mirrors the reference without einops and raises where it raises: on an image the
patch size does not divide, on a map a level's block size does not divide, and on blocks of more tokens than the
position embedding has (`seq_len`).

Fused forward.  Inside a level the fp32 residual stream is block-major, the reference's own token order: with the
level's H x W map cut into nb x nb blocks of sh x sw tokens, token (b, y, x) is row
    ((b*nb + y/sh)*nb + x/sw)*(sh*sw) + (y % sh)*sw + (x % sw),
so every level's Transformer is a plain encoder over B*nb*nb sequences of sh*sw tokens.  The layout matters only at
the level boundaries, which gather anyway:
  * patch embedding: b200vit_patchify_ln (the features are already in (p1 p2 c) order), the 1 x 1 convolution as one
    GEMM into fp32, then b200vit_nest_level_entry with pool (1, 1, 0): the LayerNorm, + pos_emb, into block-major order
    (in fold mode also the engine's bf16 copy and row statistics);
  * every level: TransformerEngine.run_blocks over the blocks (the one-call C layer loop);
  * Aggregate, between levels: b200vit_nest_im2col (block-major stream -> 3 x 3 im2col columns in map order), the
    convolution as one GEMM with bias into fp32, then b200vit_nest_level_entry with pool (3, 2, 1): LayerNorm, max-pool
    and the next level's pos_emb, into the next level's block-major order;
  * head: the last level has one block (map order); b200vit_layernorm per token (the head's LayerNorm comes before
    the mean, nest.py:161-165), b200vit_mean_pool, the cast and the classifier GEMM.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import einsum, nn

from . import _lib
from .engine import (EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, _bf16_rows, _f32, cached, common_reason,
                     head_engine, on_device)

__all__ = ["Aggregate", "Attention", "FeedForward", "LayerNorm", "NesT", "Transformer", "cast_tuple"]


def cast_tuple(val, depth):
    return val if isinstance(val, tuple) else ((val,) * depth)


class LayerNorm(nn.Module):
    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.g = nn.Parameter(torch.ones(1, dim, 1, 1))
        self.b = nn.Parameter(torch.zeros(1, dim, 1, 1))

    def forward(self, x):
        var = torch.var(x, dim=1, unbiased=False, keepdim=True)
        mean = torch.mean(x, dim=1, keepdim=True)
        return (x - mean) / (var + self.eps).sqrt() * self.g + self.b


def _norm(ln: LayerNorm) -> Norm:
    return Norm(ln.g.reshape(-1), ln.b.reshape(-1), ln.eps)


class FeedForward(nn.Module):
    def __init__(self, dim, mlp_mult=4, dropout=0.):
        super().__init__()
        self.net = nn.Sequential(
            LayerNorm(dim),
            nn.Conv2d(dim, dim * mlp_mult, 1),
            nn.GELU(),
            nn.Dropout(dropout),
            nn.Conv2d(dim * mlp_mult, dim, 1),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        return self.net(x)


class Attention(nn.Module):
    def __init__(self, dim, heads=8, dropout=0.):
        super().__init__()
        dim_head = dim // heads
        inner_dim = dim_head * heads
        self.heads = heads
        self.scale = dim_head ** -0.5

        self.norm = LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)
        self.to_qkv = nn.Conv2d(dim, inner_dim * 3, 1, bias=False)

        self.to_out = nn.Sequential(
            nn.Conv2d(inner_dim, dim, 1),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        b, c, h, w, heads = *x.shape, self.heads

        x = self.norm(x)

        qkv = self.to_qkv(x).chunk(3, dim=1)
        # 'b (h d) x y -> b h (x y) d'
        q, k, v = (t.reshape(b, heads, -1, h * w).transpose(-1, -2) for t in qkv)

        dots = einsum('b h i d, b h j d -> b h i j', q, k) * self.scale

        attn = self.attend(dots)
        attn = self.dropout(attn)

        out = einsum('b h i j, b h j d -> b h i d', attn, v)
        # 'b h (x y) d -> b (h d) x y'
        out = out.transpose(-1, -2).reshape(b, -1, h, w)
        return self.to_out(out)


def Aggregate(dim, dim_out):
    return nn.Sequential(
        nn.Conv2d(dim, dim_out, 3, padding=1),
        LayerNorm(dim_out),
        nn.MaxPool2d(3, stride=2, padding=1)
    )


class Transformer(FusedEncoder, nn.Module):
    """pos_emb, then depth x (Attention, FeedForward) with residuals (reference nest.py:84-104).  NesT's fused forward
    runs the layers through engine(); a direct call keeps the PyTorch graph."""

    def __init__(self, dim, seq_len, depth, heads, mlp_mult, dropout=0.):
        super().__init__()
        self.layers = nn.ModuleList([])
        self.pos_emb = nn.Parameter(torch.randn(seq_len))

        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dropout=dropout),
                FeedForward(dim, mlp_mult, dropout=dropout)
            ]))

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        layers = []
        for attn, ff in self.layers:
            f = ff.net
            I, D = attn.to_qkv.weight.shape[0] // 3, attn.to_qkv.weight.shape[1]
            layers.append(EncoderLayer(
                ln1=_norm(attn.norm), qkv_w=attn.to_qkv.weight.reshape(3 * I, D),
                out_w=attn.to_out[0].weight.reshape(D, I), out_b=attn.to_out[0].bias, ln2=_norm(f[0]),
                fc1_w=f[1].weight.reshape(-1, D), fc1_b=f[1].bias, fc2_w=f[4].weight.reshape(D, -1), fc2_b=f[4].bias,
                heads=attn.heads, dim_head=I // attn.heads, scale=attn.scale))
        return layers, None

    def forward(self, x):
        *_, h, w = x.shape

        pos_emb = self.pos_emb[:(h * w)]
        if pos_emb.numel() != h * w:
            # what einops raises for '(h w) -> () () h w' on a prefix shorter than the block
            raise RuntimeError(f"Rearrange: a block of {h} x {w} tokens needs {h * w} positions, pos_emb has "
                               f"{self.pos_emb.numel()} (nest.py:97-98)")
        x = x + pos_emb.reshape(1, 1, h, w)

        for attn, ff in self.layers:
            x = attn(x) + x
            x = ff(x) + x
        return x


class _ToPatches(nn.Module):
    """Rearrange('b c (h p1) (w p2) -> b (p1 p2 c) h w') (reference nest.py:138), without einops."""

    def __init__(self, p):
        super().__init__()
        self.p = p

    def forward(self, x):
        b, c, H, W = x.shape
        p = self.p
        if H % p or W % p:
            raise RuntimeError(f"Rearrange: the {H} x {W} image does not split into {p} x {p} patches (nest.py:138)")
        x = x.reshape(b, c, H // p, p, W // p, p).permute(0, 3, 5, 1, 2, 4)
        return x.reshape(b, p * p * c, H // p, W // p)


class _MeanHW(nn.Module):
    """Reduce('b c h w -> b c', 'mean') (reference nest.py:163), without einops."""

    def forward(self, x):
        if x.dim() != 4:
            raise RuntimeError(f"Reduce('b c h w -> b c'): expected 4 dims, got {x.dim()}")
        return x.mean(dim=(2, 3))


def to_blocks(x: torch.Tensor, n: int) -> torch.Tensor:
    """'b c (b1 h) (b2 w) -> (b b1 b2) c h w' with b1 = b2 = n (reference nest.py:173)."""
    b, c, H, W = x.shape
    if H % n or W % n:
        raise RuntimeError(f"Rearrange: the {H} x {W} map does not split into {n} x {n} blocks (nest.py:173)")
    x = x.reshape(b, c, n, H // n, n, W // n).permute(0, 2, 4, 1, 3, 5)
    return x.reshape(b * n * n, c, H // n, W // n)


def from_blocks(x: torch.Tensor, n: int) -> torch.Tensor:
    """'(b b1 b2) c h w -> b c (b1 h) (b2 w)' with b1 = b2 = n (reference nest.py:175)."""
    bnn, c, h, w = x.shape
    x = x.reshape(bnn // (n * n), n, n, c, h, w).permute(0, 3, 1, 4, 2, 5)
    return x.reshape(bnn // (n * n), c, n * h, n * w)


class NesT(FusedWeightsMixin, nn.Module):
    def __init__(
        self,
        *,
        image_size,
        patch_size,
        num_classes,
        dim,
        heads,
        num_hierarchies,
        block_repeats,
        mlp_mult=4,
        channels=3,
        dim_head=64,
        dropout=0.
    ):
        super().__init__()
        assert (image_size % patch_size) == 0, 'Image dimensions must be divisible by the patch size.'
        num_patches = (image_size // patch_size) ** 2  # noqa: F841  (kept from the reference)
        patch_dim = channels * patch_size ** 2
        fmap_size = image_size // patch_size
        blocks = 2 ** (num_hierarchies - 1)

        seq_len = (fmap_size // blocks) ** 2   # sequence length is held constant across hierarchy
        hierarchies = list(reversed(range(num_hierarchies)))
        mults = [2 ** i for i in reversed(hierarchies)]

        layer_heads = list(map(lambda t: t * heads, mults))
        layer_dims = list(map(lambda t: t * dim, mults))
        last_dim = layer_dims[-1]

        layer_dims = [*layer_dims, layer_dims[-1]]
        dim_pairs = zip(layer_dims[:-1], layer_dims[1:])

        self.to_patch_embedding = nn.Sequential(
            _ToPatches(patch_size),
            LayerNorm(patch_dim),
            nn.Conv2d(patch_dim, layer_dims[0], 1),
            LayerNorm(layer_dims[0])
        )

        block_repeats = cast_tuple(block_repeats, num_hierarchies)

        self.layers = nn.ModuleList([])

        for level, heads, (dim_in, dim_out), block_repeat in zip(hierarchies, layer_heads, dim_pairs, block_repeats):
            is_last = level == 0
            depth = block_repeat

            self.layers.append(nn.ModuleList([
                Transformer(dim_in, seq_len, depth, heads, mlp_mult, dropout),
                Aggregate(dim_in, dim_out) if not is_last else nn.Identity()
            ]))

        self.mlp_head = nn.Sequential(
            LayerNorm(last_dim),
            _MeanHW(),
            nn.Linear(last_dim, num_classes)
        )
        self._dropout_p = float(dropout)

    # ---------------------------------------------------------------------------------------------- dispatch
    def level_maps(self, H: int, W: int) -> List[Tuple[int, int, int]]:
        """(h, w, nb) of every level for an H x W image: its map and its nb x nb blocks.  Each Aggregate's max-pool
        (3, stride 2, padding 1) takes a map to ceil(h / 2) x ceil(w / 2)."""
        p = self.to_patch_embedding[0].p
        h, w = H // p, W // p
        maps = []
        for i in range(len(self.layers)):
            maps.append((h, w, 2 ** (len(self.layers) - 1 - i)))
            h, w = _lib.conv_out_size(h, 3, 2, 1), _lib.conv_out_size(w, 3, 2, 1)
        return maps

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        pe = self.to_patch_embedding
        p, C = pe[0].p, pe[2].in_channels // pe[0].p ** 2
        if img.shape[1] != C:
            return f"input has {img.shape[1]} channels, the model {C}"
        r = common_reason(self, img, encoders=[tr for tr, _ in self.layers], dropout_p=self._dropout_p)
        if r is not None:
            return r
        if self.training:
            return "training mode (the fused path is inference only)"
        H, W = img.shape[2], img.shape[3]
        if H % p or W % p:
            return f"the {H} x {W} image is not divisible by patch_size={p} (the reference raises)"
        for i, ((tr, _), (h, w, nb)) in enumerate(zip(self.layers, self.level_maps(H, W))):
            if h % nb or w % nb:
                return f"level {i + 1}: the {h} x {w} map does not split into {nb} x {nb} blocks (the reference raises)"
            n = (h // nb) * (w // nb)
            if n > tr.pos_emb.numel():
                return (f"level {i + 1}: blocks of {n} tokens, more than seq_len={tr.pos_emb.numel()} "
                        f"(the reference raises)")
            r = tr.engine().unsupported_reason(n)
            if r is not None:
                return f"level {i + 1}: {r}"
        return None

    def forward(self, img):
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, img):
        x = self.to_patch_embedding(img)
        b, c, h, w = x.shape

        num_hierarchies = len(self.layers)

        for level, (transformer, aggregate) in zip(reversed(range(num_hierarchies)), self.layers):
            block_size = 2 ** level
            x = to_blocks(x, block_size)
            x = transformer(x)
            x = from_blocks(x, block_size)
            x = aggregate(x)

        return self.mlp_head(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def prepared(self) -> dict:
        """'pe.g' / 'pe.b' (the patch LayerNorm), 'pe.w' / 'pe.bias' (the 1 x 1 convolution as a GEMM, K zero-padded to
        a multiple of 8), 'pe.g2' / 'pe.b2' (its LayerNorm); per level 'pos<i>'; per Aggregate 'agg<i>.w' / '.bias'
        (the 3 x 3 convolution as a GEMM over b200vit_nest_im2col's columns (ky, kx, cin)) and 'agg<i>.g' / '.b';
        'head.g' / 'head.b'."""
        params = [*self.to_patch_embedding.parameters(), *self.mlp_head[0].parameters()]
        for tr, agg in self.layers:
            params += [tr.pos_emb, *agg.parameters()]
        return cached(self, "_prepared", params, self._build)

    def _build(self) -> dict:
        _, ln1, conv, ln2 = self.to_patch_embedding
        K = conv.in_channels
        t = {"pe.g": _f32(ln1.g.reshape(-1)), "pe.b": _f32(ln1.b.reshape(-1)),
             "pe.w": _bf16_rows(conv.weight.reshape(conv.out_channels, K), (K + 7) // 8 * 8),
             "pe.bias": _f32(conv.bias),
             "pe.g2": _f32(ln2.g.reshape(-1)), "pe.b2": _f32(ln2.b.reshape(-1)),
             "head.g": _f32(self.mlp_head[0].g.reshape(-1)), "head.b": _f32(self.mlp_head[0].b.reshape(-1))}
        for i, (tr, agg) in enumerate(self.layers):
            t[f"pos{i}"] = _f32(tr.pos_emb)
            if isinstance(agg, nn.Sequential):
                c, ln = agg[0], agg[1]
                t[f"agg{i}.w"] = _bf16_rows(c.weight.detach().permute(0, 2, 3, 1).reshape(c.out_channels, -1))
                t[f"agg{i}.bias"], t[f"agg{i}.g"], t[f"agg{i}.b"] = _f32(c.bias), _f32(ln.g.reshape(-1)), \
                    _f32(ln.b.reshape(-1))
        return t

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev = img.device
        bf, f32 = dict(device=dev, dtype=torch.bfloat16), dict(device=dev, dtype=torch.float32)
        t = self.prepared()
        pe = self.to_patch_embedding
        B, p = img.shape[0], pe[0].p
        maps = self.level_maps(img.shape[2], img.shape[3])
        # patch embedding: patches + LayerNorm -> 1 x 1 convolution -> the first level's entry (LayerNorm, + pos_emb)
        h, w, _ = maps[0]
        a = torch.empty(B * h * w, t["pe.w"].shape[1], **bf)
        _lib.patchify_ln(img.contiguous(), t["pe.g"], t["pe.b"], a, p, p, eps=pe[1].eps)
        y = torch.empty(B * h * w, pe[2].out_channels, **f32)
        _lib.gemm(a, t["pe.w"], out_f32=y, bias=t["pe.bias"])
        norm, pool = (t["pe.g2"], t["pe.b2"], pe[3].eps), (1, 1, 0)
        ph, pw = h, w                              # the map y holds
        for i, ((tr, agg), (h, w, nb)) in enumerate(zip(self.layers, maps)):
            eng = tr.engine()
            M, D = B * h * w, y.shape[1]
            xb, stats = eng.entry_buffers(M, dev)
            x = torch.empty(M, D, **f32)
            _lib.nest_level_entry(y, norm[0], norm[1], t[f"pos{i}"], x, B, ph, pw, *pool, nb, eps=norm[2], xb=xb,
                                  stats=stats)
            eng.run_blocks(x, B * nb * nb, (h // nb) * (w // nb), primed=xb is not None)
            if i + 1 < len(self.layers):
                # Aggregate: 3 x 3 convolution (im2col from the block-major stream, GEMM), then the next level's entry
                col = torch.empty(M, 9 * D, **bf)
                _lib.nest_im2col(x, col, B, h, w, nb)
                y = torch.empty(M, agg[0].out_channels, **f32)
                _lib.gemm(col, t[f"agg{i}.w"], out_f32=y, bias=t[f"agg{i}.bias"])
                norm, pool = (t[f"agg{i}.g"], t[f"agg{i}.b"], agg[1].eps), (3, 2, 1)
                ph, pw = h, w
        # head: the last level is one block, in map order; LayerNorm per token, then the mean, then the classifier
        D = x.shape[1]
        xf = torch.empty_like(x)
        _lib.layernorm(x, t["head.g"], t["head.b"], out_f32=xf, eps=self.mlp_head[0].eps)
        pm = torch.empty(B, D, **f32)
        _lib.mean_pool(xf, pm, B, h * w, D)
        pooled = torch.empty(B, D, **bf)
        _lib.cast_f32_bf16(pm, pooled)
        return head_engine(self, self.mlp_head[2]).run(pooled)
