"""Drop-in `SepViT` for lucidrains/vit-pytorch's `vit_pytorch.sep_vit.SepViT` (depthwise separable self-attention:
attention inside windows that each carry a learned window token, then attention across the windows driven by those
tokens), with `ChanLayerNorm`, `OverlappingPatchEmbed`, `PEG`, `FeedForward`, `DSSA` and `Transformer` of the same
file, and a fused sm_90a forward.

Same constructor keywords and defaults, parameter names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed).  As in the reference (sep_vit.py:224, 274), SepViT's `window_size` and
`dim_head` reach no DSSA: every DSSA has its own defaults, window 7 and heads 32 wide.  The PyTorch graph mirrors the
reference without einops and raises where it raises (an AssertionError on a map that the window does not divide).

Fused forward, channels-last with an fp32 stream: token (b, y, x) of an h x w map is row (b*h + y)*w + x.  Per stage:
  * OverlappingPatchEmbed: stage 1 b200vit_conv_im2col_nchw (7 x 7, stride 4, padding 3; K = 147 zero-padded to 152),
    later stages b200vit_layernorm of the previous stage's stream (its Transformer's ChanLayerNorm) into bf16, then
    b200vit_conv_im2col_nhwc (3 x 3, stride 2, padding 1); then the convolution as one GEMM with bias, in fp32;
  * PEG: b200vit_peg into the stage's stream, and in fold mode b200vit_rowstats_cast into the engine's entry buffers;
  * Transformer: TransformerEngine.run_blocks with the map as `grid`: per layer the LN-folded QKV GEMM,
    b200vit_attention_window_token, and with more than one window b200vit_head_layernorm_gelu on the window tokens'
    outputs, their q | k GEMM and b200vit_window_mix; the out-projection residual; the GELU feed-forward (engine.py).
  * head: b200vit_mean_pool over the last map, b200vit_layernorm on the B pooled rows, the classifier GEMM.
"""
from __future__ import annotations

from functools import partial
from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import (PEG_KERNEL_SIZES, EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, WindowTokenBlock,
                     _bf16_rows, _f32, cached, common_reason, head_engine, head_ln_pool, on_device)

__all__ = ["ChanLayerNorm", "DSSA", "FeedForward", "OverlappingPatchEmbed", "PEG", "SepViT", "Transformer",
           "cast_tuple"]


def cast_tuple(val, length=1):
    return val if isinstance(val, tuple) else ((val,) * length)


class ChanLayerNorm(nn.Module):
    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.g = nn.Parameter(torch.ones(1, dim, 1, 1))
        self.b = nn.Parameter(torch.zeros(1, dim, 1, 1))

    def forward(self, x):
        var = torch.var(x, dim=1, unbiased=False, keepdim=True)
        mean = torch.mean(x, dim=1, keepdim=True)
        return (x - mean) / (var + self.eps).sqrt() * self.g + self.b


def _norm(ln: ChanLayerNorm) -> Norm:
    return Norm(ln.g.reshape(-1), ln.b.reshape(-1), ln.eps)


class OverlappingPatchEmbed(nn.Module):
    def __init__(self, dim_in, dim_out, stride=2):
        super().__init__()
        kernel_size = stride * 2 - 1
        padding = kernel_size // 2
        self.conv = nn.Conv2d(dim_in, dim_out, kernel_size, stride=stride, padding=padding)

    def forward(self, x):
        return self.conv(x)


class PEG(nn.Module):
    def __init__(self, dim, kernel_size=3):
        super().__init__()
        self.proj = nn.Conv2d(dim, dim, kernel_size=kernel_size, padding=kernel_size // 2, groups=dim, stride=1)

    def forward(self, x):
        return self.proj(x) + x


class FeedForward(nn.Module):
    def __init__(self, dim, mult=4, dropout=0.):
        super().__init__()
        inner_dim = int(dim * mult)
        self.net = nn.Sequential(
            ChanLayerNorm(dim),
            nn.Conv2d(dim, inner_dim, 1),
            nn.GELU(),
            nn.Dropout(dropout),
            nn.Conv2d(inner_dim, dim, 1),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        return self.net(x)


class _HeadsToChannels(nn.Module):
    """Rearrange('b h n c -> b (h c) n') (reference sep_vit.py:99), without einops."""

    def forward(self, x):
        b, h, n, c = x.shape
        return x.permute(0, 1, 3, 2).reshape(b, h * c, n)


class _ChannelsToHeads(nn.Module):
    """Rearrange('b (h c) n -> b h n c', h = heads) (reference sep_vit.py:101), without einops."""

    def __init__(self, heads):
        super().__init__()
        self.heads = heads

    def forward(self, x):
        b, hc, n = x.shape
        return x.reshape(b, self.heads, hc // self.heads, n).permute(0, 1, 3, 2)


class DSSA(nn.Module):
    def __init__(
        self,
        dim,
        heads=8,
        dim_head=32,
        dropout=0.,
        window_size=7
    ):
        super().__init__()
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.window_size = window_size
        inner_dim = dim_head * heads
        self.dim_head = dim_head
        self.dropout_p = float(dropout)

        self.norm = ChanLayerNorm(dim)

        self.attend = nn.Sequential(
            nn.Softmax(dim=-1),
            nn.Dropout(dropout)
        )

        self.to_qkv = nn.Conv1d(dim, inner_dim * 3, 1, bias=False)

        # window tokens

        self.window_tokens = nn.Parameter(torch.randn(dim))

        # prenorm and non-linearity for window tokens
        # then projection to queries and keys for window tokens

        self.window_tokens_to_qk = nn.Sequential(
            nn.LayerNorm(dim_head),
            nn.GELU(),
            _HeadsToChannels(),
            nn.Conv1d(inner_dim, inner_dim * 2, 1),
            _ChannelsToHeads(heads),
        )

        # window attention

        self.window_attend = nn.Sequential(
            nn.Softmax(dim=-1),
            nn.Dropout(dropout)
        )

        self.to_out = nn.Sequential(
            nn.Conv2d(inner_dim, dim, 1),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        batch, height, width, heads, wsz = x.shape[0], *x.shape[-2:], self.heads, self.window_size
        assert (height % wsz) == 0 and (width % wsz) == 0, \
            f'height {height} and width {width} must be divisible by window size {wsz}'
        X, Y = height // wsz, width // wsz
        num_windows = X * Y

        x = self.norm(x)
        c = x.shape[1]

        # 'b c (h w1) (w w2) -> (b h w) c (w1 w2)'
        x = x.reshape(batch, c, X, wsz, Y, wsz).permute(0, 2, 4, 1, 3, 5).reshape(batch * num_windows, c, wsz * wsz)

        w = self.window_tokens.reshape(1, c, 1).expand(x.shape[0], -1, -1)
        x = torch.cat((w, x), dim=-1)

        q, k, v = self.to_qkv(x).chunk(3, dim=1)

        # 'b (h d) n -> b h n d'
        q, k, v = (t.reshape(t.shape[0], heads, -1, t.shape[-1]).transpose(-1, -2) for t in (q, k, v))

        q = q * self.scale
        dots = torch.matmul(q, k.transpose(-1, -2))
        attn = self.attend(dots)
        out = torch.matmul(attn, v)

        window_tokens, windowed_fmaps = out[:, :, 0], out[:, :, 1:]

        def fold(t):
            """'(b x y) h (w1 w2) d -> b (h d) (x w1) (y w2)' of the windows' outputs t [b*x*y, h, w1*w2, d]."""
            d = t.shape[-1]
            t = t.reshape(batch, X, Y, heads, wsz, wsz, d).permute(0, 3, 6, 1, 4, 2, 5)
            return t.reshape(batch, heads * d, height, width)

        if num_windows == 1:
            return self.to_out(fold(windowed_fmaps))

        # '(b x y) h d -> b h (x y) d' and '(b x y) h n d -> b h (x y) n d'
        window_tokens = window_tokens.reshape(batch, num_windows, heads, -1).transpose(1, 2)
        windowed_fmaps = windowed_fmaps.reshape(batch, num_windows, heads, wsz * wsz, -1).transpose(1, 2)

        w_q, w_k = self.window_tokens_to_qk(window_tokens).chunk(2, dim=-1)
        w_q = w_q * self.scale
        w_dots = torch.matmul(w_q, w_k.transpose(-1, -2))
        w_attn = self.window_attend(w_dots)

        # 'b h i j, b h j w d -> b h i w d'
        b_, h_, n_, p_, d_ = windowed_fmaps.shape
        aggregated = torch.matmul(w_attn, windowed_fmaps.reshape(b_, h_, n_, p_ * d_)).reshape(b_, h_, n_, p_, d_)

        # 'b h (x y) (w1 w2) d -> b (h d) (x w1) (y w2)'
        return self.to_out(fold(aggregated.transpose(1, 2).reshape(batch * num_windows, heads, p_, d_)))


class Transformer(FusedEncoder, nn.Module):
    """depth x (DSSA, FeedForward) with residuals, then ChanLayerNorm (reference sep_vit.py:208-235).  A direct call
    on a (b, c, h, w) bf16 CUDA map runs fused through engine()."""

    def __init__(
        self,
        dim,
        depth,
        dim_head=32,
        heads=8,
        ff_mult=4,
        dropout=0.,
        norm_output=True
    ):
        super().__init__()
        self.layers = nn.ModuleList([])

        for ind in range(depth):
            self.layers.append(nn.ModuleList([
                DSSA(dim, heads=heads, dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mult=ff_mult, dropout=dropout),
            ]))

        self.norm = ChanLayerNorm(dim) if norm_output else nn.Identity()
        self._dropout_p = float(dropout)

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        layers = []
        for attn, ff in self.layers:
            f = ff.net
            I, D = attn.to_qkv.weight.shape[0] // 3, attn.to_qkv.weight.shape[1]
            ln, conv = attn.window_tokens_to_qk[0], attn.window_tokens_to_qk[3]
            layers.append(EncoderLayer(
                ln1=_norm(attn.norm), qkv_w=attn.to_qkv.weight.reshape(3 * I, D),
                out_w=attn.to_out[0].weight.reshape(D, I), out_b=attn.to_out[0].bias, ln2=_norm(f[0]),
                fc1_w=f[1].weight.reshape(-1, D), fc1_b=f[1].bias, fc2_w=f[4].weight.reshape(D, -1), fc2_b=f[4].bias,
                heads=attn.heads, dim_head=attn.dim_head, scale=attn.scale,
                attention=WindowTokenBlock(token=attn.window_tokens, ln=Norm.of(ln),
                                           wqk_w=conv.weight.reshape(2 * I, I), wqk_b=conv.bias,
                                           window=attn.window_size)))
        return layers, None if isinstance(self.norm, nn.Identity) else _norm(self.norm)

    def map_reason(self, h: int, w: int) -> Optional[str]:
        """Why an h x w map cannot run fused, or None: a map the windows do not divide (the reference raises), then
        the engine's rules."""
        for attn, _ in self.layers:
            p = attn.window_size
            if h % p or w % p:
                return f"the {h} x {w} map is not divisible by window_size={p} (the reference raises)"
        return self.engine().unsupported_reason(h * w, grid=(h, w))

    def fused_reason(self, x: torch.Tensor) -> Optional[str]:
        if x.dim() != 4:
            return "input is not a (b, c, h, w) map"
        r = common_reason(self, x, encoders=(self,), dropout_p=self._dropout_p, inside="transformer")
        if r is not None:
            return r
        if self.training:
            return "training mode (the fused path is inference only)"
        if x.shape[1] % 8:
            return f"dim={x.shape[1]} (the GEMMs need multiples of 8)"
        return self.map_reason(x.shape[2], x.shape[3])

    def forward(self, x):
        if self.fused_reason(x) is None:
            b, c, h, w = x.shape
            out = self.engine().forward_tokens(x.permute(0, 2, 3, 1).reshape(b, h * w, c), grid=(h, w))
            return out.view(b, h, w, c).permute(0, 3, 1, 2).contiguous()
        return self.forward_eager(x)

    def forward_eager(self, x):
        for attn, ff in self.layers:
            x = attn(x) + x
            x = ff(x) + x

        return self.norm(x)


class _MeanHW(nn.Module):
    """Reduce('b d h w -> b d', 'mean') (reference sep_vit.py:278), without einops."""

    def forward(self, x):
        if x.dim() != 4:
            raise RuntimeError(f"Reduce('b d h w -> b d'): expected 4 dims, got {x.dim()}")
        return x.mean(dim=(2, 3))


def conv_weights(conv: nn.Conv2d, channels_last: bool) -> Tuple[torch.Tensor, torch.Tensor]:
    """(bf16 [out, K] GEMM weight, fp32 bias) of a Conv2d: columns (cin, ky, kx) for the NCHW image
    (b200vit_conv_im2col_nchw), (ky, kx, cin) for a channels-last map (b200vit_conv_im2col_nhwc), K zero-padded to a
    multiple of 8."""
    w = conv.weight.detach()
    if channels_last:
        w = w.permute(0, 2, 3, 1)
    w = w.reshape(w.shape[0], -1)
    return _bf16_rows(w.to(torch.bfloat16), (w.shape[1] + 7) // 8 * 8), _f32(conv.bias)


def peg_weights(peg: PEG) -> Tuple[torch.Tensor, torch.Tensor]:
    """(w fp32 [k*k, C] tap major, bias fp32 [C]) of b200vit_peg."""
    conv = peg.proj
    C, kk = conv.weight.shape[0], conv.kernel_size[0] ** 2
    return conv.weight.detach().float().reshape(C, kk).t().contiguous(), _f32(conv.bias)


class SepViT(FusedWeightsMixin, nn.Module):
    def __init__(
        self,
        *,
        num_classes,
        dim,
        depth,
        heads,
        window_size=7,
        dim_head=32,
        ff_mult=4,
        channels=3,
        dropout=0.
    ):
        super().__init__()
        assert isinstance(depth, tuple), \
            'depth needs to be tuple if integers indicating number of transformer blocks at that stage'

        num_stages = len(depth)

        dims = tuple(map(lambda i: (2 ** i) * dim, range(num_stages)))
        dims = (channels, *dims)
        dim_pairs = tuple(zip(dims[:-1], dims[1:]))

        strides = (4, *((2,) * (num_stages - 1)))

        hyperparams_per_stage = [heads, window_size]
        hyperparams_per_stage = list(map(partial(cast_tuple, length=num_stages), hyperparams_per_stage))
        assert all(tuple(map(lambda arr: len(arr) == num_stages, hyperparams_per_stage)))

        self.layers = nn.ModuleList([])

        for ind, ((layer_dim_in, layer_dim), layer_depth, layer_stride, layer_heads, layer_window_size) in enumerate(
                zip(dim_pairs, depth, strides, *hyperparams_per_stage)):
            is_last = ind == (num_stages - 1)

            self.layers.append(nn.ModuleList([
                OverlappingPatchEmbed(layer_dim_in, layer_dim, stride=layer_stride),
                PEG(layer_dim),
                Transformer(dim=layer_dim, depth=layer_depth, heads=layer_heads, ff_mult=ff_mult, dropout=dropout,
                            norm_output=not is_last),
            ]))

        self.mlp_head = nn.Sequential(
            _MeanHW(),
            nn.LayerNorm(dims[-1]),
            nn.Linear(dims[-1], num_classes)
        )
        self._dropout_p = float(dropout)

    # ---------------------------------------------------------------------------------------------- dispatch
    def stage_maps(self, H: int, W: int) -> List[Tuple[int, int]]:
        """The (h, w) map of every stage for an H x W image."""
        maps = []
        for ope, _, _ in self.layers:
            c = ope.conv
            H = _lib.conv_out_size(H, c.kernel_size[0], c.stride[0], c.padding[0])
            W = _lib.conv_out_size(W, c.kernel_size[1], c.stride[1], c.padding[1])
            maps.append((H, W))
        return maps

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        if img.shape[1] != self.layers[0][0].conv.in_channels:
            return f"input has {img.shape[1]} channels, the model {self.layers[0][0].conv.in_channels}"
        r = common_reason(self, img, encoders=[t for _, _, t in self.layers], dropout_p=self._dropout_p)
        if r is not None:
            return r
        if self.training:
            return "training mode (the fused path is inference only)"
        for i, ((ope, peg, tr), (h, w)) in enumerate(zip(self.layers, self.stage_maps(img.shape[2], img.shape[3]))):
            D = ope.conv.out_channels
            if D % 8:
                return f"stage {i + 1}: width {D} (the GEMMs need multiples of 8)"
            if peg.proj.kernel_size[0] not in PEG_KERNEL_SIZES:
                return (f"PEG kernel_size={peg.proj.kernel_size[0]} (the positional-encoding kernel is built for 1, 3, "
                        f"5 and 7)")
            r = tr.map_reason(h, w)
            if r is not None:
                return f"stage {i + 1}: {r}"
        return None

    def forward(self, x):
        if self.fused_reason(x) is None:
            with on_device(x):
                return self.forward_fused(x)
        return self.forward_eager(x)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, x):
        for ope, peg, transformer in self.layers:
            x = ope(x)
            x = peg(x)
            x = transformer(x)

        return self.mlp_head(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def prepared(self) -> dict:
        """'ope<i>.w' / '.b' (the patch convolutions as GEMMs) and 'peg<i>.w' / '.b' of every stage."""
        params = [p for ope, peg, _ in self.layers for p in (*ope.parameters(), *peg.parameters())]
        return cached(self, "_prepared", params, self._build)

    def _build(self) -> dict:
        t = {}
        for i, (ope, peg, _) in enumerate(self.layers):
            t[f"ope{i}.w"], t[f"ope{i}.b"] = conv_weights(ope.conv, channels_last=i > 0)
            t[f"peg{i}.w"], t[f"peg{i}.b"] = peg_weights(peg)
        return t

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev = img.device
        bf, f32 = dict(device=dev, dtype=torch.bfloat16), dict(device=dev, dtype=torch.float32)
        t = self.prepared()
        B = img.shape[0]
        x, h, w, prev = None, 0, 0, None
        for i, ((ope, peg, tr), (oh, ow)) in enumerate(zip(self.layers, self.stage_maps(img.shape[2], img.shape[3]))):
            c = ope.conv
            k, s, pad = c.kernel_size[0], c.stride[0], c.padding[0]
            M, D = B * oh * ow, c.out_channels
            # OverlappingPatchEmbed: im2col + GEMM; after stage 1 on the previous stage's ChanLayerNorm output
            col = torch.empty(M, t[f"ope{i}.w"].shape[1], **bf)
            if i == 0:
                _lib.conv_im2col_nchw(img.contiguous(), col, k, s, pad)
            else:
                xn = torch.empty(x.shape, **bf)
                prev.engine().final_norm(x, out_bf16=xn)
                _lib.conv_im2col_nhwc(xn, col, B, h, w, k, s, pad)
            y = torch.empty(M, D, **f32)
            _lib.gemm(col, t[f"ope{i}.w"], out_f32=y, bias=t[f"ope{i}.b"])
            h, w = oh, ow
            # PEG out of place (every token reads its neighbours), then the engine's entry buffers
            x = torch.empty_like(y)
            _lib.peg(y, t[f"peg{i}.w"], t[f"peg{i}.b"], x, B, h, w, peg.proj.kernel_size[0])
            eng = tr.engine()
            xb, stats = eng.entry_buffers(M, dev)
            if xb is not None:
                _lib.rowstats_cast(x, xb, stats)
            eng.run_blocks(x, B, h * w, primed=xb is not None, grid=(h, w))
            prev = tr
        # head: mean over the last map, LayerNorm of the B pooled rows, the classifier
        pooled = head_ln_pool(self, self.mlp_head[1], x, B, h * w, mean=True)
        return head_engine(self, self.mlp_head[2]).run(pooled)
