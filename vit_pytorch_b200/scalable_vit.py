"""Drop-in `ScalableViT` for lucidrains/vit-pytorch's `vit_pytorch.scalable_vit.ScalableViT` (scalable self-attention
over sub-sampled keys and interactive windowed self-attention), with `ChanLayerNorm`, `Downsample`, `PEG`,
`FeedForward`, `ScalableSelfAttention`, `InteractiveWindowedSelfAttention`, `Transformer` and the helpers of the same
file, and a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed).  The PyTorch graph below mirrors the reference module for module, without einops,
and raises where it raises.  Note the reference's layer loop (scalable_vit.py:228-236): it unpacks each layer's
modules [SSA, FeedForward, PEG, FeedForward, IWSA] as (ssa, ff1, peg, iwsa, ff2), so a layer runs SSA, FeedForward,
PEG, FeedForward, then the windowed attention, each with its residual; both graphs here run that order.

Fused forward, on the channels-last map x fp32 [B*h*w, C] (token (b, y, x) at row (b*h + y)*w + x):
  * to_patches: b200vit_conv_im2col_nchw (7 x 7, stride 4, padding 3) and the GEMM with bias into the stream;
  * per stage, through TransformerEngine.run_blocks with the stage's grid, two EncoderLayers per reference layer:
    (SSA, FeedForward) with a StridedKV record (b200vit_attention_kv_ex), then (FeedForward, IWSA) with `ff_first` and
    an InteractiveWindows record (the LIM convolution as im2col + GEMM, then b200vit_attention_iwsa).  The first
    reference layer's PEG runs between the two: run_blocks over layer 0, b200vit_peg into a second buffer (and in fold
    mode b200vit_rowstats_cast into the entry buffers), run_blocks over the rest;
  * between stages: the Transformer's ChanLayerNorm (b200vit_layernorm), b200vit_conv_im2col_nhwc (3 x 3, stride 2,
    padding 1) and the Downsample GEMM with bias into the next stage's stream;
  * head: b200vit_mean_pool, the LayerNorm of the B pooled rows, the classifier GEMM.
A dim_key that is a multiple of 8 and at most 64 runs at the next multiple of 16 (40 as 48): the q and k projection
weights get zero rows per head, which add exactly 0 to every score; the scale stays dim_key ** -0.5.
"""
from __future__ import annotations

from functools import partial
from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import (KV_EX_KEY_WIDTHS, KV_EX_VALUE_WIDTHS, PEG_KERNEL_SIZES, EncoderLayer, FusedEncoder,
                     FusedWeightsMixin, InteractiveWindows, Norm, StridedKV, cached, common_reason,
                     depthwise_peg_weights, head_engine, head_ln_pool, on_device)
from .sep_vit import _MeanHW, conv_weights

__all__ = ["ChanLayerNorm", "Downsample", "FeedForward", "InteractiveWindowedSelfAttention", "PEG",
           "ScalableSelfAttention", "ScalableViT", "Transformer", "cast_tuple", "default", "exists", "pair"]


def exists(val):
    return val is not None


def default(val, d):
    return val if exists(val) else d


def pair(t):
    return t if isinstance(t, tuple) else (t, t)


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


class Downsample(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.conv = nn.Conv2d(dim_in, dim_out, 3, stride=2, padding=1)

    def forward(self, x):
        return self.conv(x)


class PEG(nn.Module):
    def __init__(self, dim, kernel_size=3):
        super().__init__()
        self.proj = nn.Conv2d(dim, dim, kernel_size=kernel_size, padding=kernel_size // 2, groups=dim, stride=1)

    def forward(self, x):
        return self.proj(x) + x


class FeedForward(nn.Module):
    def __init__(self, dim, expansion_factor=4, dropout=0.):
        super().__init__()
        inner_dim = dim * expansion_factor
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


def _split_heads(t: torch.Tensor, heads: int) -> torch.Tensor:
    """'b (h d) ... -> b h (...) d'"""
    b = t.shape[0]
    return t.reshape(b, heads, t.shape[1] // heads, -1).transpose(-1, -2)


class ScalableSelfAttention(nn.Module):
    def __init__(self, dim, heads=8, dim_key=32, dim_value=32, dropout=0., reduction_factor=1):
        super().__init__()
        self.heads = heads
        self.scale = dim_key ** -0.5
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)

        self.norm = ChanLayerNorm(dim)
        self.to_q = nn.Conv2d(dim, dim_key * heads, 1, bias=False)
        self.to_k = nn.Conv2d(dim, dim_key * heads, reduction_factor, stride=reduction_factor, bias=False)
        self.to_v = nn.Conv2d(dim, dim_value * heads, reduction_factor, stride=reduction_factor, bias=False)

        self.to_out = nn.Sequential(
            nn.Conv2d(dim_value * heads, dim, 1),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        height, width, heads = *x.shape[-2:], self.heads
        x = self.norm(x)
        q, k, v = self.to_q(x), self.to_k(x), self.to_v(x)
        q, k, v = (_split_heads(t, heads) for t in (q, k, v))
        dots = torch.matmul(q, k.transpose(-1, -2)) * self.scale
        attn = self.dropout(self.attend(dots))
        out = torch.matmul(attn, v)
        # 'b h (x y) d -> b (h d) x y'
        b = out.shape[0]
        out = out.transpose(-1, -2).reshape(b, -1, height, width)
        return self.to_out(out)


class InteractiveWindowedSelfAttention(nn.Module):
    def __init__(self, dim, window_size, heads=8, dim_key=32, dim_value=32, dropout=0.):
        super().__init__()
        self.heads = heads
        self.scale = dim_key ** -0.5
        self.window_size = window_size
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)

        self.norm = ChanLayerNorm(dim)
        self.local_interactive_module = nn.Conv2d(dim_value * heads, dim_value * heads, 3, padding=1)

        self.to_q = nn.Conv2d(dim, dim_key * heads, 1, bias=False)
        self.to_k = nn.Conv2d(dim, dim_key * heads, 1, bias=False)
        self.to_v = nn.Conv2d(dim, dim_value * heads, 1, bias=False)

        self.to_out = nn.Sequential(
            nn.Conv2d(dim_value * heads, dim, 1),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        height, width, heads, wsz = *x.shape[-2:], self.heads, self.window_size
        x = self.norm(x)
        wsz_h, wsz_w = default(wsz, height), default(wsz, width)
        assert (height % wsz_h) == 0 and (width % wsz_w) == 0, \
            f'height ({height}) or width ({width}) of feature map is not divisible by the window size ({wsz_h}, {wsz_w})'

        q, k, v = self.to_q(x), self.to_k(x), self.to_v(x)
        local_out = self.local_interactive_module(v)

        b, X, Y = x.shape[0], height // wsz_h, width // wsz_w

        def windows(t):     # 'b (h d) (x w1) (y w2) -> (b x y) h (w1 w2) d'
            d = t.shape[1] // heads
            return (t.reshape(b, heads, d, X, wsz_h, Y, wsz_w).permute(0, 3, 5, 1, 4, 6, 2)
                    .reshape(b * X * Y, heads, wsz_h * wsz_w, d))

        q, k, v = map(windows, (q, k, v))
        dots = torch.matmul(q, k.transpose(-1, -2)) * self.scale
        attn = self.dropout(self.attend(dots))
        out = torch.matmul(attn, v)
        # '(b x y) h (w1 w2) d -> b (h d) (x w1) (y w2)'
        d = out.shape[-1]
        out = out.reshape(b, X, Y, heads, wsz_h, wsz_w, d).permute(0, 3, 6, 1, 4, 2, 5).reshape(b, heads * d, height,
                                                                                              width)
        out = out + local_out
        return self.to_out(out)


def padded_key_width(dk: int) -> int:
    """The head width the kernels run a dim_key at: the next multiple of 16 (dk itself when it is one)."""
    return (dk + 15) // 16 * 16


def _pad_heads(w: torch.Tensor, heads: int, dp: int) -> torch.Tensor:
    """A projection weight [heads * d, ...] with dp - d zero rows appended to every head: [heads * dp, ...]."""
    w = w.detach()
    d = w.shape[0] // heads
    if d == dp:
        return w
    w = w.reshape(heads, d, *w.shape[1:])
    return torch.cat((w, w.new_zeros(heads, dp - d, *w.shape[2:])), dim=1).reshape(heads * dp, *w.shape[2:])


class Transformer(FusedEncoder, nn.Module):
    """The reference's Transformer; called on a bf16 channels-first map on the GPU it runs fused (run_fused, then its
    ChanLayerNorm), else its PyTorch graph."""

    def __init__(self, dim, depth, heads=8, ff_expansion_factor=4, dropout=0., ssa_dim_key=32, ssa_dim_value=32,
                 ssa_reduction_factor=1, iwsa_dim_key=32, iwsa_dim_value=32, iwsa_window_size=None, norm_output=True):
        super().__init__()
        self.layers = nn.ModuleList([])
        for ind in range(depth):
            is_first = ind == 0

            self.layers.append(nn.ModuleList([
                ScalableSelfAttention(dim, heads=heads, dim_key=ssa_dim_key, dim_value=ssa_dim_value,
                                      reduction_factor=ssa_reduction_factor, dropout=dropout),
                FeedForward(dim, expansion_factor=ff_expansion_factor, dropout=dropout),
                PEG(dim) if is_first else None,
                FeedForward(dim, expansion_factor=ff_expansion_factor, dropout=dropout),
                InteractiveWindowedSelfAttention(dim, heads=heads, dim_key=iwsa_dim_key, dim_value=iwsa_dim_value,
                                                 window_size=iwsa_window_size, dropout=dropout)
            ]))

        self.norm = ChanLayerNorm(dim) if norm_output else nn.Identity()
        self._dropout_p = float(dropout)

    # ---------------------------------------------------------------------------------------------- dispatch
    def map_reason(self, h: int, w: int) -> Optional[str]:
        """Why an h x w map cannot run fused, or None: widths outside the built set, the reference's own failures
        (a window that does not divide the map, a map smaller than reduction_factor), then the engine's rules."""
        ssa, _, peg, _, iwsa = self.layers[0]
        D = ssa.to_q.in_channels
        if D % 8:
            return f"width {D} (the GEMMs need multiples of 8)"
        for name, a in (("ssa", ssa), ("iwsa", iwsa)):
            dk, dv = a.to_q.out_channels // a.heads, a.to_v.out_channels // a.heads
            if dk % 8 or dv % 8:
                return f"{name}_dim_key={dk}, {name}_dim_value={dv} (not multiples of 8)"
            if padded_key_width(dk) not in KV_EX_KEY_WIDTHS or dv not in KV_EX_VALUE_WIDTHS:
                return (f"{name}_dim_key={dk}, {name}_dim_value={dv} (the attention kernels are built for dim_key 8 "
                        f"to 64 and dim_value 32 or 64)")
        wh, ww = default(iwsa.window_size, h), default(iwsa.window_size, w)
        if h % wh or w % ww:
            return f"height ({h}) or width ({w}) of feature map is not divisible by the window size ({wh}, {ww})"
        r = ssa.to_k.kernel_size[0]
        if min(h, w) < r:
            return f"the {h} x {w} map is smaller than reduction_factor={r}"
        if peg.proj.kernel_size[0] not in PEG_KERNEL_SIZES:
            return f"PEG kernel_size={peg.proj.kernel_size[0]} (the positional-encoding kernel is built for 1-7)"
        return self.engine().unsupported_reason(h * w, grid=(h, w))

    def fused_reason(self, x: torch.Tensor) -> Optional[str]:
        if x.dim() != 4:
            return "input is not a (b, c, h, w) map"
        r = common_reason(self, x, encoders=(self,), dropout_p=self._dropout_p, inside="transformer")
        if r is not None:
            return r
        return self.map_reason(x.shape[2], x.shape[3])

    def forward(self, x):
        if self.fused_reason(x) is None:
            with on_device(x):
                b, c, h, w = x.shape
                xs = torch.empty(b * h * w, c, device=x.device, dtype=torch.float32)
                xs.copy_(x.permute(0, 2, 3, 1).reshape(b * h * w, c))
                xs = self.run_fused(xs, b, h, w)
                out = torch.empty(b * h * w, c, device=x.device, dtype=torch.bfloat16)
                if self.engine().norm is not None:
                    self.engine().final_norm(xs, out_bf16=out)
                else:
                    _lib.cast_f32_bf16(xs.view(-1), out.view(-1))
                return out.view(b, h, w, c).permute(0, 3, 1, 2).contiguous()
        return self.forward_eager(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def peg_weights(self) -> dict:
        conv = self.layers[0][2].proj
        return cached(self, "_peg", list(conv.parameters()), lambda: depthwise_peg_weights(conv))

    def run_fused(self, x: torch.Tensor, B: int, h: int, w: int) -> torch.Tensor:
        """The layers on the channels-last fp32 stream x [B*h*w, D] (no final norm): the first layer's SSA +
        FeedForward in place, its PEG into a new buffer (every token reads its neighbours) and in fold mode the entry
        buffers, then the rest in place there.  Returns that buffer."""
        eng, M = self.engine(), B * h * w
        eng.run_blocks(x, B, h * w, layers=[0], grid=(h, w))
        pw = self.peg_weights()
        y = torch.empty_like(x)
        _lib.peg(x, pw["w"], pw["b"], y, B, h, w, self.layers[0][2].proj.kernel_size[0])
        x = y
        xb, stats = eng.entry_buffers(M, x.device)
        if xb is not None:
            _lib.rowstats_cast(x, xb, stats)
        eng.run_blocks(x, B, h * w, primed=xb is not None, layers=range(1, 2 * len(self.layers)), grid=(h, w))
        return x

    def forward_eager(self, x):
        # the reference's names: its 4th module (a FeedForward) is bound to `iwsa`, its 5th (the IWSA) to `ff2`
        for ssa, ff1, peg, iwsa, ff2 in self.layers:
            x = ssa(x) + x
            x = ff1(x) + x

            if exists(peg):
                x = peg(x)

            x = iwsa(x) + x
            x = ff2(x) + x

        return self.norm(x)

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        """Two EncoderLayers per reference layer: (SSA, FeedForward) with StridedKV, then (FeedForward, IWSA) with
        ff_first and InteractiveWindows; q and k weights padded per head to padded_key_width."""
        layers = []
        for ssa, ff1, _, ff2, iwsa in self.layers:
            for a, f in ((ssa, ff1), (iwsa, ff2)):
                H, D = a.heads, a.to_q.weight.shape[1]
                dk, dv = a.to_q.weight.shape[0] // H, a.to_v.weight.shape[0] // H
                dp = padded_key_width(dk)
                q = _pad_heads(a.to_q.weight, H, dp).reshape(H * dp, D)
                n = f.net
                common = dict(
                    ln1=_norm(a.norm), out_w=a.to_out[0].weight.reshape(D, H * dv), out_b=a.to_out[0].bias,
                    ln2=_norm(n[0]), fc1_w=n[1].weight.reshape(-1, D), fc1_b=n[1].bias,
                    fc2_w=n[4].weight.reshape(D, -1), fc2_b=n[4].bias, heads=H, dim_head=dp, scale=a.scale)
                if a is ssa:
                    kv_w = torch.cat((_pad_heads(a.to_k.weight, H, dp), a.to_v.weight.detach()))
                    layers.append(EncoderLayer(qkv_w=q, attention=StridedKV(a.to_k.kernel_size[0], kv_w, dv),
                                               **common))
                else:
                    k = _pad_heads(a.to_k.weight, H, dp).reshape(H * dp, D)
                    qkv_w = torch.cat((q, k, a.to_v.weight.detach().reshape(H * dv, D)))
                    lim = a.local_interactive_module
                    layers.append(EncoderLayer(qkv_w=qkv_w, ff_first=True,
                                               attention=InteractiveWindows(a.window_size, lim.weight, lim.bias),
                                               **common))
        return layers, None if isinstance(self.norm, nn.Identity) else _norm(self.norm)


class ScalableViT(FusedWeightsMixin, nn.Module):
    def __init__(
        self,
        *,
        num_classes,
        dim,
        depth,
        heads,
        reduction_factor,
        window_size=None,
        iwsa_dim_key=32,
        iwsa_dim_value=32,
        ssa_dim_key=32,
        ssa_dim_value=32,
        ff_expansion_factor=4,
        channels=3,
        dropout=0.
    ):
        super().__init__()
        self.to_patches = nn.Conv2d(channels, dim, 7, stride=4, padding=3)

        assert isinstance(depth, tuple), \
            'depth needs to be tuple if integers indicating number of transformer blocks at that stage'

        num_stages = len(depth)
        dims = tuple(map(lambda i: (2 ** i) * dim, range(num_stages)))

        hyperparams_per_stage = [
            heads,
            ssa_dim_key,
            ssa_dim_value,
            reduction_factor,
            iwsa_dim_key,
            iwsa_dim_value,
            window_size,
        ]

        hyperparams_per_stage = list(map(partial(cast_tuple, length=num_stages), hyperparams_per_stage))
        assert all(tuple(map(lambda arr: len(arr) == num_stages, hyperparams_per_stage)))

        self.layers = nn.ModuleList([])

        for ind, (layer_dim, layer_depth, layer_heads, layer_ssa_dim_key, layer_ssa_dim_value,
                  layer_ssa_reduction_factor, layer_iwsa_dim_key, layer_iwsa_dim_value, layer_window_size) in \
                enumerate(zip(dims, depth, *hyperparams_per_stage)):
            is_last = ind == (num_stages - 1)

            self.layers.append(nn.ModuleList([
                Transformer(dim=layer_dim, depth=layer_depth, heads=layer_heads,
                            ff_expansion_factor=ff_expansion_factor, dropout=dropout, ssa_dim_key=layer_ssa_dim_key,
                            ssa_dim_value=layer_ssa_dim_value, ssa_reduction_factor=layer_ssa_reduction_factor,
                            iwsa_dim_key=layer_iwsa_dim_key, iwsa_dim_value=layer_iwsa_dim_value,
                            iwsa_window_size=layer_window_size, norm_output=not is_last),
                Downsample(layer_dim, layer_dim * 2) if not is_last else None
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
        H, W = _lib.conv_out_size(H, 7, 4, 3), _lib.conv_out_size(W, 7, 4, 3)
        maps = []
        for _ in self.layers:
            maps.append((H, W))
            H, W = _lib.conv_out_size(H, 3, 2, 1), _lib.conv_out_size(W, 3, 2, 1)
        return maps

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        if img.shape[1] != self.to_patches.in_channels:
            return f"input has {img.shape[1]} channels, the model {self.to_patches.in_channels}"
        r = common_reason(self, img, encoders=[t for t, _ in self.layers], dropout_p=self._dropout_p)
        if r is not None:
            return r
        for i, ((tr, _), (h, w)) in enumerate(zip(self.layers, self.stage_maps(img.shape[2], img.shape[3]))):
            r = tr.map_reason(h, w)
            if r is not None:
                return f"stage {i + 1}: {r}"
        return None

    def forward(self, img):
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, img):
        x = self.to_patches(img)

        for transformer, downsample in self.layers:
            x = transformer(x)

            if exists(downsample):
                x = downsample(x)

        return self.mlp_head(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def prepared(self) -> dict:
        """'patch.w' / '.b' (to_patches as a GEMM) and 'down<i>.w' / '.b' (the Downsample convolutions); every
        Transformer keeps its own PEG weights (Transformer.peg_weights)."""
        params = list(self.to_patches.parameters())
        for tr, down in self.layers:
            params += list(down.parameters()) if down is not None else []
        return cached(self, "_prepared", params, self._build)

    def _build(self) -> dict:
        t = {}
        t["patch.w"], t["patch.b"] = conv_weights(self.to_patches, channels_last=False)
        for i, (tr, down) in enumerate(self.layers):
            if down is not None:
                t[f"down{i}.w"], t[f"down{i}.b"] = conv_weights(down.conv, channels_last=True)
        return t

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev = img.device
        bf, f32 = dict(device=dev, dtype=torch.bfloat16), dict(device=dev, dtype=torch.float32)
        t = self.prepared()
        B = img.shape[0]
        maps = self.stage_maps(img.shape[2], img.shape[3])
        # to_patches: im2col of the NCHW image + GEMM into the fp32 stream
        h, w = maps[0]
        col = torch.empty(B * h * w, t["patch.w"].shape[1], **bf)
        _lib.conv_im2col_nchw(img.contiguous(), col, 7, 4, 3)
        x = torch.empty(B * h * w, self.to_patches.out_channels, **f32)
        _lib.gemm(col, t["patch.w"], out_f32=x, bias=t["patch.b"])
        for i, ((tr, down), (h, w)) in enumerate(zip(self.layers, maps)):
            eng = tr.engine()
            x = tr.run_fused(x, B, h, w)
            if down is not None:
                # the Transformer's ChanLayerNorm, then Downsample as im2col + GEMM into the next stage's stream
                xn = torch.empty(x.shape, **bf)
                eng.final_norm(x, out_bf16=xn)
                oh, ow = maps[i + 1]
                col = torch.empty(B * oh * ow, t[f"down{i}.w"].shape[1], **bf)
                _lib.conv_im2col_nhwc(xn, col, B, h, w, 3, 2, 1)
                x = torch.empty(B * oh * ow, down.conv.out_channels, **f32)
                _lib.gemm(col, t[f"down{i}.w"], out_f32=x, bias=t[f"down{i}.b"])
        # head: mean over the last map, LayerNorm of the B pooled rows, the classifier
        pooled = head_ln_pool(self, self.mlp_head[1], x, B, h * w, mean=True)
        return head_engine(self, self.mlp_head[2]).run(pooled)
