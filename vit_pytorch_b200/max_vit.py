"""Drop-in `MaxViT` for lucidrains/vit-pytorch's `vit_pytorch.max_vit.MaxViT` (multi-axis attention: block and grid
window attention with a relative-position bias, after an MBConv with squeeze-excitation), with `Residual`,
`FeedForward`, `SqueezeExcitation`, `MBConvResidual`, `Dropsample`, `MBConv`, `Attention` and the helpers `exists`,
`default` and `cast_tuple` of the same file, and a fused sm_90a forward.

Same constructor keywords, parameter and buffer names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed): `conv_stem.{0,1}`, `layers.i` one block per transformer block of every
stage, each `Sequential(MBConv, to block windows, Residual(Attention), Residual(FeedForward), back, to grid windows,
Residual(Attention), Residual(FeedForward), back)`, and `mlp_head` (mean, LayerNorm, Linear) (reference
max_vit.py:208-291).  `rel_pos_indices` stays a non-persistent buffer.  The PyTorch graph below mirrors the reference
module for module (the einops rearrangements as parameter-free modules at the same indices), so hooks on any
submodule keep working there, and it raises where the reference raises.

Fused forward, channels-last throughout: token (b, y, x) of an h x w map is row (b*h + y)*w + x of the fp32 stream
[B*h*w, D] and of its bf16 copy.  No token is ever moved into window order; only the attention kernel knows the
partition, as an address map.
  * conv_stem: b200vit_conv_im2col_nchw + GEMM (bias), then b200vit_conv_im2col_nhwc + GEMM (bias), bf16 out;
  * MBConv (max_vit.py:90-117): the 1 x 1 GEMM with its BatchNorm folded, bias and GELU, to bf16;
    b200vit_mbconv_dwconv (3 x 3 depthwise, stride 2 in a stage's first block, BatchNorm folded, GELU) with the
    per-image channel sums; squeeze-excitation as b200vit_se_pool, GEMM with SiLU, GEMM with sigmoid over the B pooled
    rows, b200vit_se_scale; the last 1 x 1 GEMM with its BatchNorm folded, added into the stream (MBConvResidual) or
    starting the stage's fresh fp32 stream;
  * block attention + FeedForward, then grid attention + FeedForward: two EncoderLayers through
    TransformerEngine.run_blocks with b200vit_attention_window_relpos (Windows.dilated False, then True);
  * head: b200vit_mean_pool, b200vit_layernorm (the reference normalises after pooling), the classifier GEMM.
BatchNorm runs on its running statistics: a BatchNorm2d in training mode sends the call to the PyTorch graph.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import einsum, nn

from . import _lib
from .engine import (EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, Windows, _bf16_rows, cached, common_reason,
                     head_engine, head_norm, on_device)
from .levit import _conv_weight, fold_bn
from .xcit import batchnorm_reason

__all__ = ["Attention", "Dropsample", "FeedForward", "MBConv", "MBConvResidual", "MaxViT", "Residual",
           "SqueezeExcitation", "cast_tuple", "default", "exists", "mbconv_weights"]


def exists(val):
    return val is not None


def default(val, d):
    return val if exists(val) else d


def cast_tuple(val, length=1):
    return val if isinstance(val, tuple) else ((val,) * length)


class Residual(nn.Module):
    def __init__(self, dim, fn):
        super().__init__()
        self.fn = fn

    def forward(self, x):
        return self.fn(x) + x


class FeedForward(nn.Module):
    def __init__(self, dim, mult=4, dropout=0.):
        super().__init__()
        inner_dim = int(dim * mult)
        self.net = nn.Sequential(
            nn.LayerNorm(dim),
            nn.Linear(dim, inner_dim),
            nn.GELU(),
            nn.Dropout(dropout),
            nn.Linear(inner_dim, dim),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        return self.net(x)


class _MeanHW(nn.Module):
    """Reduce('b c h w -> b c', 'mean') (reference max_vit.py:53, 280), without einops."""

    def forward(self, x):
        if x.dim() != 4:
            raise RuntimeError(f"Reduce('b c h w -> b c'): expected 4 dims, got {x.dim()}")
        return x.mean(dim=(2, 3))


class _Unsqueeze2(nn.Module):
    """Rearrange('b c -> b c 1 1') (reference max_vit.py:58), without einops."""

    def forward(self, x):
        return x[:, :, None, None]


class _ToWindows(nn.Module):
    """Rearrange('b d (x w1) (y w2) -> b x y w1 w2 d') (block) or 'b d (w1 x) (w2 y) -> b x y w1 w2 d' (grid), w1 =
    w2 = w (reference max_vit.py:264, 269), without einops; raises where einops does."""

    def __init__(self, w: int, grid: bool) -> None:
        super().__init__()
        self.w, self.grid = w, grid

    def forward(self, t):
        b, d, H, W = t.shape
        w = self.w
        if H % w or W % w:
            raise RuntimeError(f"Rearrange: a {H} x {W} map is not divisible into {w} x {w} windows")
        X, Y = H // w, W // w
        if self.grid:
            return t.reshape(b, d, w, X, w, Y).permute(0, 3, 5, 2, 4, 1)
        return t.reshape(b, d, X, w, Y, w).permute(0, 2, 4, 3, 5, 1)


class _FromWindows(nn.Module):
    """Rearrange('b x y w1 w2 d -> b d (x w1) (y w2)') (block) or '... -> b d (w1 x) (w2 y)' (grid) (reference
    max_vit.py:267, 272), without einops."""

    def __init__(self, grid: bool) -> None:
        super().__init__()
        self.grid = grid

    def forward(self, t):
        b, X, Y, w1, w2, d = t.shape
        if self.grid:
            return t.permute(0, 5, 3, 1, 4, 2).reshape(b, d, w1 * X, w2 * Y)
        return t.permute(0, 5, 1, 3, 2, 4).reshape(b, d, X * w1, Y * w2)


class SqueezeExcitation(nn.Module):
    def __init__(self, dim, shrinkage_rate=0.25):
        super().__init__()
        hidden_dim = int(dim * shrinkage_rate)

        self.gate = nn.Sequential(
            _MeanHW(),
            nn.Linear(dim, hidden_dim, bias=False),
            nn.SiLU(),
            nn.Linear(hidden_dim, dim, bias=False),
            nn.Sigmoid(),
            _Unsqueeze2()
        )

    def forward(self, x):
        return x * self.gate(x)


class MBConvResidual(nn.Module):
    def __init__(self, fn, dropout=0.):
        super().__init__()
        self.fn = fn
        self.dropsample = Dropsample(dropout)

    def forward(self, x):
        out = self.fn(x)
        out = self.dropsample(out)
        return out + x


class Dropsample(nn.Module):
    def __init__(self, prob=0):
        super().__init__()
        self.prob = prob

    def forward(self, x):
        device = x.device

        if self.prob == 0. or (not self.training):
            return x

        keep_mask = torch.FloatTensor((x.shape[0], 1, 1, 1), device=device).uniform_() > self.prob
        return x * keep_mask / (1 - self.prob)


def MBConv(
    dim_in,
    dim_out,
    *,
    downsample,
    expansion_rate=4,
    shrinkage_rate=0.25,
    dropout=0.
):
    hidden_dim = int(expansion_rate * dim_out)
    stride = 2 if downsample else 1

    net = nn.Sequential(
        nn.Conv2d(dim_in, hidden_dim, 1),
        nn.BatchNorm2d(hidden_dim),
        nn.GELU(),
        nn.Conv2d(hidden_dim, hidden_dim, 3, stride=stride, padding=1, groups=hidden_dim),
        nn.BatchNorm2d(hidden_dim),
        nn.GELU(),
        SqueezeExcitation(hidden_dim, shrinkage_rate=shrinkage_rate),
        nn.Conv2d(hidden_dim, dim_out, 1),
        nn.BatchNorm2d(dim_out)
    )

    if dim_in == dim_out and not downsample:
        net = MBConvResidual(net, dropout=dropout)

    return net


class Attention(nn.Module):
    """Window attention over (b, x, y, w1, w2, d) windows with a learned bias per head looked up from the signed
    offset between the query's and the key's local coordinates (reference max_vit.py:121-206)."""

    def __init__(
        self,
        dim,
        dim_head=32,
        dropout=0.,
        window_size=7
    ):
        super().__init__()
        assert (dim % dim_head) == 0, 'dimension should be divisible by dimension per head'

        self.heads = dim // dim_head
        self.scale = dim_head ** -0.5

        self.norm = nn.LayerNorm(dim)
        self.to_qkv = nn.Linear(dim, dim * 3, bias=False)

        self.attend = nn.Sequential(
            nn.Softmax(dim=-1),
            nn.Dropout(dropout)
        )

        self.to_out = nn.Sequential(
            nn.Linear(dim, dim, bias=False),
            nn.Dropout(dropout)
        )

        # relative positional bias

        self.rel_pos_bias = nn.Embedding((2 * window_size - 1) ** 2, self.heads)

        pos = torch.arange(window_size)
        grid = torch.stack(torch.meshgrid(pos, pos, indexing='ij'))
        grid = grid.reshape(2, -1).t()                                         # 'c i j -> (i j) c'
        rel_pos = grid[:, None, :] - grid[None, :, :]
        rel_pos += window_size - 1
        rel_pos_indices = (rel_pos * torch.tensor([2 * window_size - 1, 1])).sum(dim=-1)

        self.register_buffer('rel_pos_indices', rel_pos_indices, persistent=False)

        self.window_size = window_size
        self.dim_head = dim_head

    def forward(self, x):
        batch, height, width, window_height, window_width, _ = x.shape
        h = self.heads

        x = self.norm(x)

        # flatten: 'b x y w1 w2 d -> (b x y) (w1 w2) d'
        x = x.reshape(batch * height * width, window_height * window_width, -1)

        # project for queries, keys, values, split heads: 'b n (h d) -> b h n d'
        q, k, v = self.to_qkv(x).chunk(3, dim=-1)
        q, k, v = (t.reshape(t.shape[0], t.shape[1], h, -1).transpose(1, 2) for t in (q, k, v))

        q = q * self.scale

        sim = einsum('b h i d, b h j d -> b h i j', q, k)

        # add positional bias: 'i j h -> h i j'
        bias = self.rel_pos_bias(self.rel_pos_indices)
        sim = sim + bias.permute(2, 0, 1)

        attn = self.attend(sim)

        out = einsum('b h i j, b h j d -> b h i d', attn, v)

        # merge heads: 'b h (w1 w2) d -> b w1 w2 (h d)'
        out = out.transpose(1, 2).reshape(out.shape[0], window_height, window_width, -1)

        out = self.to_out(out)
        # '(b x y) ... -> b x y ...'
        return out.reshape(batch, height, width, *out.shape[1:])


# -------------------------------------------------------------------------------------------------- prepared weights
def mbconv_weights(mb: nn.Module) -> dict:
    """The prepared weights of one MBConv (or MBConvResidual): 'w1' bf16 / 'b1' fp32 (the 1 x 1 expansion with its
    BatchNorm folded), 'w9' fp32 [9, hidden] tap-major / 'b9' fp32 (the depthwise convolution with its BatchNorm
    folded), 'se1' / 'se2' bf16 (the squeeze-excitation Linears), 'w3' bf16 / 'b3' fp32 (the 1 x 1 projection with
    its BatchNorm folded)."""
    net = mb.fn if isinstance(mb, MBConvResidual) else mb
    conv1, bn1, _, dw, bn2, _, se, conv3, bn3 = net
    w1, b1 = fold_bn(conv1.weight, conv1.bias, bn1)
    w9, b9 = fold_bn(dw.weight, dw.bias, bn2)
    w3, b3 = fold_bn(conv3.weight, conv3.bias, bn3)
    return {"w1": _bf16_rows(w1), "b1": b1.contiguous(), "w9": w9.t().contiguous(), "b9": b9.contiguous(),
            "se1": _bf16_rows(se.gate[1].weight), "se2": _bf16_rows(se.gate[3].weight),
            "w3": _bf16_rows(w3), "b3": b3.contiguous()}


class _BlockAttention(FusedEncoder):
    """The attention and feed-forward pairs of one MaxViT block (positions 2, 3 and 6, 7 of its Sequential) as two
    EncoderLayers for the engine: block windows, then grid windows.  Not a submodule: it only reads the block's."""

    def __init__(self, block: nn.Sequential) -> None:
        self.block = block
        self.layers = (block[2], block[6])

    def parameters(self):
        return [p for i in (2, 3, 6, 7) for p in self.block[i].parameters()]

    def encoder_layers(self) -> Tuple[List[EncoderLayer], None]:
        layers = []
        for ai, fi, grid in ((2, 3, False), (6, 7, True)):
            a, f = self.block[ai].fn, self.block[fi].fn.net
            layers.append(EncoderLayer(
                ln1=Norm.of(a.norm), qkv_w=a.to_qkv.weight, out_w=a.to_out[0].weight, out_b=None, ln2=Norm.of(f[0]),
                fc1_w=f[1].weight, fc1_b=f[1].bias, fc2_w=f[4].weight, fc2_b=f[4].bias, heads=a.heads,
                dim_head=a.dim_head, scale=a.scale,
                attention=Windows(a.window_size, rel_pos_bias=a.rel_pos_bias.weight, dilated=grid)))
        return layers, None


class MaxViT(FusedWeightsMixin, nn.Module):
    def __init__(
        self,
        *,
        num_classes,
        dim,
        depth,
        dim_head=32,
        dim_conv_stem=None,
        window_size=7,
        mbconv_expansion_rate=4,
        mbconv_shrinkage_rate=0.25,
        dropout=0.1,
        channels=3
    ):
        super().__init__()
        assert isinstance(depth, tuple), 'depth needs to be tuple if integers indicating number of transformer blocks at that stage'

        # convolutional stem

        dim_conv_stem = default(dim_conv_stem, dim)

        self.conv_stem = nn.Sequential(
            nn.Conv2d(channels, dim_conv_stem, 3, stride=2, padding=1),
            nn.Conv2d(dim_conv_stem, dim_conv_stem, 3, padding=1)
        )

        # variables

        num_stages = len(depth)

        dims = tuple(map(lambda i: (2 ** i) * dim, range(num_stages)))
        dims = (dim_conv_stem, *dims)
        dim_pairs = tuple(zip(dims[:-1], dims[1:]))

        self.layers = nn.ModuleList([])

        # shorthand for window size for efficient block - grid like attention

        w = window_size

        # iterate through stages

        for ind, ((layer_dim_in, layer_dim), layer_depth) in enumerate(zip(dim_pairs, depth)):
            for stage_ind in range(layer_depth):
                is_first = stage_ind == 0
                stage_dim_in = layer_dim_in if is_first else layer_dim

                block = nn.Sequential(
                    MBConv(
                        stage_dim_in,
                        layer_dim,
                        downsample=is_first,
                        expansion_rate=mbconv_expansion_rate,
                        shrinkage_rate=mbconv_shrinkage_rate
                    ),
                    _ToWindows(w, grid=False),  # block-like attention
                    Residual(layer_dim, Attention(dim=layer_dim, dim_head=dim_head, dropout=dropout, window_size=w)),
                    Residual(layer_dim, FeedForward(dim=layer_dim, dropout=dropout)),
                    _FromWindows(grid=False),

                    _ToWindows(w, grid=True),  # grid-like attention
                    Residual(layer_dim, Attention(dim=layer_dim, dim_head=dim_head, dropout=dropout, window_size=w)),
                    Residual(layer_dim, FeedForward(dim=layer_dim, dropout=dropout)),
                    _FromWindows(grid=True),
                )

                self.layers.append(block)

        # mlp head out

        self.mlp_head = nn.Sequential(
            _MeanHW(),
            nn.LayerNorm(dims[-1]),
            nn.Linear(dims[-1], num_classes)
        )

        self.channels = channels
        self.window_size = window_size
        self._depth = depth
        self._dropout_p = float(dropout)

    # ---------------------------------------------------------------------------------------------- dispatch
    def stage_maps(self, H: int, W: int) -> List[Tuple[int, int]]:
        """The (h, w) token map of every block for an H x W image: the stem halves it (rounding up), every stage's first
        MBConv halves it again."""
        h, w = _lib.conv_out_size(H, 3, 2, 1), _lib.conv_out_size(W, 3, 2, 1)
        maps = []
        for block in self.layers:
            if not isinstance(block[0], MBConvResidual):
                h, w = -(-h // 2), -(-w // 2)
            maps.append((h, w))
        return maps

    def _encoders(self) -> List[_BlockAttention]:
        """One _BlockAttention per block, made on first use; the blocks of a stage share one engine workspace (same
        shapes, never running at the same time)."""
        encs = self.__dict__.get("_block_encoders")
        if encs is None:
            encs = []
            for block in self.layers:
                e = _BlockAttention(block)
                if isinstance(block[0], MBConvResidual):
                    e.engine().share_workspace(encs[-1].engine())
                encs.append(e)
            self.__dict__["_block_encoders"] = encs
        return encs

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4 or img.shape[1] != self.channels:
            return f"input is not (B, {self.channels}, H, W)"
        if any(d == 0 for d in self._depth):
            return "depth == 0"
        r = common_reason(self, img, dropout_p=self._dropout_p)
        if r is not None:
            return r
        r = batchnorm_reason(self)
        if r is not None:
            return r
        if self.conv_stem[0].out_channels % 8:
            return f"dim_conv_stem={self.conv_stem[0].out_channels} (the GEMMs need multiples of 8)"
        w = self.window_size
        for i, (block, (h, ww)) in enumerate(zip(self.layers, self.stage_maps(img.shape[2], img.shape[3]))):
            if h % w or ww % w:
                return f"block {i}: the {h} x {ww} map is not divisible into {w} x {w} windows (the reference raises)"
            mb = block[0]
            net = mb.fn if isinstance(mb, MBConvResidual) else mb
            widths = (net[0].in_channels, net[0].out_channels, net[6].gate[1].out_features, net[7].out_channels)
            if any(c % 8 or c == 0 for c in widths):
                return (f"block {i}: MBConv widths {widths[0]} -> {widths[1]} (squeeze-excitation {widths[2]}) -> "
                        f"{widths[3]} (the GEMMs need multiples of 8)")
        for e, (h, ww) in zip(self._encoders(), self.stage_maps(img.shape[2], img.shape[3])):
            r = e.engine().unsupported_reason(h * ww, grid=(h, ww))
            if r is not None:
                return r
        return None

    def forward(self, x):
        if self.fused_reason(x) is None:
            with on_device(x):
                return self.forward_fused(x)
        return self.forward_eager(x)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, x):
        x = self.conv_stem(x)

        for stage in self.layers:
            x = stage(x)

        return self.mlp_head(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def prepared_buffers(self) -> List[torch.Tensor]:
        """Every BatchNorm's running statistics, which the folded weights are made of, and its batch counter (as
        levit.LeViT.prepared_buffers)."""
        return [b for m in self.modules() if isinstance(m, nn.BatchNorm2d)
                for b in (m.running_mean, m.running_var, m.num_batches_tracked) if b is not None]

    def prepared(self) -> dict:
        """The stem's and every MBConv's prepared weights: 'stem<i>.w' / '.b' and '<block>.<name>' (mbconv_weights)."""
        params = list(self.conv_stem.parameters()) + [p for b in self.layers for p in b[0].parameters()]
        return cached(self, "_prepared", params + self.prepared_buffers(), self._build)

    def _build(self) -> dict:
        t = {}
        for i, conv in enumerate(self.conv_stem):
            t[f"stem{i}.w"], t[f"stem{i}.b"] = _conv_weight(conv, i > 0), conv.bias.detach().float().contiguous()
        for i, block in enumerate(self.layers):
            t.update({f"{i}.{k}": v for k, v in mbconv_weights(block[0]).items()})
        return t

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev = img.device
        bf, f32 = dict(device=dev, dtype=torch.bfloat16), dict(device=dev, dtype=torch.float32)
        t = self.prepared()
        B, _, H, W = img.shape
        # conv_stem: im2col + GEMM (with bias) twice, channels-last bf16 out
        h, w = _lib.conv_out_size(H, 3, 2, 1), _lib.conv_out_size(W, 3, 2, 1)
        a = torch.empty(B * h * w, t["stem0.w"].shape[1], **bf)
        _lib.conv_im2col_nchw(img.contiguous(), a, 3, 2, 1)
        s0 = torch.empty(B * h * w, self.conv_stem[0].out_channels, **bf)
        _lib.gemm(a, t["stem0.w"], out_bf16=s0, bias=t["stem0.b"])
        a = torch.empty(B * h * w, t["stem1.w"].shape[1], **bf)
        _lib.conv_im2col_nhwc(s0, a, B, h, w, 3, 1, 1)
        xb = torch.empty(B * h * w, self.conv_stem[1].out_channels, **bf)
        _lib.gemm(a, t["stem1.w"], out_bf16=xb, bias=t["stem1.b"])
        x = None
        for i, (block, enc) in enumerate(zip(self.layers, self._encoders())):
            p = f"{i}."
            residual = isinstance(block[0], MBConvResidual)
            s = 1 if residual else 2
            C, Cse = t[p + "w1"].shape[0], t[p + "se1"].shape[0]
            oh, ow = -(-h // s), -(-w // s)
            # MBConv: 1 x 1 + BatchNorm + GELU, depthwise 3 x 3 + BatchNorm + GELU, squeeze-excitation, 1 x 1 + BatchNorm
            hid = torch.empty(B * h * w, C, **bf)
            _lib.gemm(xb, t[p + "w1"], out_bf16=hid, bias=t[p + "b1"], gelu=True)
            hid2 = torch.empty(B * oh * ow, C, **bf)
            part = torch.empty(B, _lib.mbconv_parts(oh, ow), C, **f32)
            _lib.mbconv_dwconv(hid, t[p + "w9"], t[p + "b9"], hid2, part, B, h, w, s)
            pooled = torch.empty(B, C, **bf)
            _lib.se_pool(part, pooled, oh * ow)
            squeezed = torch.empty(B, Cse, **bf)
            _lib.gemm_silu(pooled, t[p + "se1"], out_bf16=squeezed)
            gate = torch.empty(B, C, **bf)
            _lib.gemm_sigmoid(squeezed, t[p + "se2"], out_bf16=gate)
            _lib.se_scale(hid2, gate, B, oh * ow)
            h, w = oh, ow
            if residual:
                _lib.gemm(hid2, t[p + "w3"], out_f32=x, bias=t[p + "b3"], resid=x)
            else:
                # a stage's first block: the fresh stream of the stage's width
                x = torch.empty(B * h * w, t[p + "w3"].shape[0], **f32)
                _lib.gemm(hid2, t[p + "w3"], out_f32=x, bias=t[p + "b3"])
            # block attention + FeedForward, grid attention + FeedForward
            eng = enc.engine()
            eng.run_blocks(x, B, h * w, grid=(h, w))
            xb = eng.stream_bf16(x)
        # head: the mean over the map, LayerNorm, the classifier GEMM
        D = x.shape[1]
        pm = torch.empty(B, D, **f32)
        _lib.mean_pool(x, pm, B, h * w, D)
        ln = self.mlp_head[1]
        g, b = head_norm(self, ln)
        pooled = torch.empty(B, D, **bf)
        _lib.layernorm(pm, g, b, out_bf16=pooled, eps=ln.eps)
        return head_engine(self, self.mlp_head[2]).run(pooled)
