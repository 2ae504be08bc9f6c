"""Drop-in `CrossFormer` for lucidrains/vit-pytorch's `vit_pytorch.crossformer.CrossFormer` (cross-scale embeddings and
short / long distance window attention under a dynamic position bias), with `CrossEmbedLayer`, `DynamicPositionBias`,
`LayerNorm`, `FeedForward`, `Attention`, `Transformer` and the helper `cast_tuple` of the same file, and a fused sm_90a
forward.

Same constructor keywords, parameter and buffer names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed): `layers.i` the four stages, each `ModuleList(CrossEmbedLayer,
Transformer)`, and `to_logits` (mean, Linear) (reference crossformer.py:175-245).  `rel_pos_indices` stays a
non-persistent buffer.  The PyTorch graph below mirrors the reference module for module, without einops, so hooks on
any submodule keep working there, and it raises where the reference raises: a bf16 model raises in the dynamic position
bias (the reference feeds it float32 offsets, crossformer.py:149), scales whose maps differ raise in `torch.cat`, a map a
window does not divide raises in the window rearrangement.

Fused forward, channels-last throughout: token (b, y, x) of an h x w map is row (b*h + y)*w + x of the fp32 stream
[B*h*w, D] and of its bf16 copy.  No token is ever moved into window order; only the attention kernel knows the
partition, as an address map.  Per stage:
  * the cross-scale embedding (crossformer.py:14-36): stage 1 is one b200vit_cross_embed_nchw launch over the image
    (every scale, their concatenation and biases, written into the fp32 stream); later stages run, per scale,
    b200vit_conv_im2col_nhwc of the previous stage's bf16 stream copy and a GEMM with bias into the scale's column slice
    of the fp32 stream;
  * the Transformer through TransformerEngine.run_blocks with the stage's grid.  Each depth step is two EncoderLayers:
    short-distance attention (block windows of `local_window_size`) + FeedForward, then long-distance attention (grid
    windows of `global_window_size`) + FeedForward, the attention by b200vit_attention_window_relpos under the dynamic
    position bias table.  In fold mode the first layer's rowstats_cast writes the stream's bf16 copy and row statistics;
  * head: b200vit_mean_pool over the last map, the cast to bf16, the classifier GEMM.
The dynamic position bias depends on the parameters only, so it is evaluated once per weight version, in fp32 from the
(bf16) parameters, when the engine's prepared weights are built.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import einsum, nn

from . import _lib
from .cct import CONV_MAX_KERNEL
from .engine import (EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, Windows, _bf16_rows, _f32, cached,
                     common_reason, head_engine, on_device)
from .max_vit import _MeanHW

__all__ = ["Attention", "CrossEmbedLayer", "CrossFormer", "DynamicPositionBias", "FeedForward", "LayerNorm",
           "Transformer", "cast_tuple", "dpb_table"]


def cast_tuple(val, length=1):
    return val if isinstance(val, tuple) else ((val,) * length)


class CrossEmbedLayer(nn.Module):
    def __init__(
        self,
        dim_in,
        dim_out,
        kernel_sizes,
        stride=2
    ):
        super().__init__()
        kernel_sizes = sorted(kernel_sizes)
        num_scales = len(kernel_sizes)

        # calculate the dimension at each scale
        dim_scales = [int(dim_out / (2 ** i)) for i in range(1, num_scales)]
        dim_scales = [*dim_scales, dim_out - sum(dim_scales)]

        self.convs = nn.ModuleList([])
        for kernel, dim_scale in zip(kernel_sizes, dim_scales):
            self.convs.append(nn.Conv2d(dim_in, dim_scale, kernel, stride=stride, padding=(kernel - stride) // 2))

    def forward(self, x):
        fmaps = tuple(map(lambda conv: conv(x), self.convs))
        return torch.cat(fmaps, dim=1)


class _SqueezeLast(nn.Module):
    """Rearrange('... () -> ...') (reference crossformer.py:53), without einops."""

    def forward(self, x):
        if x.shape[-1] != 1:
            raise RuntimeError(f"Rearrange('... () -> ...'): last axis has length {x.shape[-1]}, not 1")
        return x.squeeze(-1)


def DynamicPositionBias(dim):
    return nn.Sequential(
        nn.Linear(2, dim),
        nn.LayerNorm(dim),
        nn.ReLU(),
        nn.Linear(dim, dim),
        nn.LayerNorm(dim),
        nn.ReLU(),
        nn.Linear(dim, dim),
        nn.LayerNorm(dim),
        nn.ReLU(),
        nn.Linear(dim, 1),
        _SqueezeLast()
    )


class LayerNorm(nn.Module):
    """LayerNorm over the channel dim of an NCHW map: biased variance, eps inside the square root, affine `g` / `b` of
    shape (1, dim, 1, 1) (reference crossformer.py:58-68)."""

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
    return Norm(ln.g.view(-1), ln.b.view(-1), ln.eps)


def FeedForward(dim, mult=4, dropout=0.):
    return nn.Sequential(
        LayerNorm(dim),
        nn.Conv2d(dim, dim * mult, 1),
        nn.GELU(),
        nn.Dropout(dropout),
        nn.Conv2d(dim * mult, dim, 1)
    )


def _rel_offsets(w: int, device) -> torch.Tensor:
    """The (2w + 1)^2 offsets in [-w, w]^2, row-major, as float32 [(2w + 1)^2, 2] (reference crossformer.py:146-148)."""
    pos = torch.arange(-w, w + 1, device=device)
    return torch.stack(torch.meshgrid(pos, pos, indexing='ij')).reshape(2, -1).t().float()


def _to_windows(x: torch.Tensor, w: int, long: bool) -> torch.Tensor:
    """'b d (h s1) (w s2) -> (b h w) d s1 s2' (short) or 'b d (l1 h) (l2 w) -> (b h w) d l1 l2' (long), window w
    (reference crossformer.py:127-131); raises where einops does."""
    b, d, H, W = x.shape
    if H % w or W % w:
        raise RuntimeError(f"Rearrange: a {H} x {W} map is not divisible into {w} x {w} windows")
    X, Y = H // w, W // w
    if long:
        return x.reshape(b, d, w, X, w, Y).permute(0, 3, 5, 1, 2, 4).reshape(b * X * Y, d, w, w)
    return x.reshape(b, d, X, w, Y, w).permute(0, 2, 4, 1, 3, 5).reshape(b * X * Y, d, w, w)


def _from_windows(x: torch.Tensor, b: int, X: int, Y: int, long: bool) -> torch.Tensor:
    """The inverse of _to_windows (reference crossformer.py:159-163)."""
    _, d, w, _ = x.shape
    x = x.reshape(b, X, Y, d, w, w)
    if long:
        return x.permute(0, 3, 4, 1, 5, 2).reshape(b, d, w * X, w * Y)
    return x.permute(0, 3, 1, 4, 2, 5).reshape(b, d, X * w, Y * w)


class Attention(nn.Module):
    def __init__(
        self,
        dim,
        attn_type,
        window_size,
        dim_head=32,
        dropout=0.
    ):
        super().__init__()
        assert attn_type in {'short', 'long'}, 'attention type must be one of local or distant'
        heads = dim // dim_head
        self.heads = heads
        self.scale = dim_head ** -0.5
        inner_dim = dim_head * heads

        self.attn_type = attn_type
        self.window_size = window_size

        self.norm = LayerNorm(dim)

        self.dropout = nn.Dropout(dropout)

        self.to_qkv = nn.Conv2d(dim, inner_dim * 3, 1, bias=False)
        self.to_out = nn.Conv2d(inner_dim, dim, 1)

        # positions

        self.dpb = DynamicPositionBias(dim // 4)

        # calculate and store indices for retrieving bias

        pos = torch.arange(window_size)
        grid = torch.stack(torch.meshgrid(pos, pos, indexing='ij'))
        grid = grid.reshape(2, -1).t()                                         # 'c i j -> (i j) c'
        rel_pos = grid[:, None] - grid[None, :]
        rel_pos += window_size - 1
        rel_pos_indices = (rel_pos * torch.tensor([2 * window_size - 1, 1])).sum(dim=-1)

        self.register_buffer('rel_pos_indices', rel_pos_indices, persistent=False)

    def forward(self, x):
        b, _, height, width = x.shape
        heads, wsz, device = self.heads, self.window_size, x.device
        long = self.attn_type == 'long'

        # prenorm
        x = self.norm(x)

        # rearrange for short or long distance attention
        x = _to_windows(x, wsz, long)

        # queries / keys / values, split heads: 'b (h d) x y -> b h (x y) d'
        q, k, v = self.to_qkv(x).chunk(3, dim=1)
        q, k, v = (t.reshape(t.shape[0], heads, -1, wsz * wsz).transpose(2, 3) for t in (q, k, v))
        q = q * self.scale

        sim = einsum('b h i d, b h j d -> b h i j', q, k)

        # add dynamic positional bias (float32 offsets, as the reference: a bf16 model raises here)
        biases = self.dpb(_rel_offsets(wsz, device))
        rel_pos_bias = biases[self.rel_pos_indices]

        sim = sim + rel_pos_bias

        # attend
        attn = sim.softmax(dim=-1)
        attn = self.dropout(attn)

        # merge heads: 'b h (x y) d -> b (h d) x y'
        out = einsum('b h i j, b h j d -> b h i d', attn, v)
        out = out.transpose(2, 3).reshape(out.shape[0], -1, wsz, wsz)
        out = self.to_out(out)

        # rearrange back for long or short distance attention
        return _from_windows(out, b, height // wsz, width // wsz, long)


def dpb_table(attn: Attention) -> torch.Tensor:
    """The relative-position table b200vit_attention_window_relpos reads for `attn`: fp32 [(2w - 1)^2, heads].  The
    reference evaluates its DynamicPositionBias at the (2w + 1)^2 offsets in [-w, w]^2 but indexes the outputs with the
    stride 2w - 1 of `rel_pos_indices` (crossformer.py:115, 149-150), so the table is the FIRST (2w - 1)^2 outputs in
    order, shared by all heads.  Evaluated in fp32 from the parameters whatever their dtype, without autograd."""
    w = attn.window_size
    with torch.no_grad():
        x = _rel_offsets(w, attn.rel_pos_indices.device)
        for m in attn.dpb:
            if isinstance(m, nn.Linear):
                x = F.linear(x, m.weight.float(), m.bias.float())
            elif isinstance(m, nn.LayerNorm):
                x = F.layer_norm(x, m.normalized_shape, m.weight.float(), m.bias.float(), m.eps)
            elif isinstance(m, nn.ReLU):
                x = F.relu(x)
            else:
                x = m(x)
        return x[: (2 * w - 1) ** 2, None].expand(-1, attn.heads).contiguous()


class Transformer(FusedEncoder, nn.Module):
    """depth x (short Attention, FeedForward, long Attention, FeedForward), each added to the stream (reference
    crossformer.py:167-199).  The fused forward runs it through engine()."""

    def __init__(
        self,
        dim,
        *,
        local_window_size,
        global_window_size,
        depth=4,
        dim_head=32,
        attn_dropout=0.,
        ff_dropout=0.,
    ):
        super().__init__()
        self.layers = nn.ModuleList([])

        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, attn_type='short', window_size=local_window_size, dim_head=dim_head,
                          dropout=attn_dropout),
                FeedForward(dim, dropout=ff_dropout),
                Attention(dim, attn_type='long', window_size=global_window_size, dim_head=dim_head,
                          dropout=attn_dropout),
                FeedForward(dim, dropout=ff_dropout)
            ]))

    def forward(self, x):
        for short_attn, short_ff, long_attn, long_ff in self.layers:
            x = short_attn(x) + x
            x = short_ff(x) + x
            x = long_attn(x) + x
            x = long_ff(x) + x

        return x

    def encoder_layers(self) -> Tuple[List[EncoderLayer], None]:
        """Two EncoderLayers per depth step: (short attention, FeedForward) over block windows, then (long attention,
        FeedForward) over grid windows, each with its dynamic position bias table (dpb_table)."""
        layers = []
        for step in self.layers:
            for a, f in ((step[0], step[1]), (step[2], step[3])):
                I, D = a.to_qkv.out_channels // 3, a.to_qkv.in_channels
                layers.append(EncoderLayer(
                    ln1=_norm(a.norm), qkv_w=a.to_qkv.weight.reshape(3 * I, D),
                    out_w=a.to_out.weight.reshape(D, I), out_b=a.to_out.bias, ln2=_norm(f[0]),
                    fc1_w=f[1].weight.reshape(-1, D), fc1_b=f[1].bias, fc2_w=f[4].weight.reshape(D, -1),
                    fc2_b=f[4].bias, heads=a.heads, dim_head=I // a.heads, scale=a.scale,
                    attention=Windows(a.window_size, rel_pos_bias=dpb_table(a), dilated=a.attn_type == 'long')))
        return layers, None


def embed_weights(cel: CrossEmbedLayer, first: bool) -> dict:
    """The prepared weights of a stage's cross-scale embedding.  Stage 1 ('w' bf16 packed by _lib.cross_embed_pack,
    'b' fp32 every scale's bias in output column order); later stages, per scale i, 'w<i>' bf16 [n_i, k*k*C] in the
    column order (tap row, tap column, channel) of b200vit_conv_im2col_nhwc and 'b<i>' fp32."""
    if first:
        return {"w": _lib.cross_embed_pack([c.weight for c in cel.convs]),
                "b": torch.cat([_f32(c.bias) for c in cel.convs])}
    t = {}
    for i, c in enumerate(cel.convs):
        t[f"w{i}"] = _bf16_rows(c.weight.detach().permute(0, 2, 3, 1).reshape(c.out_channels, -1))
        t[f"b{i}"] = _f32(c.bias)
    return t


def _stage_reason(i: int, cel: CrossEmbedLayer, cin: int) -> Optional[str]:
    """Why stage i's cross-scale embedding cannot run fused (its shapes only), or None."""
    widths = [c.out_channels for c in cel.convs]
    ks = [c.kernel_size[0] for c in cel.convs]
    s = cel.convs[0].stride[0]
    dim = sum(widths)
    if dim % 8 or any(n % 8 for n in widths):
        return f"stage {i + 1}: dim {dim} with scale widths {widths} (the kernels need multiples of 8)"
    if dim < 32:
        return f"stage {i + 1}: dim {dim} < dim_head 32 (no attention heads)"
    if any(k < s for k in ks):
        return f"stage {i + 1}: kernel sizes {ks} below the stride {s} (negative padding)"
    if i == 0:
        if (len(ks) > _lib.CROSS_EMBED_MAX_SCALES or cin > _lib.CROSS_EMBED_MAX_CHANNELS
                or max(ks) > _lib.CROSS_EMBED_MAX_KERNEL or s > _lib.CROSS_EMBED_MAX_STRIDE
                or max(widths) > _lib.CROSS_EMBED_MAX_WIDTH):
            return (f"stage 1: {len(ks)} scales, kernels {ks}, stride {s}, widths {widths} on {cin} channels (the "
                    f"cross-scale embedding kernel takes at most {_lib.CROSS_EMBED_MAX_SCALES} scales, kernel "
                    f"{_lib.CROSS_EMBED_MAX_KERNEL}, stride {_lib.CROSS_EMBED_MAX_STRIDE}, width "
                    f"{_lib.CROSS_EMBED_MAX_WIDTH}, {_lib.CROSS_EMBED_MAX_CHANNELS} channels)")
    elif max(ks) > CONV_MAX_KERNEL:
        return f"stage {i + 1}: kernel sizes {ks} (the im2col kernel takes at most {CONV_MAX_KERNEL})"
    return None


class CrossFormer(FusedWeightsMixin, nn.Module):
    def __init__(
        self,
        *,
        dim=(64, 128, 256, 512),
        depth=(2, 2, 8, 2),
        global_window_size=(8, 4, 2, 1),
        local_window_size=7,
        cross_embed_kernel_sizes=((4, 8, 16, 32), (2, 4), (2, 4), (2, 4)),
        cross_embed_strides=(4, 2, 2, 2),
        num_classes=1000,
        attn_dropout=0.,
        ff_dropout=0.,
        channels=3
    ):
        super().__init__()

        dim = cast_tuple(dim, 4)
        depth = cast_tuple(depth, 4)
        global_window_size = cast_tuple(global_window_size, 4)
        local_window_size = cast_tuple(local_window_size, 4)
        cross_embed_kernel_sizes = cast_tuple(cross_embed_kernel_sizes, 4)
        cross_embed_strides = cast_tuple(cross_embed_strides, 4)

        assert len(dim) == 4
        assert len(depth) == 4
        assert len(global_window_size) == 4
        assert len(local_window_size) == 4
        assert len(cross_embed_kernel_sizes) == 4
        assert len(cross_embed_strides) == 4

        # dimensions

        last_dim = dim[-1]
        dims = [channels, *dim]
        dim_in_and_out = tuple(zip(dims[:-1], dims[1:]))

        # layers

        self.layers = nn.ModuleList([])

        for (dim_in, dim_out), layers, global_wsz, local_wsz, cel_kernel_sizes, cel_stride in zip(
                dim_in_and_out, depth, global_window_size, local_window_size, cross_embed_kernel_sizes,
                cross_embed_strides):
            self.layers.append(nn.ModuleList([
                CrossEmbedLayer(dim_in, dim_out, cel_kernel_sizes, stride=cel_stride),
                Transformer(dim_out, local_window_size=local_wsz, global_window_size=global_wsz, depth=layers,
                            attn_dropout=attn_dropout, ff_dropout=ff_dropout)
            ]))

        # final logits

        self.to_logits = nn.Sequential(
            _MeanHW(),
            nn.Linear(last_dim, num_classes)
        )
        self.channels = channels
        self._dropout_p = max(float(attn_dropout), float(ff_dropout))

    # ---------------------------------------------------------------------------------------------- dispatch
    def stage_maps(self, H: int, W: int) -> List[List[Tuple[int, int]]]:
        """Per stage, the (h, w) map every scale of its cross-scale embedding gives (padding (k - s) // 2), each stage
        fed the first scale's map of the one before, up to the first stage whose scales disagree or whose map is
        empty."""
        maps = []
        for cel, _ in self.layers:
            ms = []
            for c in cel.convs:
                k, s = c.kernel_size[0], c.stride[0]
                p = (k - s) // 2
                ms.append((_lib.conv_out_size(H, k, s, p), _lib.conv_out_size(W, k, s, p)))
            maps.append(ms)
            H, W = ms[0]
            if len(set(ms)) > 1 or H < 1 or W < 1:
                break
        return maps

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4 or img.shape[1] != self.channels:
            return f"input is not (B, {self.channels}, H, W)"
        r = common_reason(self, img, encoders=[t for _, t in self.layers], dropout_p=self._dropout_p)
        if r is not None:
            return r
        cin = self.channels
        for i, (cel, _) in enumerate(self.layers):
            r = _stage_reason(i, cel, cin)
            if r is not None:
                return r
            cin = sum(c.out_channels for c in cel.convs)
        maps = self.stage_maps(img.shape[2], img.shape[3])
        for i, ((cel, t), ms) in enumerate(zip(self.layers, maps)):
            if len(set(ms)) > 1:
                return f"stage {i + 1}: the scales give maps {ms} (the reference's torch.cat raises)"
            h, w = ms[0]
            if h < 1 or w < 1:
                return f"stage {i + 1}: the map of a {img.shape[2]} x {img.shape[3]} image is empty"
            for name, a in (("local", t.layers[0][0]), ("global", t.layers[0][2])):
                ws = a.window_size
                if h % ws or w % ws:
                    return (f"stage {i + 1}: the {h} x {w} map is not divisible into {name} {ws} x {ws} windows (the "
                            f"reference raises)")
            r = t.engine().unsupported_reason(h * w, grid=(h, w))
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
        for cel, transformer in self.layers:
            x = cel(x)
            x = transformer(x)

        return self.to_logits(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def _embed_weights(self, i: int, cel: CrossEmbedLayer) -> dict:
        return cached(self, f"_embed{i}", list(cel.parameters()), lambda: embed_weights(cel, i == 0))

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev = img.device
        bf, f32 = dict(device=dev, dtype=torch.bfloat16), dict(device=dev, dtype=torch.float32)
        B = img.shape[0]
        src, H, W = img.contiguous(), img.shape[2], img.shape[3]
        x = None
        for i, ((cel, t), ms) in enumerate(zip(self.layers, self.stage_maps(H, W))):
            m = self._embed_weights(i, cel)
            h, w = ms[0]
            widths = [c.out_channels for c in cel.convs]
            ks = [c.kernel_size[0] for c in cel.convs]
            s = cel.convs[0].stride[0]
            M = B * h * w
            x = torch.empty(M, sum(widths), **f32)
            if i == 0:
                # every scale of the image's embedding in one launch
                _lib.cross_embed_nchw(src, m["w"], m["b"], x, ks, widths, s)
            else:
                # per scale: im2col of the previous stream copy, the GEMM with bias into the scale's column slice
                off = 0
                for j, (k, n) in enumerate(zip(ks, widths)):
                    a = torch.empty(M, m[f"w{j}"].shape[1], **bf)
                    _lib.conv_im2col_nhwc(src, a, B, H, W, k, s, (k - s) // 2)
                    _lib.gemm(a, m[f"w{j}"], out_f32=x[:, off:off + n], bias=m[f"b{j}"])
                    off += n
            eng = t.engine()
            eng.run_blocks(x, B, h * w, grid=(h, w))
            src, H, W = eng.stream_bf16(x), h, w
        # head: the mean over the last map, then the classifier GEMM
        D = x.shape[1]
        pm = torch.empty(B, D, **f32)
        _lib.mean_pool(x, pm, B, H * W, D)
        pooled = torch.empty(B, D, **bf)
        _lib.cast_f32_bf16(pm, pooled)
        return head_engine(self, self.to_logits[1]).run(pooled)
