"""Drop-in `LeViT` for lucidrains/vit-pytorch's `vit_pytorch.levit.LeViT`, with `Transformer`, `Attention`,
`FeedForward` and the helpers `exists`, `default`, `cast_tuple` and `always` of the same file, and a fused sm_90a
forward.

Same constructor keywords, parameter and buffer names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed): `conv_embedding.{0..3}` the four stride-2 convolutions, `backbone.i` the
Transformers (each stage's, then the downsampling one before the next stage), `Attention` = `to_q`, `to_k`, `to_v`
(1 x 1 Conv2d + BatchNorm2d each), `to_out` (GELU, Conv2d, BatchNorm2d with its weight initialised to zero, Dropout),
`pos_bias` (an Embedding of F*F rows by heads) and the `pos_indices` buffer; `distill_head` (when
`num_distill_classes` is set) and `mlp_head` (reference levit.py:27-195).  The PyTorch graph below mirrors the
reference module for module, so hooks on any submodule keep working there, and it raises where the reference raises.

Fused forward, on the token-major map x fp32 [B*F*F, C] (token (b, y, x) at row (b*F + y)*F + x) and its bf16 copy:
  * conv_embedding (levit.py:153-158): b200vit_conv_im2col_nchw on the image, then three times
    b200vit_conv_im2col_nhwc on the previous convolution's bf16 channels-last output, each followed by its GEMM with
    the bias; the last GEMM writes the fp32 stream and its bf16 copy;
  * per Transformer layer, five launches: the QKV GEMM over [to_q; to_k; to_v] with each BatchNorm folded into its rows
    and a bias, b200vit_attention_posbias with the bias table pos_bias.weight^T / scale and GELU on its output (the
    downsampling layer's stride-2 queries are gathered from the same full-grid QKV), the to_out GEMM with its
    BatchNorm folded (with the residual in place, or, for the downsampling layer, into the next stage's fresh stream),
    the fc1 GEMM with Hardswish, the fc2 GEMM with the residual (levit.py:110-127);
  * head: b200vit_mean_pool, the cast to bf16, then one GEMM over [mlp_head; distill_head], split into
    (out, distill) when there is a distill head (levit.py:174-195).
BatchNorm runs on its running statistics: a BatchNorm2d in training mode (batch statistics mix the images of a batch)
sends the call to the PyTorch graph.  There is no LayerNorm in the model, so B200VIT_LN_MODE changes nothing here.
"""
from __future__ import annotations

from math import ceil
from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import FusedWeightsMixin, _bf16_rows, _f32, cached, common_reason, on_device
from .xcit import batchnorm_reason

__all__ = ["Attention", "FeedForward", "LeViT", "Transformer", "always", "attention_weights", "bias_table",
           "cast_tuple", "default", "exists", "fold_bn", "posbias_reason"]

DIM_KEYS = (16, 32, 64)          # b200vit_attention_posbias
DIM_VALUES = (32, 64, 128)
MAX_KEYS = _lib.ATTN_POSBIAS_MAX_KEYS


def exists(val):
    return val is not None


def default(val, d):
    return val if exists(val) else d


def cast_tuple(val, l=3):
    val = val if isinstance(val, tuple) else (val,)
    return (*val, *((val[-1],) * max(l - len(val), 0)))


def always(val):
    return lambda *args, **kwargs: val


class FeedForward(nn.Module):
    def __init__(self, dim, mult, dropout=0.):
        super().__init__()
        self.net = nn.Sequential(
            nn.Conv2d(dim, dim * mult, 1),
            nn.Hardswish(),
            nn.Dropout(dropout),
            nn.Conv2d(dim * mult, dim, 1),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        return self.net(x)


class Attention(nn.Module):
    """q / k heads dim_key wide, v heads dim_value wide, a learned bias per head looked up from |dy| * F + |dx|, GELU
    before the output projection; to_q has stride 2 when `downsample` (reference levit.py:40-108)."""

    def __init__(self, dim, fmap_size, heads=8, dim_key=32, dim_value=64, dropout=0., dim_out=None, downsample=False):
        super().__init__()
        inner_dim_key = dim_key * heads
        inner_dim_value = dim_value * heads
        dim_out = default(dim_out, dim)

        self.heads = heads
        self.scale = dim_key ** -0.5

        self.to_q = nn.Sequential(nn.Conv2d(dim, inner_dim_key, 1, stride=(2 if downsample else 1), bias=False),
                                  nn.BatchNorm2d(inner_dim_key))
        self.to_k = nn.Sequential(nn.Conv2d(dim, inner_dim_key, 1, bias=False), nn.BatchNorm2d(inner_dim_key))
        self.to_v = nn.Sequential(nn.Conv2d(dim, inner_dim_value, 1, bias=False), nn.BatchNorm2d(inner_dim_value))

        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)

        out_batch_norm = nn.BatchNorm2d(dim_out)
        nn.init.zeros_(out_batch_norm.weight)

        self.to_out = nn.Sequential(
            nn.GELU(),
            nn.Conv2d(inner_dim_value, dim_out, 1),
            out_batch_norm,
            nn.Dropout(dropout)
        )

        # positional bias

        self.pos_bias = nn.Embedding(fmap_size * fmap_size, heads)

        q_range = torch.arange(0, fmap_size, step=(2 if downsample else 1))
        k_range = torch.arange(fmap_size)

        q_pos = torch.stack(torch.meshgrid(q_range, q_range, indexing='ij'), dim=-1)
        k_pos = torch.stack(torch.meshgrid(k_range, k_range, indexing='ij'), dim=-1)

        q_pos, k_pos = (t.reshape(-1, 2) for t in (q_pos, k_pos))
        rel_pos = (q_pos[:, None, ...] - k_pos[None, :, ...]).abs()

        x_rel, y_rel = rel_pos.unbind(dim=-1)
        pos_indices = (x_rel * fmap_size) + y_rel

        self.register_buffer('pos_indices', pos_indices)

        self.fmap_size = fmap_size
        self.dim_key = dim_key
        self.dim_value = dim_value
        self.stride = 2 if downsample else 1

    def apply_pos_bias(self, fmap):
        bias = self.pos_bias(self.pos_indices)
        bias = bias.permute(2, 0, 1).unsqueeze(0)              # 'i j h -> () h i j'
        return fmap + (bias / self.scale)

    def forward(self, x):
        b, n, *_, h = *x.shape, self.heads

        q = self.to_q(x)
        y = q.shape[2]

        qkv = (q, self.to_k(x), self.to_v(x))
        # 'b (h d) ... -> b h (...) d'
        q, k, v = (t.reshape(b, h, t.shape[1] // h, -1).transpose(2, 3) for t in qkv)

        dots = torch.einsum('b h i d, b h j d -> b h i j', q, k) * self.scale

        dots = self.apply_pos_bias(dots)

        attn = self.attend(dots)
        attn = self.dropout(attn)

        out = torch.einsum('b h i j, b h j d -> b h i d', attn, v)
        # 'b h (x y) d -> b (h d) x y' with y = the query map's width
        out = out.transpose(2, 3).reshape(b, -1, out.shape[2] // y, y)
        return self.to_out(out)


class Transformer(nn.Module):
    def __init__(self, dim, fmap_size, depth, heads, dim_key, dim_value, mlp_mult=2, dropout=0., dim_out=None,
                 downsample=False):
        super().__init__()
        dim_out = default(dim_out, dim)
        self.layers = nn.ModuleList([])
        self.attn_residual = (not downsample) and dim == dim_out

        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, fmap_size=fmap_size, heads=heads, dim_key=dim_key, dim_value=dim_value,
                          dropout=dropout, downsample=downsample, dim_out=dim_out),
                FeedForward(dim_out, mlp_mult, dropout=dropout)
            ]))

    def forward(self, x):
        for attn, ff in self.layers:
            attn_res = (x if self.attn_residual else 0)
            x = attn(x) + attn_res
            x = ff(x) + x
        return x


class _Squeeze(nn.Module):
    """Rearrange('... () () -> ...') (reference levit.py:176), without einops."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if x.shape[-2:] != (1, 1):
            raise RuntimeError(f"Rearrange('... () () -> ...'): the last two dims are {tuple(x.shape[-2:])}")
        return x.reshape(x.shape[:-2])


# -------------------------------------------------------------------------------------------------- prepared weights
def fold_bn(w: torch.Tensor, b: Optional[torch.Tensor], bn: nn.BatchNorm2d) -> Tuple[torch.Tensor, torch.Tensor]:
    """(w', b') fp32 of a 1 x 1 convolution [out, in(, 1, 1)] with bias b (or None) followed by BatchNorm2d `bn` in
    eval mode:  w' = w g / sqrt(var + eps),  b' = (b - mean) g / sqrt(var + eps) + beta  (as engine.lpi_weights)."""
    f = lambda t: t.detach().float()                                                    # noqa: E731
    inv = f(bn.weight) / torch.sqrt(f(bn.running_var) + bn.eps)
    w2 = f(w).reshape(w.shape[0], -1) * inv[:, None]
    b0 = f(b) if b is not None else torch.zeros_like(inv)
    return w2, (b0 - f(bn.running_mean)) * inv + f(bn.bias)


def bias_table(attn: Attention) -> torch.Tensor:
    """fp32 [heads, F*F]: pos_bias.weight^T / scale, what b200vit_attention_posbias adds at index |dy| * F + |dx|."""
    return (attn.pos_bias.weight.detach().float().t() / attn.scale).contiguous()


def attention_weights(attn: Attention, ff: FeedForward) -> dict:
    """The prepared weights of one layer: 'qkv.w' bf16 / 'qkv.b' fp32 ([to_q; to_k; to_v] with their BatchNorms
    folded), 'table' (bias_table), 'out.w' / 'out.b' (to_out's convolution with its BatchNorm folded), 'fc1.w' /
    'fc1.b', 'fc2.w' / 'fc2.b'."""
    parts = [fold_bn(seq[0].weight, None, seq[1]) for seq in (attn.to_q, attn.to_k, attn.to_v)]
    ow, ob = fold_bn(attn.to_out[1].weight, attn.to_out[1].bias, attn.to_out[2])
    fc1, fc2 = ff.net[0], ff.net[3]
    return {"qkv.w": _bf16_rows(torch.cat([w for w, _ in parts])), "qkv.b": torch.cat([b for _, b in parts]).contiguous(),
            "table": bias_table(attn), "out.w": _bf16_rows(ow), "out.b": ob.contiguous(),
            "fc1.w": _bf16_rows(fc1.weight.reshape(fc1.out_channels, -1)), "fc1.b": _f32(fc1.bias),
            "fc2.w": _bf16_rows(fc2.weight.reshape(fc2.out_channels, -1)), "fc2.b": _f32(fc2.bias)}


def posbias_reason(attn: Attention) -> Optional[str]:
    """None if b200vit_attention_posbias is built for this Attention's widths and key count, else why not."""
    if attn.dim_key not in DIM_KEYS:
        return f"dim_key={attn.dim_key} (the position-bias attention kernel is built for 16, 32 and 64)"
    if attn.dim_value not in DIM_VALUES:
        return f"dim_value={attn.dim_value} (the position-bias attention kernel is built for 32, 64 and 128)"
    if attn.fmap_size ** 2 > MAX_KEYS:
        return f"{attn.fmap_size ** 2} keys (the position-bias attention kernel takes at most {MAX_KEYS})"
    return None


def _conv_weight(conv: nn.Conv2d, channels_last_input: bool) -> torch.Tensor:
    """bf16 [Cout, K] GEMM weight with K padded to a multiple of 8: columns (cin, ky, kx) for the NCHW image, (ky, kx,
    cin) for a channels-last input (b200vit_conv_im2col_nchw / _nhwc)."""
    w = conv.weight.detach()
    if channels_last_input:
        w = w.permute(0, 2, 3, 1)
    w = w.reshape(w.shape[0], -1)
    return _bf16_rows(w, (w.shape[1] + 7) // 8 * 8)


class LeViT(FusedWeightsMixin, nn.Module):
    def __init__(
        self,
        *,
        image_size,
        num_classes,
        dim,
        depth,
        heads,
        mlp_mult,
        stages=3,
        dim_key=32,
        dim_value=64,
        dropout=0.,
        num_distill_classes=None
    ):
        super().__init__()

        dims = cast_tuple(dim, stages)
        depths = cast_tuple(depth, stages)
        layer_heads = cast_tuple(heads, stages)

        assert all(map(lambda t: len(t) == stages, (dims, depths, layer_heads))), \
            'dimensions, depths, and heads must be a tuple that is less than the designated number of stages'

        self.conv_embedding = nn.Sequential(
            nn.Conv2d(3, 32, 3, stride=2, padding=1),
            nn.Conv2d(32, 64, 3, stride=2, padding=1),
            nn.Conv2d(64, 128, 3, stride=2, padding=1),
            nn.Conv2d(128, dims[0], 3, stride=2, padding=1)
        )

        fmap_size = image_size // (2 ** 4)
        layers = []

        for ind, dim, depth, heads in zip(range(stages), dims, depths, layer_heads):
            is_last = ind == (stages - 1)
            layers.append(Transformer(dim, fmap_size, depth, heads, dim_key, dim_value, mlp_mult, dropout))

            if not is_last:
                next_dim = dims[ind + 1]
                layers.append(Transformer(dim, fmap_size, 1, heads * 2, dim_key, dim_value, dim_out=next_dim,
                                          downsample=True))
                fmap_size = ceil(fmap_size / 2)

        self.backbone = nn.Sequential(*layers)

        self.pool = nn.Sequential(
            nn.AdaptiveAvgPool2d(1),
            _Squeeze()
        )

        self.distill_head = nn.Linear(dim, num_distill_classes) if exists(num_distill_classes) else always(None)
        self.mlp_head = nn.Linear(dim, num_classes)

        self._dropout_p = float(dropout)

    # ---------------------------------------------------------------------------------------------- dispatch
    def conv_grid(self, H: int, W: int) -> Optional[Tuple[List[Tuple[int, int]], int, int]]:
        """(per convolution of conv_embedding its output (h, w), the final h, w) for an H x W image; None where a
        convolution has no output (the reference's Conv2d raises)."""
        grids = []
        for _ in self.conv_embedding:
            H, W = _lib.conv_out_size(H, 3, 2, 1), _lib.conv_out_size(W, 3, 2, 1)
            if H < 1 or W < 1:
                return None
            grids.append((H, W))
        return grids, H, W

    def transformers(self) -> List[Transformer]:
        return list(self.backbone)

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4 or img.shape[1] != 3:
            return "input is not (B, 3, H, W)"
        r = common_reason(self, img, encoders=self.transformers(), dropout_p=self._dropout_p)
        if r is not None:
            return r
        r = batchnorm_reason(self)
        if r is not None:
            return r
        first = self.transformers()[0].layers[0][0]
        g = self.conv_grid(img.shape[2], img.shape[3])
        if g is None:
            return "a convolution of conv_embedding has no output for this image (the reference raises)"
        _, h, w = g
        if h != first.fmap_size or w != first.fmap_size:
            return (f"the convolutions give a {h} x {w} grid, not the {first.fmap_size} x {first.fmap_size} of the "
                    f"position bias (the reference's bias add fails)")
        for t in self.transformers():
            for attn, ff in t.layers:
                r = posbias_reason(attn)
                if r is not None:
                    return r
                for c in (attn.to_q[0], attn.to_v[0], attn.to_out[1], ff.net[0], ff.net[3]):
                    if c.in_channels % 8 or c.out_channels % 8:
                        return (f"a 1 x 1 convolution of {c.in_channels} -> {c.out_channels} channels (the GEMMs need "
                                "multiples of 8)")
        return None

    def forward(self, img):
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, img):
        x = self.conv_embedding(img)

        x = self.backbone(x)

        x = self.pool(x)

        out = self.mlp_head(x)
        distill = self.distill_head(x)

        if exists(distill):
            return out, distill

        return out

    # ---------------------------------------------------------------------------------------------- fused kernels
    def prepared_buffers(self) -> List[torch.Tensor]:
        """Every BatchNorm's running statistics, which the folded weights are made of, and its batch counter (a
        train-mode forward updates the statistics in place without bumping their version counters, but its
        `num_batches_tracked.add_(1)` bumps the counter's)."""
        return [b for m in self.modules() if isinstance(m, nn.BatchNorm2d)
                for b in (m.running_mean, m.running_var, m.num_batches_tracked) if b is not None]

    def prepared(self) -> dict:
        """Every prepared weight, keyed '<transformer>.<layer>.<name>' (attention_weights), 'conv<i>.w' / '.b' and
        'head.w' / 'head.b' ([mlp_head; distill_head])."""
        return cached(self, "_prepared", list(self.parameters()) + self.prepared_buffers(), self._build)

    def _build(self) -> dict:
        t = {}
        for i, conv in enumerate(self.conv_embedding):
            t[f"conv{i}.w"], t[f"conv{i}.b"] = _conv_weight(conv, i > 0), _f32(conv.bias)
        for i, tr in enumerate(self.transformers()):
            for j, (attn, ff) in enumerate(tr.layers):
                t.update({f"{i}.{j}.{k}": v for k, v in attention_weights(attn, ff).items()})
        heads = [self.mlp_head] + ([self.distill_head] if isinstance(self.distill_head, nn.Linear) else [])
        t["head.w"] = _bf16_rows(torch.cat([h.weight.detach() for h in heads]))
        t["head.b"] = torch.cat([_f32(h.bias) for h in heads]).contiguous()
        return t

    def forward_fused(self, img: torch.Tensor):
        dev, bf = img.device, dict(device=img.device, dtype=torch.bfloat16)
        f32 = dict(device=img.device, dtype=torch.float32)
        t = self.prepared()
        B = img.shape[0]
        grids, _, _ = self.conv_grid(img.shape[2], img.shape[3])
        # conv_embedding: im2col + GEMM (with bias) four times, channels-last bf16 in between
        src, (H, W) = img.contiguous(), img.shape[2:]
        x = xb = None
        for i, (conv, (oh, ow)) in enumerate(zip(self.conv_embedding, grids)):
            w = t[f"conv{i}.w"]
            a = torch.empty(B * oh * ow, w.shape[1], **bf)
            if i == 0:
                _lib.conv_im2col_nchw(src, a, 3, 2, 1)
            else:
                _lib.conv_im2col_nhwc(src, a, B, H, W, 3, 2, 1)
            if i + 1 < len(grids):
                src = torch.empty(B * oh * ow, conv.out_channels, **bf)
                _lib.gemm(a, w, out_bf16=src, bias=t[f"conv{i}.b"])
            else:
                x = torch.empty(B * oh * ow, conv.out_channels, **f32)
                xb = torch.empty(B * oh * ow, conv.out_channels, **bf)
                _lib.gemm(a, w, out_f32=x, out_bf16=xb, bias=t[f"conv{i}.b"])
            H, W = oh, ow
        # backbone: five launches per layer
        F = H
        for i, tr in enumerate(self.transformers()):
            for j, (attn, ff) in enumerate(tr.layers):
                p = f"{i}.{j}."
                Hh, dk, dv, s = attn.heads, attn.dim_key, attn.dim_value, attn.stride
                Fq = -(-F // s)
                qkv = torch.empty(B * F * F, t[p + "qkv.w"].shape[0], **bf)
                _lib.gemm(xb, t[p + "qkv.w"], out_bf16=qkv, bias=t[p + "qkv.b"])
                o = torch.empty(B * Fq * Fq, Hh * dv, **bf)
                _lib.attention_posbias(qkv, o, t[p + "table"], B, F, s, Hh, dk, dv, attn.scale, gelu_out=True)
                D = t[p + "out.w"].shape[0]
                if tr.attn_residual:
                    _lib.gemm(o, t[p + "out.w"], out_f32=x, out_bf16=xb, bias=t[p + "out.b"], resid=x)
                else:
                    # the downsampling layer (and any layer without the attention residual): a fresh stream
                    x = torch.empty(B * Fq * Fq, D, **f32)
                    xb = torch.empty(B * Fq * Fq, D, **bf)
                    _lib.gemm(o, t[p + "out.w"], out_f32=x, out_bf16=xb, bias=t[p + "out.b"])
                F = Fq
                hdn = torch.empty(B * F * F, t[p + "fc1.w"].shape[0], **bf)
                _lib.gemm_hardswish(xb, t[p + "fc1.w"], out_bf16=hdn, bias=t[p + "fc1.b"])
                _lib.gemm(hdn, t[p + "fc2.w"], out_f32=x, out_bf16=xb, bias=t[p + "fc2.b"], resid=x)
        # head: the mean over the map, then [mlp_head; distill_head] as one GEMM
        D = x.shape[1]
        pm = torch.empty(B, D, **f32)
        _lib.mean_pool(x, pm, B, F * F, D)
        pooled = torch.empty(B, D, **bf)
        _lib.cast_f32_bf16(pm, pooled)
        out = torch.empty(B, t["head.w"].shape[0], **bf)
        _lib.gemm(pooled, t["head.w"], out_bf16=out, bias=t["head.b"])
        nc = self.mlp_head.out_features
        if isinstance(self.distill_head, nn.Linear):
            return out[:, :nc], out[:, nc:]
        return out
