"""Drop-in `CvT` for lucidrains/vit-pytorch's `vit_pytorch.cvt.CvT` (convolutional token embeddings and convolutional
projections), with `Transformer`, `Attention`, `DepthWiseConv2d`, `FeedForward`, `LayerNorm` and the helpers
`group_dict_by_key` and `group_by_key_prefix_and_remove_prefix` of the same file, and a fused sm_90a forward.

Same constructor keywords, parameter and buffer names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed): `layers.{0,1,2}` the three stages, each `Sequential(Conv2d, LayerNorm,
Transformer)`, and `to_logits` (average pool, the parameter-free squeeze, Linear) (reference cvt.py:114-173).  The
PyTorch graph below mirrors the reference module for module, without einops, so hooks on any submodule keep working
there, and it raises where the reference raises.

Fused forward, channels-last throughout: token (b, y, x) of an h x w map is row (b*h + y)*w + x of the fp32 stream
[B*h*w, D] and of its bf16 copy.  Per stage:
  * the convolutional embedding (cvt.py:156-157): b200vit_conv_im2col_nchw of the image (stage 1) or
    b200vit_conv_im2col_nhwc of the previous stage's bf16 stream copy, the GEMM with bias into fp32, then
    b200vit_embed_tokens for the channel LayerNorm, writing the stage's stream and, in fold mode, its bf16 copy and row
    statistics;
  * the Transformer through TransformerEngine.run_blocks with the stage's grid.  Per layer: layernorm(x -> xb),
    b200vit_conv_proj_dw (both depthwise projections with their BatchNorms folded, from one read of xb), the query and
    key / value 1 x 1 GEMMs, b200vit_attention_kv, the out-projection GEMM with the residual; then the pre-LN
    feed-forward block (engine.py);
  * head: b200vit_mean_pool over the last map, the cast to bf16, the classifier GEMM.
BatchNorm runs on its running statistics: a BatchNorm2d in training mode sends the call to the PyTorch graph.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import einsum, nn

from . import _lib
from .cct import CONV_MAX_KERNEL
from .engine import (ConvProj, EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, _bf16_rows, _f32, cached,
                     common_reason, head_engine, on_device)
from .levit import _Squeeze
from .xcit import batchnorm_reason

__all__ = ["Attention", "CvT", "DepthWiseConv2d", "FeedForward", "LayerNorm", "Transformer",
           "group_by_key_prefix_and_remove_prefix", "group_dict_by_key"]


def group_dict_by_key(cond, d):
    return_val = [dict(), dict()]
    for key in d.keys():
        match = bool(cond(key))
        ind = int(not match)
        return_val[ind][key] = d[key]
    return (*return_val,)


def group_by_key_prefix_and_remove_prefix(prefix, d):
    kwargs_with_prefix, kwargs = group_dict_by_key(lambda x: x.startswith(prefix), d)
    kwargs_without_prefix = dict(map(lambda x: (x[0][len(prefix):], x[1]), tuple(kwargs_with_prefix.items())))
    return kwargs_without_prefix, kwargs


class LayerNorm(nn.Module):
    """LayerNorm over the channel dim of an NCHW map: biased variance, eps inside the square root, affine `g` / `b` of
    shape (1, dim, 1, 1) (reference cvt.py:25-35)."""

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
    def __init__(self, dim, mult=4, dropout=0.):
        super().__init__()
        self.net = nn.Sequential(
            LayerNorm(dim),
            nn.Conv2d(dim, dim * mult, 1),
            nn.GELU(),
            nn.Dropout(dropout),
            nn.Conv2d(dim * mult, dim, 1),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        return self.net(x)


class DepthWiseConv2d(nn.Module):
    def __init__(self, dim_in, dim_out, kernel_size, padding, stride, bias=True):
        super().__init__()
        self.net = nn.Sequential(
            nn.Conv2d(dim_in, dim_in, kernel_size=kernel_size, padding=padding, groups=dim_in, stride=stride,
                      bias=bias),
            nn.BatchNorm2d(dim_in),
            nn.Conv2d(dim_in, dim_out, kernel_size=1, bias=bias)
        )

    def forward(self, x):
        return self.net(x)


def _heads(t: torch.Tensor, h: int) -> torch.Tensor:
    """'b (h d) x y -> (b h) (x y) d'"""
    b, c, x, y = t.shape
    return t.reshape(b * h, c // h, x * y).transpose(1, 2)


class Attention(nn.Module):
    def __init__(self, dim, proj_kernel, kv_proj_stride, heads=8, dim_head=64, dropout=0.):
        super().__init__()
        inner_dim = dim_head * heads
        padding = proj_kernel // 2
        self.heads = heads
        self.scale = dim_head ** -0.5

        self.norm = LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)

        self.to_q = DepthWiseConv2d(dim, inner_dim, proj_kernel, padding=padding, stride=1, bias=False)
        self.to_kv = DepthWiseConv2d(dim, inner_dim * 2, proj_kernel, padding=padding, stride=kv_proj_stride,
                                     bias=False)

        self.to_out = nn.Sequential(
            nn.Conv2d(inner_dim, dim, 1),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        b, _, _, y = x.shape
        h = self.heads

        x = self.norm(x)
        q, k, v = (self.to_q(x), *self.to_kv(x).chunk(2, dim=1))
        q, k, v = (_heads(t, h) for t in (q, k, v))

        dots = einsum('b i d, b j d -> b i j', q, k) * self.scale

        attn = self.attend(dots)
        attn = self.dropout(attn)

        out = einsum('b i j, b j d -> b i d', attn, v)
        n = out.shape[1]
        if n % y:
            # what einops raises for '(b h) (x y) d -> b (h d) x y' (an even proj_kernel grows the query map by one)
            raise RuntimeError(f"Rearrange: {n} query tokens do not split into rows of y={y} (cvt.py:96)")
        out = out.reshape(b, h, n, -1).permute(0, 1, 3, 2).reshape(b, -1, n // y, y)
        return self.to_out(out)


class Transformer(FusedEncoder, nn.Module):
    """depth x (Attention, FeedForward), each added to the stream (reference cvt.py:99-112).  The fused forward runs it
    through engine()."""

    def __init__(self, dim, proj_kernel, kv_proj_stride, depth, heads, dim_head=64, mlp_mult=4, dropout=0.):
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, proj_kernel=proj_kernel, kv_proj_stride=kv_proj_stride, heads=heads,
                          dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mlp_mult, dropout=dropout)
            ]))

    def forward(self, x):
        for attn, ff in self.layers:
            x = attn(x) + x
            x = ff(x) + x
        return x

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        """One EncoderLayer per (Attention, FeedForward) pair, with ConvProj: qkv_w the queries' 1 x 1 rows, kv_proj_w
        the keys' and values' (rows k | v, the order of chunk(2, dim=1))."""
        layers = []
        for a, ff in self.layers:
            f = ff.net
            dq, bq, pq = a.to_q.net
            dkv, bkv, pkv = a.to_kv.net
            D, I = dq.in_channels, pq.out_channels
            P = ConvProj(q_w=dq.weight, q_bn_w=bq.weight, q_bn_b=bq.bias, q_bn_mean=bq.running_mean,
                         q_bn_var=bq.running_var, q_bn_eps=bq.eps, kv_w=dkv.weight, kv_bn_w=bkv.weight,
                         kv_bn_b=bkv.bias, kv_bn_mean=bkv.running_mean, kv_bn_var=bkv.running_var, kv_bn_eps=bkv.eps,
                         kernel_size=dq.kernel_size[0], stride=dkv.stride[0], kv_proj_w=pkv.weight.reshape(2 * I, D))
            layers.append(EncoderLayer(
                ln1=_norm(a.norm), qkv_w=pq.weight.reshape(I, D), out_w=a.to_out[0].weight.reshape(D, I),
                out_b=a.to_out[0].bias, ln2=_norm(f[0]), fc1_w=f[1].weight.reshape(-1, D), fc1_b=f[1].bias,
                fc2_w=f[4].weight.reshape(D, -1), fc2_b=f[4].bias, heads=a.heads, dim_head=I // a.heads,
                scale=a.scale, attention=P))
        return layers, None

    def prepared_buffers(self) -> List[torch.Tensor]:
        """Every BatchNorm's running statistics, which the folded projection weights are made of, and its batch counter
        (as levit.LeViT.prepared_buffers)."""
        return [b for m in self.modules() if isinstance(m, nn.BatchNorm2d)
                for b in (m.running_mean, m.running_var, m.num_batches_tracked) if b is not None]


def embed_weights(conv: nn.Conv2d, ln: LayerNorm, channels_last_input: bool) -> dict:
    """The prepared weights of a stage's convolutional embedding: 'w' bf16 [emb_dim, K] (columns (cin, ky, kx) for
    the NCHW image with K zero-padded to a multiple of 64, (ky, kx, cin) for a channels-last map), 'b' fp32 (its
    bias), 'g' / 'beta' fp32 (the channel LayerNorm)."""
    w = conv.weight.detach()
    if channels_last_input:
        w = w.permute(0, 2, 3, 1)
    w = w.reshape(w.shape[0], -1)
    kp = w.shape[1] if channels_last_input else (w.shape[1] + 63) // 64 * 64
    return {"w": _bf16_rows(w, kp), "b": _f32(conv.bias), "g": _f32(ln.g.reshape(-1)), "beta": _f32(ln.b.reshape(-1))}


class CvT(FusedWeightsMixin, nn.Module):
    def __init__(
        self,
        *,
        num_classes,
        s1_emb_dim=64,
        s1_emb_kernel=7,
        s1_emb_stride=4,
        s1_proj_kernel=3,
        s1_kv_proj_stride=2,
        s1_heads=1,
        s1_depth=1,
        s1_mlp_mult=4,
        s2_emb_dim=192,
        s2_emb_kernel=3,
        s2_emb_stride=2,
        s2_proj_kernel=3,
        s2_kv_proj_stride=2,
        s2_heads=3,
        s2_depth=2,
        s2_mlp_mult=4,
        s3_emb_dim=384,
        s3_emb_kernel=3,
        s3_emb_stride=2,
        s3_proj_kernel=3,
        s3_kv_proj_stride=2,
        s3_heads=6,
        s3_depth=10,
        s3_mlp_mult=4,
        dropout=0.,
        channels=3
    ):
        super().__init__()
        kwargs = dict(locals())

        dim = channels
        layers = []

        for prefix in ('s1', 's2', 's3'):
            config, kwargs = group_by_key_prefix_and_remove_prefix(f'{prefix}_', kwargs)

            layers.append(nn.Sequential(
                nn.Conv2d(dim, config['emb_dim'], kernel_size=config['emb_kernel'],
                          padding=(config['emb_kernel'] // 2), stride=config['emb_stride']),
                LayerNorm(config['emb_dim']),
                Transformer(dim=config['emb_dim'], proj_kernel=config['proj_kernel'],
                            kv_proj_stride=config['kv_proj_stride'], depth=config['depth'], heads=config['heads'],
                            mlp_mult=config['mlp_mult'], dropout=dropout)
            ))

            dim = config['emb_dim']

        self.layers = nn.Sequential(*layers)

        self.to_logits = nn.Sequential(
            nn.AdaptiveAvgPool2d(1),
            _Squeeze(),
            nn.Linear(dim, num_classes)
        )
        self.channels = channels
        self._dropout_p = float(dropout)

    # ---------------------------------------------------------------------------------------------- dispatch
    def stage_maps(self, H: int, W: int) -> List[Tuple[int, int]]:
        """The (h, w) token map of every stage for an H x W image (each embedding convolution pads k // 2), up to the
        first empty one."""
        maps = []
        for stage in self.layers:
            conv = stage[0]
            k, s = conv.kernel_size[0], conv.stride[0]
            H, W = _lib.conv_out_size(H, k, s, k // 2), _lib.conv_out_size(W, k, s, k // 2)
            maps.append((H, W))
            if H < 1 or W < 1:
                break
        return maps

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4 or img.shape[1] != self.channels:
            return f"input is not (B, {self.channels}, H, W)"
        r = common_reason(self, img, encoders=[s[2] for s in self.layers], dropout_p=self._dropout_p)
        if r is None:
            r = batchnorm_reason(self)
        if r is not None:
            return r
        for i, stage in enumerate(self.layers):
            conv = stage[0]
            if conv.out_channels % 8:
                return f"stage {i + 1}: emb_dim={conv.out_channels} (the kernels need multiples of 8)"
            if conv.kernel_size[0] > CONV_MAX_KERNEL:
                return f"stage {i + 1}: emb_kernel={conv.kernel_size[0]} (the im2col kernels take at most " \
                       f"{CONV_MAX_KERNEL})"
        for i, ((h, w), stage) in enumerate(zip(self.stage_maps(img.shape[2], img.shape[3]), self.layers)):
            if h < 1 or w < 1:
                return f"stage {i + 1}: the map of a {img.shape[2]} x {img.shape[3]} image is empty"
            # the engine's rules: proj_kernel 1, 3, 5 or 7 (an even one also makes the reference raise), dim_head,
            # at most 16384 tokens (and so keys) per map
            r = stage[2].engine().unsupported_reason(h * w, grid=(h, w))
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
        latents = self.layers(x)
        return self.to_logits(latents)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def _embed_weights(self, i: int, stage: nn.Sequential) -> dict:
        conv, ln = stage[0], stage[1]
        return cached(self, f"_embed{i}", list(conv.parameters()) + list(ln.parameters()),
                      lambda: embed_weights(conv, ln, i > 0))

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev, bf = img.device, dict(device=img.device, dtype=torch.bfloat16)
        B = img.shape[0]
        src, H, W = img.contiguous(), img.shape[2], img.shape[3]
        x = None
        for i, (stage, (h, w)) in enumerate(zip(self.layers, self.stage_maps(H, W))):
            # the convolutional embedding: im2col + GEMM with bias, then the channel LayerNorm into the stream
            conv, ln, t = stage
            m = self._embed_weights(i, stage)
            k, s = conv.kernel_size[0], conv.stride[0]
            M, D = B * h * w, conv.out_channels
            a = torch.empty(M, m["w"].shape[1], **bf)
            if i == 0:
                _lib.conv_im2col_nchw(src, a, k, s, k // 2)
            else:
                _lib.conv_im2col_nhwc(src, a, B, H, W, k, s, k // 2)
            y = torch.empty(M, D, device=dev, dtype=torch.float32)
            _lib.gemm(a, m["w"], out_f32=y, bias=m["b"])
            eng = t.engine()
            xb, stats = eng.entry_buffers(M, dev)
            x = torch.empty(M, D, device=dev, dtype=torch.float32)
            _lib.embed_tokens(y, m["g"], m["beta"], None, None, x, B, h * w, 0, eps=ln.eps, xb=xb, stats=stats)
            eng.run_blocks(x, B, h * w, primed=xb is not None, grid=(h, w))
            src, H, W = eng.stream_bf16(x), h, w
        # head: the mean over the last map, then the classifier GEMM
        D = x.shape[1]
        pm = torch.empty(B, D, device=dev, dtype=torch.float32)
        _lib.mean_pool(x, pm, B, H * W, D)
        pooled = torch.empty(B, D, **bf)
        _lib.cast_f32_bf16(pm, pooled)
        return head_engine(self, self.to_logits[2]).run(pooled)
