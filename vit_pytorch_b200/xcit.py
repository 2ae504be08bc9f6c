"""Drop-in `XCiT` for lucidrains/vit-pytorch's `vit_pytorch.xcit.XCiT` (cross-covariance image transformer), with
`XCATransformer`, `Transformer`, `XCAttention`, `Attention`, `LocalPatchInteraction`, `FeedForward`, `LayerScale` and
`dropout_layers` of the same file, and a fused sm_90a forward.

Same constructor keywords, parameter and buffer names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed): `xcit_transformer.layers.i.{0,1,2}.{scale, fn}` (LayerScale's `scale` is a
(dim,) vector), `XCAttention` = `temperature` (heads, 1, 1), `norm`, `to_qkv`, `to_out`; `LocalPatchInteraction.net` =
LayerNorm, (rearrange), depthwise Conv2d, BatchNorm2d (with its running statistics), GELU, depthwise Conv2d,
(rearrange); `pos_embedding` (1, num_patches, dim) without a cls row, `cls_token` (dim,), `final_norm`,
`cls_transformer`, `mlp_head.{0,1}` (reference xcit.py:42-283).  The PyTorch graph below mirrors the reference module
for module, with 4-D (b, h, w, d) tokens into `xcit_transformer`, so hooks on any submodule keep working there.

Fused forward (engine.py):
  * patch embedding as vit.py (patchify, LayerNorm, Linear, LayerNorm) plus the positional table, no cls row
    (xcit.py:263-268);
  * xcit_transformer: per kept layer the LN-folded QKV GEMM, b200vit_attention_xca (softmax over channels, tau =
    temperature.exp()), the to_out GEMM with LayerScale folded in and the residual, b200vit_local_patch_interaction
    (LayerNorm, conv1 with BatchNorm folded in, GELU, conv2 with LayerScale folded in, residual) into a second fp32
    stream with its bf16 copy and row statistics, the LN-folded fc1 GEMM + GELU on it, and the fc2 GEMM (LayerScale
    folded in) with that stream as the residual, written back to the first (xcit.py:205-213);
  * final_norm of the patch rows, in bf16: the context of the class stage (xcit.py:276);
  * cls_transformer (xcit.py:278-281): one stacked to_kv GEMM of all class-attention layers over the context, then per
    kept layer LayerNorm of the cls rows, [to_q; to_kv] GEMM, b200vit_attention_cls, to_out GEMM with the residual,
    LayerNorm, fc1 GEMM + GELU, fc2 GEMM with the residual (CrossAttentionEngine);
  * head: LayerNorm of mlp_head[0] on the cls rows, then the head GEMM (xcit.py:283).
Layer dropout (xcit.py:25-38) draws its subset on every call, in eval too, from the same CPU generator in the same order
as the reference: the XCA transformer first, then the cls transformer.  BatchNorm runs on its running statistics: a
BatchNorm2d in training mode (batch statistics mix the images of a batch) sends the call to the PyTorch graph.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from .cait import dropout_layers
from .engine import (CrossAttentionEngine, CrossCovariance, CrossLayer, EncoderLayer, FeedForwardBlock,
                     FusedWeightsMixin, LPIBlock, Norm, _f32, cached, cls_row_index, common_reason, head_engine,
                     head_ln_pool, lpi_reason, on_device, patch_engine)
from . import _lib
from .vit import FeedForward, FusedTransformer, Patchify

__all__ = ["Attention", "FeedForward", "LayerScale", "LocalPatchInteraction", "Transformer", "XCAttention",
           "XCATransformer", "XCiT", "dropout_layers"]


class LayerScale(nn.Module):
    """fn(x) times a learned (dim,) vector whose initial value depends on the layer's depth (reference
    xcit.py:42-56)."""

    def __init__(self, dim: int, fn: nn.Module, depth: int) -> None:
        super().__init__()
        # the reference's condition, kept as written: `18 > depth <= 24` is False for every depth above 18, so layers
        # 19 and later start at 1e-6
        if depth <= 18:
            init_eps = 0.1
        elif 18 > depth <= 24:
            init_eps = 1e-5
        else:
            init_eps = 1e-6
        self.fn = fn
        self.scale = nn.Parameter(torch.full((dim,), init_eps))

    def forward(self, x: torch.Tensor, **kwargs) -> torch.Tensor:
        return self.fn(x, **kwargs) * self.scale


class Attention(nn.Module):
    """Pre-LN attention of the class stage; with `context`, the keys and values come from [LN(x); context] (reference
    xcit.py:72-107)."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, dropout: float = 0.) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.norm = nn.LayerNorm(dim)
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim, inner_dim * 2, bias=False)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout))

    def forward(self, x: torch.Tensor, context: Optional[torch.Tensor] = None) -> torch.Tensor:
        b, n, _ = x.shape
        h = self.heads
        x = self.norm(x)
        context = x if context is None else torch.cat((x, context), dim=1)
        k, v = self.to_kv(context).chunk(2, dim=-1)
        q, k, v = (t.reshape(b, t.shape[1], h, -1).transpose(1, 2) for t in (self.to_q(x), k, v))
        sim = torch.einsum('b h i d, b h j d -> b h i j', q, k) * self.scale
        attn = self.dropout(self.attend(sim))
        out = torch.einsum('b h i j, b h j d -> b h i d', attn, v)
        out = out.transpose(1, 2).reshape(b, n, -1)
        return self.to_out(out)


class XCAttention(nn.Module):
    """Cross-covariance attention: softmax over the channels of each head of the L2-normalised q^T k, scaled by a
    learned per-head temperature.exp() (reference xcit.py:109-148).  Takes tokens of any shape (b, ..., d)."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, dropout: float = 0.) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.dim_head = dim_head
        self.norm = nn.LayerNorm(dim)
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        self.temperature = nn.Parameter(torch.ones(heads, 1, 1))
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        shape = x.shape
        b, h = shape[0], self.heads
        x = self.norm(x.reshape(b, -1, shape[-1]))
        n = x.shape[1]
        q, k, v = self.to_qkv(x).chunk(3, dim=-1)
        q, k, v = (t.reshape(b, n, h, -1).permute(0, 2, 3, 1) for t in (q, k, v))      # b h d n
        q, k = F.normalize(q, dim=-1, p=2), F.normalize(k, dim=-1, p=2)
        sim = torch.einsum('b h i n, b h j n -> b h i j', q, k) * self.temperature.exp()
        attn = self.dropout(self.attend(sim))
        out = torch.einsum('b h i j, b h j n -> b h i n', attn, v)
        out = out.permute(0, 3, 1, 2).reshape(b, n, -1)                                # b n (h d)
        return self.to_out(out.reshape(*shape[:-1], -1))


class _Permute(nn.Module):
    """The reference's Rearrange between channels-last tokens and channels-first maps (no parameters)."""

    def __init__(self, *dims: int) -> None:
        super().__init__()
        self.dims = dims

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x.permute(*self.dims)

    def extra_repr(self) -> str:
        return f"dims={self.dims}"


class LocalPatchInteraction(nn.Module):
    """LayerNorm, then depthwise k x k conv, BatchNorm2d, GELU, depthwise k x k conv over the (b, h, w, d) token grid
    (reference xcit.py:150-167)."""

    def __init__(self, dim: int, kernel_size: int = 3) -> None:
        super().__init__()
        assert (kernel_size % 2) == 1
        padding = kernel_size // 2
        self.net = nn.Sequential(
            nn.LayerNorm(dim),
            _Permute(0, 3, 1, 2),                  # b h w c -> b c h w
            nn.Conv2d(dim, dim, kernel_size, padding=padding, groups=dim),
            nn.BatchNorm2d(dim),
            nn.GELU(),
            nn.Conv2d(dim, dim, kernel_size, padding=padding, groups=dim),
            _Permute(0, 2, 3, 1),                  # b c h w -> b h w c
        )

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.net(x)


def batchnorm_reason(module: nn.Module) -> Optional[str]:
    """None if every BatchNorm2d inside `module` normalises with running statistics, else the reason the eager PyTorch
    graph is used: batch statistics mix the images of a batch, which no per-sample kernel computes."""
    for m in module.modules():
        if isinstance(m, nn.BatchNorm2d) and (m.training or m.running_mean is None or m.running_var is None):
            return "a BatchNorm2d is in training mode or has no running statistics (batch statistics)"
    return None


class Transformer(nn.Module):
    """The class stage: depth x (LayerScale(Attention), LayerScale(FeedForward)) residual blocks over the cls rows with
    the patch rows as context, with layer dropout (reference xcit.py:169-189).  The fused forward runs it through
    CrossAttentionEngine."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.,
                 layer_dropout: float = 0.) -> None:
        super().__init__()
        self.layers = nn.ModuleList([])
        self.layer_dropout = layer_dropout
        self.dropout_p = float(dropout)
        for ind in range(depth):
            layer = ind + 1
            self.layers.append(nn.ModuleList([
                LayerScale(dim, Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout), depth=layer),
                LayerScale(dim, FeedForward(dim, mlp_dim, dropout=dropout), depth=layer),
            ]))

    def forward(self, x: torch.Tensor, context: Optional[torch.Tensor] = None) -> torch.Tensor:
        for attn, ff in dropout_layers(self.layers, dropout=self.layer_dropout):
            x = attn(x, context=context) + x
            x = ff(x) + x
        return x

    def kept_layers(self) -> List[int]:
        """The indices of the layers this call runs (draws exactly what the PyTorch graph's call draws)."""
        return list(dropout_layers(list(range(len(self.layers))), dropout=self.layer_dropout))

    # ---------------------------------------------------------------------------------------------- fused kernels
    def cross_params(self, direction: int) -> List[torch.Tensor]:
        return list(self.parameters())

    def cross_layers(self, direction: int) -> List[CrossLayer]:
        """The layers as class attention over a context (CrossAttentionEngine): the cls rows query [LN(cls); context]."""
        out = []
        for ls_attn, ls_ff in self.layers:
            attn, ff = ls_attn.fn, ls_ff.fn
            o = attn.to_out[0]
            out.append(CrossLayer(
                proj_in=None, ln=Norm.of(attn.norm), q_w=attn.to_q.weight, kv_w=attn.to_kv.weight, out_w=o.weight,
                out_b=o.bias, proj_out=None, heads=attn.heads, dim_head=attn.dim_head, scale=float(attn.scale),
                out_scale=ls_attn.scale,
                ff=FeedForwardBlock(Norm.of(ff.net[0]), ff.net[1].weight, ff.net[1].bias, ff.net[4].weight,
                                    ff.net[4].bias),
                ff_scale=ls_ff.scale))
        return out

    def cross_engine(self) -> CrossAttentionEngine:
        eng = self.__dict__.get("_cross_engine")
        if eng is None:
            eng = self._cross_engine = CrossAttentionEngine(self, 0)
        return eng


class XCATransformer(FusedTransformer):
    """depth x (LayerScale(XCAttention), LayerScale(LocalPatchInteraction), LayerScale(FeedForward)) residual blocks
    with layer dropout, no final LayerNorm (reference xcit.py:191-213).  Callable on (B, H, W, D) tokens; runs fused
    when eligible."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, local_patch_kernel_size: int = 3,
                 dropout: float = 0., layer_dropout: float = 0.) -> None:
        super().__init__()
        self.layers = nn.ModuleList([])
        self.layer_dropout = layer_dropout
        self.dropout_p = float(dropout)
        for ind in range(depth):
            layer = ind + 1
            self.layers.append(nn.ModuleList([
                LayerScale(dim, XCAttention(dim, heads=heads, dim_head=dim_head, dropout=dropout), depth=layer),
                LayerScale(dim, LocalPatchInteraction(dim, local_patch_kernel_size), depth=layer),
                LayerScale(dim, FeedForward(dim, mlp_dim, dropout=dropout), depth=layer),
            ]))

    def forward_eager(self, x: torch.Tensor) -> torch.Tensor:
        for cross_covariance_attn, local_patch_interaction, ff in dropout_layers(self.layers, dropout=self.layer_dropout):
            x = cross_covariance_attn(x) + x
            x = local_patch_interaction(x) + x
            x = ff(x) + x
        return x

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(x) is None:
            B, H, W, D = x.shape
            out = self.engine().forward_tokens(x.reshape(B, H * W, D), layers=self.kept_layers(), grid=(H, W))
            return out.view(B, H, W, D)
        return self.forward_eager(x)

    def fused_reason(self, x: torch.Tensor) -> Optional[str]:
        """None if forward(x) will run the fused kernels, else why not."""
        r = common_reason(self, x, encoders=(self,), dropout_p=self.dropout_p, inside="transformer")
        if r is None and x.dim() != 4:
            r = "input is not (B, H, W, D)"
        return r or self.grid_reason(x.shape[1], x.shape[2])

    def grid_reason(self, h: int, w: int) -> Optional[str]:
        """The shape-dependent part of fused_reason for an h x w token grid."""
        r = batchnorm_reason(self) or self.engine().unsupported_reason(h * w)
        return r or lpi_reason(self.layers[0][1].fn.net[2].kernel_size[0], w)

    def kept_layers(self) -> List[int]:
        """The indices of the layers this call runs (draws exactly what the PyTorch graph's call draws)."""
        return list(dropout_layers(list(range(len(self.layers))), dropout=self.layer_dropout))

    # ---------------------------------------------------------------------------------------------- fused kernels
    def prepared_buffers(self) -> List[torch.Tensor]:
        """BatchNorm's running statistics, which the folded conv1 weights are made of, and its batch counter.  A
        train-mode forward updates the statistics in place without bumping their version counters, but its
        `num_batches_tracked.add_(1)` bumps the counter's, so the key changes after it as after an explicit in-place
        write to the statistics."""
        return [b for _, lpi, _ in self.layers
                for b in (lpi.fn.net[3].running_mean, lpi.fn.net[3].running_var, lpi.fn.net[3].num_batches_tracked)
                if b is not None]

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        layers = []
        for ls_attn, ls_lpi, ls_ff in self.layers:
            attn, net, ff = ls_attn.fn, ls_lpi.fn.net, ls_ff.fn
            fc1, fc2, out = ff.net[1], ff.net[4], attn.to_out[0]
            conv1, bn, conv2 = net[2], net[3], net[5]
            layers.append(EncoderLayer(
                ln1=Norm.of(attn.norm), qkv_w=attn.to_qkv.weight, out_w=out.weight, out_b=out.bias,
                ln2=Norm.of(ff.net[0]), fc1_w=fc1.weight, fc1_b=fc1.bias, fc2_w=fc2.weight, fc2_b=fc2.bias,
                heads=attn.heads, dim_head=attn.dim_head, scale=1.0, out_scale=ls_attn.scale, ff_scale=ls_ff.scale,
                attention=CrossCovariance(attn.temperature),
                lpi=LPIBlock(ln=Norm.of(net[0]), conv1_w=conv1.weight, conv1_b=conv1.bias, bn_w=bn.weight,
                             bn_b=bn.bias, bn_mean=bn.running_mean, bn_var=bn.running_var, bn_eps=bn.eps,
                             conv2_w=conv2.weight, conv2_b=conv2.bias, scale=ls_lpi.scale,
                             kernel_size=conv1.kernel_size[0])))
        return layers, None


class _Patchify2d(Patchify):
    """'b c (h p1) (w p2) -> b h w (p1 p2 c)' (the Rearrange at reference xcit.py:240)."""

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        b, _, hh, ww = img.shape
        return super().forward(img).reshape(b, hh // self.patch_height, ww // self.patch_width, -1)


class XCiT(FusedWeightsMixin, nn.Module):
    # the cls token is not part of the patch sequence: it joins in the class stage
    cls_in_sequence = False

    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, cls_depth, heads, mlp_dim, dim_head=64,
                 dropout=0., emb_dropout=0., local_patch_kernel_size=3, layer_dropout=0.) -> None:
        super().__init__()
        assert image_size % patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        num_patches = (image_size // patch_size) ** 2
        patch_dim = 3 * patch_size ** 2
        self.patch_size = (patch_size, patch_size)

        self.to_patch_embedding = nn.Sequential(
            _Patchify2d(patch_size, patch_size),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.pos_embedding = nn.Parameter(torch.randn(1, num_patches, dim))
        self.cls_token = nn.Parameter(torch.randn(dim))
        self.dropout = nn.Dropout(emb_dropout)
        self.xcit_transformer = XCATransformer(dim, depth, heads, dim_head, mlp_dim, local_patch_kernel_size, dropout,
                                               layer_dropout)
        self.final_norm = nn.LayerNorm(dim)
        self.cls_transformer = Transformer(dim, cls_depth, heads, dim_head, mlp_dim, dropout, layer_dropout)
        self.mlp_head = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, num_classes))

        self._emb_dropout_p = float(emb_dropout)
        self._rows: dict = {}

    # ---------------------------------------------------------------------------------------------- dispatch
    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        ph, pw = self.patch_size
        if img.shape[1] * ph * pw != self.to_patch_embedding[1].normalized_shape[0]:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        xt, ct = self.xcit_transformer, self.cls_transformer
        r = common_reason(self, img, encoders=(xt, ct),
                          dropout_p=max(self._emb_dropout_p, xt.dropout_p, ct.dropout_p))
        if r is not None:
            return r
        if img.shape[2] % ph or img.shape[3] % pw:
            return "image not divisible by the patch size"
        gh, gw = img.shape[2] // ph, img.shape[3] // pw
        if gh * gw > self.pos_embedding.shape[1]:
            return f"{gh * gw} patches exceed the positional table ({self.pos_embedding.shape[1]})"
        return xt.grid_reason(gh, gw)

    def graph_reason(self) -> Optional[str]:
        """None if a CUDA graph of the fused forward replays what the module computes (GraphedForward)."""
        if self.xcit_transformer.layer_dropout > 0 or self.cls_transformer.layer_dropout > 0:
            return ("layer_dropout > 0 draws the layers to run on every call; a CUDA graph would replay the subset of "
                    "the captured call")
        return None

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, img: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(img)                  # b h w d
        b, gh, gw, d = x.shape
        x = x.reshape(b, gh * gw, d)
        x += self.pos_embedding[:, :gh * gw]
        x = x.reshape(b, gh, gw, d)
        x = self.dropout(x)
        x = self.xcit_transformer(x)
        x = self.final_norm(x)
        cls_tokens = self.cls_token.reshape(1, 1, d).expand(b, 1, d)
        x = x.reshape(b, gh * gw, d)
        cls_tokens = self.cls_transformer(cls_tokens, context=x)
        return self.mlp_head(cls_tokens[:, 0])

    # ---------------------------------------------------------------------------------------------- fused kernels
    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        D, dev = self.cls_token.shape[-1], img.device
        pe, eng = patch_engine(self), self.xcit_transformer.engine()
        pos = pe.prepared(dev)["pos"].view(-1, D)
        B, N = pe.geometry(img)
        grid = (img.shape[2] // self.patch_size[0], img.shape[3] // self.patch_size[1])
        xb, stats = eng.entry_buffers(B * N, dev)
        x, B, N = pe.run(img, xb=xb, stats=stats, pos=pos)
        eng.run_blocks(x, B, N, primed=xb is not None, layers=self.xcit_transformer.kept_layers(), grid=grid)
        # final_norm of the patch rows: the context of every class-attention layer
        fn = self.final_norm
        g, bt = cached(self, "_final_norm", list(fn.parameters()), lambda: (_f32(fn.weight), _f32(fn.bias)))
        ctx = torch.empty(B * N, D, device=dev, dtype=torch.bfloat16)
        _lib.layernorm(x, g, bt, out_bf16=ctx, eps=fn.eps)
        cls = self.cls_token.detach().reshape(1, D).float().expand(B, D).contiguous()
        cls_b = torch.empty(B, D, device=dev, dtype=torch.bfloat16)
        self.cls_transformer.cross_engine().run(cls, cls_b, 1, ctx, N, B, cls_row_index(self._rows, B, 1, dev), skip=0,
                                                layers=self.cls_transformer.kept_layers())
        pooled = head_ln_pool(self, self.mlp_head[0], cls, B, 1, mean=False)
        return head_engine(self, self.mlp_head[1]).run(pooled)
