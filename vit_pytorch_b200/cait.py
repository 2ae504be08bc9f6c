"""Drop-in `CaiT` for lucidrains/vit-pytorch's `vit_pytorch.cait.CaiT` (class-attention image transformer with talking
heads and LayerScale), with `Transformer`, `Attention`, `FeedForward`, `LayerScale` and `dropout_layers` of the same
file, and a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed): `patch_transformer.layers.i.{0,1}.{scale, fn}` (LayerScale's `scale` before `fn`),
`Attention` = `norm`, `to_q`, `to_kv`, `mix_heads_pre_attn`, `mix_heads_post_attn`, `to_out`, `pos_embedding`
(1, num_patches, dim) without a cls row, `cls_token` (1, 1, dim), `mlp_head.{0,1}` (reference cait.py:31-178).  The
PyTorch graph below mirrors the reference module for module, so hooks on any submodule keep working there.

Fused forward (engine.py):
  * patch embedding as vit.py (Rearrange, LayerNorm, Linear, LayerNorm) plus the positional table, no cls row
    (cait.py:167-171);
  * patch_transformer: the layers `dropout_layers` keeps, vit.py's schedule with b200vit_attention_headmix_ex (scores
    mixed across heads before the softmax, probabilities after it) and LayerScale folded into the to_out and fc2
    weights; no final LayerNorm (cait.py:105-122);
  * cls_transformer (cait.py:175-176): one stacked to_kv GEMM of all class-attention layers over the patch rows, then
    per kept layer LayerNorm of the cls rows, [to_q; to_kv] GEMM, b200vit_attention_cls_headmix, to_out GEMM with the
    residual, LayerNorm, fc1 GEMM + GELU, fc2 GEMM with the residual (CrossAttentionEngine);
  * head: LayerNorm of mlp_head[0] on the cls rows, then the head GEMM (cait.py:178).
Layer dropout (cait.py:14-27) draws its subset on every call, in eval too, from the same CPU generator in the same order
as the reference: the patch transformer first, then the cls transformer.  The fused path draws through the same
`dropout_layers`, so under one seed the reference, the PyTorch graph and the fused kernels run the same layers.
"""
from __future__ import annotations

from random import randrange
from typing import List, Optional, Sequence, Tuple

import torch
from torch import nn

from .engine import (CrossAttentionEngine, CrossLayer, EncoderLayer, FeedForwardBlock, FusedWeightsMixin, HeadMix, Norm,
                     cls_row_index, common_reason, head_engine, head_ln_pool, headmix_reason, on_device, patch_engine)
from .vit import FeedForward, FusedTransformer, Patchify

__all__ = ["Attention", "CaiT", "FeedForward", "LayerScale", "Transformer", "dropout_layers"]


def dropout_layers(layers: Sequence, dropout: float) -> list:
    """The layers kept by layer dropout (reference cait.py:14-27): each dropped with probability `dropout`, drawn on
    the CPU generator; if all would be dropped, one (random.randrange) is kept."""
    if dropout == 0:
        return layers
    num_layers = len(layers)
    to_drop = torch.zeros(num_layers).uniform_(0., 1.) < dropout
    if all(to_drop):
        rand_index = randrange(num_layers)
        to_drop[rand_index] = False
    return [layer for (layer, drop) in zip(layers, to_drop) if not drop]


class LayerScale(nn.Module):
    """fn(x) times a learned [1, 1, dim] vector whose initial value depends on the layer's depth (reference
    cait.py:31-45)."""

    def __init__(self, dim: int, fn: nn.Module, depth: int) -> None:
        super().__init__()
        if depth <= 18:
            init_eps = 0.1
        elif depth <= 24:
            init_eps = 1e-5
        else:
            init_eps = 1e-6
        self.scale = nn.Parameter(torch.zeros(1, 1, dim).fill_(init_eps))
        self.fn = fn

    def forward(self, x: torch.Tensor, **kwargs) -> torch.Tensor:
        return self.fn(x, **kwargs) * self.scale


class Attention(nn.Module):
    """Pre-LN attention with talking heads: the scores mixed across heads before the softmax, the probabilities after
    it; with `context`, the keys and values come from [LN(x); context] (reference cait.py:61-103)."""

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
        self.mix_heads_pre_attn = nn.Parameter(torch.randn(heads, heads))
        self.mix_heads_post_attn = nn.Parameter(torch.randn(heads, heads))
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout))

    def forward(self, x: torch.Tensor, context: Optional[torch.Tensor] = None) -> torch.Tensor:
        b, n, _ = x.shape
        h = self.heads
        x = self.norm(x)
        context = x if context is None else torch.cat((x, context), dim=1)
        k, v = self.to_kv(context).chunk(2, dim=-1)
        q, k, v = (t.reshape(b, t.shape[1], h, -1).transpose(1, 2) for t in (self.to_q(x), k, v))
        dots = torch.einsum('b h i d, b h j d -> b h i j', q, k) * self.scale
        dots = torch.einsum('b h i j, h g -> b g i j', dots, self.mix_heads_pre_attn)
        attn = self.dropout(self.attend(dots))
        attn = torch.einsum('b h i j, h g -> b g i j', attn, self.mix_heads_post_attn)
        out = torch.einsum('b h i j, b h j d -> b h i d', attn, v)
        out = out.transpose(1, 2).reshape(b, n, -1)
        return self.to_out(out)


class Transformer(FusedTransformer):
    """depth x (LayerScale(Attention), LayerScale(FeedForward)) residual blocks with layer dropout, no final LayerNorm
    (reference cait.py:105-122).  Callable on (B, N, D) tokens, optionally with a context; without one it runs fused
    when eligible."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.,
                 layer_dropout: float = 0.) -> None:
        super().__init__()
        self.layers = nn.ModuleList([])
        self.layer_dropout = layer_dropout
        self.dropout_p = float(dropout)
        for ind in range(depth):
            self.layers.append(nn.ModuleList([
                LayerScale(dim, Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout), depth=ind + 1),
                LayerScale(dim, FeedForward(dim, mlp_dim, dropout=dropout), depth=ind + 1),
            ]))

    def forward_eager(self, x: torch.Tensor, context: Optional[torch.Tensor] = None) -> torch.Tensor:
        for attn, ff in dropout_layers(self.layers, dropout=self.layer_dropout):
            x = attn(x, context=context) + x
            x = ff(x) + x
        return x

    def forward(self, x: torch.Tensor, context: Optional[torch.Tensor] = None) -> torch.Tensor:
        if context is None and self.fused_reason(x) is None:
            return self.engine().forward_tokens(x, layers=self.kept_layers())
        return self.forward_eager(x, context)

    def kept_layers(self) -> List[int]:
        """The indices of the layers this call runs: dropout_layers over the layer indices, which draws exactly what
        the PyTorch graph's call on the layers draws."""
        return list(dropout_layers(list(range(len(self.layers))), dropout=self.layer_dropout))

    # ---------------------------------------------------------------------------------------------- fused kernels
    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        layers = []
        for ls_attn, ls_ff in self.layers:
            attn, ff = ls_attn.fn, ls_ff.fn
            fc1, fc2, out = ff.net[1], ff.net[4], attn.to_out[0]
            layers.append(EncoderLayer(
                ln1=Norm.of(attn.norm), qkv_w=torch.cat([attn.to_q.weight, attn.to_kv.weight]),
                out_w=out.weight, out_b=out.bias,
                ln2=Norm.of(ff.net[0]), fc1_w=fc1.weight, fc1_b=fc1.bias, fc2_w=fc2.weight, fc2_b=fc2.bias,
                heads=attn.heads, dim_head=attn.dim_head, scale=float(attn.scale),
                attention=HeadMix(post=attn.mix_heads_post_attn, ln=None, pre=attn.mix_heads_pre_attn),
                out_scale=ls_attn.scale, ff_scale=ls_ff.scale))
        return layers, None

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
                pre=attn.mix_heads_pre_attn, post=attn.mix_heads_post_attn, out_scale=ls_attn.scale,
                ff=FeedForwardBlock(Norm.of(ff.net[0]), ff.net[1].weight, ff.net[1].bias, ff.net[4].weight,
                                    ff.net[4].bias),
                ff_scale=ls_ff.scale))
        return out

    def cross_engine(self) -> CrossAttentionEngine:
        eng = self.__dict__.get("_cross_engine")
        if eng is None:
            eng = self._cross_engine = CrossAttentionEngine(self, 0)
        return eng


class CaiT(FusedWeightsMixin, nn.Module):
    # the cls token is not part of the patch sequence: it joins in the class-attention stage
    cls_in_sequence = False

    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, cls_depth, heads, mlp_dim, dim_head=64,
                 dropout=0., emb_dropout=0., layer_dropout=0.) -> None:
        super().__init__()
        assert image_size % patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        num_patches = (image_size // patch_size) ** 2
        patch_dim = 3 * patch_size ** 2
        self.patch_size = (patch_size, patch_size)

        self.to_patch_embedding = nn.Sequential(
            Patchify(patch_size, patch_size),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.pos_embedding = nn.Parameter(torch.randn(1, num_patches, dim))
        self.cls_token = nn.Parameter(torch.randn(1, 1, dim))
        self.dropout = nn.Dropout(emb_dropout)
        self.patch_transformer = Transformer(dim, depth, heads, dim_head, mlp_dim, dropout, layer_dropout)
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
        pt, ct = self.patch_transformer, self.cls_transformer
        r = common_reason(self, img, encoders=(pt, ct),
                          dropout_p=max(self._emb_dropout_p, pt.dropout_p, ct.dropout_p))
        if r is not None:
            return r
        if img.shape[2] % ph or img.shape[3] % pw:
            return "image not divisible by the patch size"
        n = (img.shape[2] // ph) * (img.shape[3] // pw)
        if n > self.pos_embedding.shape[1]:
            return f"{n} patches exceed the positional table ({self.pos_embedding.shape[1]})"
        r = pt.engine().unsupported_reason(n)
        if r is None:
            a = ct.layers[0][0].fn
            r = headmix_reason(a.heads, a.dim_head)
        return r

    def graph_reason(self) -> Optional[str]:
        """None if a CUDA graph of the fused forward replays what the module computes (GraphedForward)."""
        if self.patch_transformer.layer_dropout > 0 or self.cls_transformer.layer_dropout > 0:
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
        x = self.to_patch_embedding(img)
        b, n, _ = x.shape
        x += self.pos_embedding[:, :n]
        x = self.dropout(x)
        x = self.patch_transformer(x)
        cls_tokens = self.cls_token.expand(b, -1, -1)
        x = self.cls_transformer(cls_tokens, context=x)
        return self.mlp_head(x[:, 0])

    # ---------------------------------------------------------------------------------------------- fused kernels
    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        D, dev = self.cls_token.shape[-1], img.device
        pe, eng = patch_engine(self), self.patch_transformer.engine()
        pos = pe.prepared(dev)["pos"].view(-1, D)
        B, N = pe.geometry(img)
        xb, stats = eng.entry_buffers(B * N, dev)
        x, B, N = pe.run(img, xb=xb, stats=stats, pos=pos)
        eng.run_blocks(x, B, N, primed=xb is not None, layers=self.patch_transformer.kept_layers())
        ctx = eng.stream_bf16(x)                      # the patch rows: the context of every class-attention layer
        cls = self.cls_token.detach().reshape(1, D).float().expand(B, D).contiguous()
        cls_b = torch.empty(B, D, device=dev, dtype=torch.bfloat16)
        self.cls_transformer.cross_engine().run(cls, cls_b, 1, ctx, N, B, cls_row_index(self._rows, B, 1, dev), skip=0,
                                                layers=self.cls_transformer.kept_layers())
        pooled = head_ln_pool(self, self.mlp_head[0], cls, B, 1, mean=False)
        return head_engine(self, self.mlp_head[1]).run(pooled)
