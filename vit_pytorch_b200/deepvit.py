"""Drop-in `DeepViT` for lucidrains/vit-pytorch's `vit_pytorch.deepvit.DeepViT` (re-attention), with `Transformer`,
`Attention` and `FeedForward` of the same file, and a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed): `transformer.layers.i.0.reattn_weights` before `.0.norm`, `.0.reattn_norm.1` (the
LayerNorm over heads), `pos_embedding` (1, n + 1, dim), `cls_token` (1, 1, dim), `mlp_head.{0,1}` (reference
deepvit.py:22-129).  The PyTorch graph below mirrors the reference module for module, so hooks on any submodule keep
working there.

Fused forward (engine.py):
  * patch embedding and token assembly as vit.py (Rearrange, LayerNorm, Linear, LayerNorm, cls row, positional table);
  * encoder layers: vit.py's schedule with b200vit_attention_headmix in place of the attention kernel: softmax, then
    the probabilities mixed across heads by reattn_weights and a LayerNorm over the heads of every (query, key) pair,
    all in one kernel (deepvit.py:54-67); the Transformer has no final LayerNorm;
  * pool: LayerNorm of mlp_head[0] on the cls rows, or the mean over all n + 1 tokens and then that LayerNorm; then the
    head GEMM (deepvit.py:117-129).
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import nn

from .engine import (EncoderLayer, FusedWeightsMixin, HeadMix, Norm, classify, common_reason, fused_encode,
                     head_ln_pool, hooked_transformer_tokens, on_device, patch_engine, transformer_is_hooked)
from .vit import FeedForward, FusedTransformer, Patchify

__all__ = ["Attention", "DeepViT", "FeedForward", "Transformer"]


class _HeadsLast(nn.Module):
    """'b h i j -> b i j h' (the first Rearrange of reattn_norm, deepvit.py:37-41)."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x.permute(0, 2, 3, 1)


class _HeadsFirst(nn.Module):
    """'b i j h -> b h i j'."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x.permute(0, 3, 1, 2)


class Attention(nn.Module):
    """Pre-LN multi-head attention with re-attention: the softmax probabilities are mixed across heads by the learned
    [heads, heads] matrix reattn_weights, then LayerNorm'ed over the heads (reference deepvit.py:22-67)."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, dropout: float = 0.) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.norm = nn.LayerNorm(dim)
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        self.dropout = nn.Dropout(dropout)
        self.reattn_weights = nn.Parameter(torch.randn(heads, heads))
        self.reattn_norm = nn.Sequential(_HeadsLast(), nn.LayerNorm(heads), _HeadsFirst())
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, n, _ = x.shape
        x = self.norm(x)
        q, k, v = (t.reshape(b, n, self.heads, -1).transpose(1, 2) for t in self.to_qkv(x).chunk(3, dim=-1))
        dots = torch.einsum('b h i d, b h j d -> b h i j', q, k) * self.scale
        attn = dots.softmax(dim=-1)
        attn = self.dropout(attn)
        attn = torch.einsum('b h i j, h g -> b g i j', attn, self.reattn_weights)
        attn = self.reattn_norm(attn)
        out = torch.einsum('b h i j, b h j d -> b h i d', attn, v)
        out = out.transpose(1, 2).reshape(b, n, -1)
        return self.to_out(out)


class Transformer(FusedTransformer):
    """depth x (re-attention, feed-forward) residual blocks, no final LayerNorm (reference deepvit.py:69-82).
    Callable on arbitrary (B, N, D) tokens; runs fused when eligible."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.) -> None:
        super().__init__()
        self.dropout_p = float(dropout)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        layers = []
        for attn, ff in self.layers:
            fc1, fc2 = ff.net[1], ff.net[4]
            out = attn.to_out[0]
            layers.append(EncoderLayer(
                ln1=Norm.of(attn.norm), qkv_w=attn.to_qkv.weight, out_w=out.weight, out_b=out.bias,
                ln2=Norm.of(ff.net[0]), fc1_w=fc1.weight, fc1_b=fc1.bias, fc2_w=fc2.weight, fc2_b=fc2.bias,
                heads=attn.heads, dim_head=attn.dim_head, scale=float(attn.scale),
                attention=HeadMix(post=attn.reattn_weights, ln=Norm.of(attn.reattn_norm[1]))))
        return layers, None


class DeepViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, pool='cls', channels=3,
                 dim_head=64, dropout=0., emb_dropout=0.) -> None:
        super().__init__()
        assert image_size % patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        num_patches = (image_size // patch_size) ** 2
        patch_dim = channels * patch_size ** 2
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        self.patch_size = (patch_size, patch_size)

        self.to_patch_embedding = nn.Sequential(
            Patchify(patch_size, patch_size),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.pos_embedding = nn.Parameter(torch.randn(1, num_patches + 1, dim))
        self.cls_token = nn.Parameter(torch.randn(1, 1, dim))
        self.dropout = nn.Dropout(emb_dropout)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim, dropout)
        self.pool = pool
        self.to_latent = nn.Identity()
        self.mlp_head = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, num_classes))

        self._emb_dropout_p = float(emb_dropout)

    # ---------------------------------------------------------------------------------------------- dispatch
    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        ph, pw = self.patch_size
        if img.shape[1] * ph * pw != self.to_patch_embedding[1].normalized_shape[0]:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        r = common_reason(self, img, encoders=(self.transformer,),
                          dropout_p=max(self._emb_dropout_p, self.transformer.dropout_p),
                          skip=(self.to_latent, self.transformer))
        if r is not None:
            return r
        if img.shape[2] % ph or img.shape[3] % pw:
            return "image not divisible by the patch size"
        n = (img.shape[2] // ph) * (img.shape[3] // pw)
        if n + 1 > self.pos_embedding.shape[1]:
            return f"{n + 1} tokens exceed the positional table ({self.pos_embedding.shape[1]})"
        return self.transformer.engine().unsupported_reason(n + 1)

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
        x += self.pos_embedding[:, :(n + 1)]
        x = self.dropout(x)
        x = self.transformer(x)
        x = x.mean(dim=1) if self.pool == 'mean' else x[:, 0]
        x = self.to_latent(x)
        return self.mlp_head(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        D = self.cls_token.shape[-1]
        pos = patch_engine(self).prepared(img.device)["pos"].view(-1, D)
        if transformer_is_hooked(self):                # Extractor (reference extractor.py:50-59): hook on .transformer
            x, B, N = patch_engine(self).run(img, pos=pos)
            out = hooked_transformer_tokens(self, x, B, N)
            x = out.reshape(B * N, D).float().contiguous()
        else:
            x, B, N = fused_encode(self, img, pos=pos)  # fp32 residual stream [B*N, D]
        pooled = head_ln_pool(self, self.mlp_head[0], x, B, N, mean=self.pool == 'mean')
        return classify(self, self.mlp_head[1], pooled)
