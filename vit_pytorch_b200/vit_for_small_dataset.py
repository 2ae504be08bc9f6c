"""Drop-in `ViT` for lucidrains/vit-pytorch's `vit_pytorch.vit_for_small_dataset.ViT` ("Vision Transformer for
Small-Size Datasets": shifted patch tokenization and locality self-attention), with `SPT`, `LSA`, `Transformer` and
`FeedForward` of the same file, and a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed): `to_patch_embedding.to_patch_tokens.{1,2}`, `pos_embedding` (1, n + 1, dim),
`cls_token` (1, 1, dim), `transformer.layers.i.0.temperature` before `.0.norm`, `mlp_head.{0,1}` (reference
vit_for_small_dataset.py:30-140).  The PyTorch graph below mirrors the reference module for module, so hooks on any
submodule keep working there.

Fused forward (engine.py):
  * SPT: b200vit_patchify_spt_ln gathers the image and its four one-pixel shifts straight into the '(p1 p2 c)' rows
    over 5C channels with LayerNorm(5 C p^2), then the patch GEMM; b200vit_embed_tokens without a LayerNorm adds the cls
    row and the positional table (vit_for_small_dataset.py:92-96,127-132).
  * LSA layers: the encoder layers of vit.py with the softmax scale temperature.exp() of each layer (evaluated in the
    parameter's dtype when the prepared weights are built, so a forward never reads a device value) and each query's
    own key excluded (B200VIT_ATTN_MASK_SELF, vit_for_small_dataset.py:53-57).
  * pool: LayerNorm of mlp_head[0] on the cls rows (row_index), or the mean over all n + 1 tokens and then that
    LayerNorm; then the head GEMM (vit_for_small_dataset.py:134-140).
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from .engine import (EncoderLayer, FusedWeightsMixin, Norm, classify, cls_row_index, common_reason, fused_encode,
                     head_norm, hooked_transformer_tokens, on_device, patch_engine, transformer_is_hooked)
from .vit import FeedForward, FusedTransformer, Patchify, pair

__all__ = ["FeedForward", "LSA", "Transformer", "SPT", "ViT"]

SPT_SHIFTS = ((1, -1, 0, 0), (-1, 1, 0, 0), (0, 0, 1, -1), (0, 0, -1, 1))


class LSA(nn.Module):
    """Locality self-attention: pre-LN multi-head attention with a learned softmax temperature and each token's own key
    masked out (reference vit_for_small_dataset.py:30-64)."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, dropout: float = 0.) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.dim_head = dim_head
        self.temperature = nn.Parameter(torch.log(torch.tensor(dim_head ** -0.5)))
        self.norm = nn.LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, n, _ = x.shape
        x = self.norm(x)
        q, k, v = (t.reshape(b, n, self.heads, -1).transpose(1, 2) for t in self.to_qkv(x).chunk(3, dim=-1))
        dots = torch.matmul(q, k.transpose(-1, -2)) * self.temperature.exp()
        mask = torch.eye(dots.shape[-1], device=dots.device, dtype=torch.bool)
        dots = dots.masked_fill(mask, -torch.finfo(dots.dtype).max)
        attn = self.dropout(self.attend(dots))
        out = torch.matmul(attn, v).transpose(1, 2).reshape(b, n, -1)
        return self.to_out(out)


class Transformer(FusedTransformer):
    """depth x (LSA, FeedForward) residual blocks, no final LayerNorm (reference vit_for_small_dataset.py:66-79).
    Callable on arbitrary (B, N, D) tokens; runs fused when eligible."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.) -> None:
        super().__init__()
        self.dropout_p = float(dropout)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                LSA(dim, heads=heads, dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        layers = []
        for attn, ff in self.layers:
            fc1, fc2 = ff.net[1], ff.net[4]
            out = attn.to_out[0]
            # the eager graph multiplies by temperature.exp() in the parameter's dtype: the same rounded value here.
            # Reading it syncs, which is why this only runs when TransformerEngine.prepared() rebuilds (a parameter
            # version changed), never inside a steady-state forward or a CUDA-graph capture.
            scale = float(attn.temperature.detach().exp())
            layers.append(EncoderLayer(
                ln1=Norm.of(attn.norm), qkv_w=attn.to_qkv.weight, out_w=out.weight, out_b=out.bias,
                ln2=Norm.of(ff.net[0]), fc1_w=fc1.weight, fc1_b=fc1.bias, fc2_w=fc2.weight, fc2_b=fc2.bias,
                heads=attn.heads, dim_head=attn.dim_head, scale=scale, mask_self=True))
        return layers, None


class SPT(nn.Module):
    """Shifted patch tokenization: the image and its four one-pixel shifts, concatenated on the channel axis, cut into
    '(p1 p2 c)' patches, LayerNorm, Linear (reference vit_for_small_dataset.py:81-96)."""

    def __init__(self, *, dim: int, patch_size: int, channels: int = 3) -> None:
        super().__init__()
        patch_dim = patch_size * patch_size * 5 * channels
        self.to_patch_tokens = nn.Sequential(
            Patchify(patch_size, patch_size),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
        )

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        shifted_x = [F.pad(x, shift) for shift in SPT_SHIFTS]
        x_with_shifts = torch.cat((x, *shifted_x), dim=1)
        return self.to_patch_tokens(x_with_shifts)


class ViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, pool='cls', channels=3,
                 dim_head=64, dropout=0., emb_dropout=0.) -> None:
        super().__init__()
        image_height, image_width = pair(image_size)
        self.patch_size = patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, \
            'Image dimensions must be divisible by the patch size.'
        num_patches = (image_height // patch_height) * (image_width // patch_width)
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'

        self.to_patch_embedding = SPT(dim=dim, patch_size=patch_size, channels=channels)
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
        if img.shape[1] * 5 * ph * pw != self.to_patch_embedding.to_patch_tokens[1].normalized_shape[0]:
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
        # b200vit_patchify_spt_ln stages the p + 2 image rows of a patch row (every channel) and its column table
        rs = (img.shape[3] + 16) // 8 * 8
        if 20 * img.shape[1] * ph * ph + img.shape[1] * (ph + 2) * rs * 2 > 200 * 1024:
            return "one row of patches exceeds the SPT kernel's shared-memory slab"
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
    def _pool(self, x: torch.Tensor, B: int, N: int) -> torch.Tensor:
        """x fp32 [B*N, D] encoder output -> mlp_head[0](x[:, 0]) or mlp_head[0](x.mean(1)), bf16 [B, D]."""
        D = x.shape[1]
        dev = x.device
        g, b = head_norm(self, self.mlp_head[0])
        eps = self.mlp_head[0].eps
        pooled = torch.empty(B, D, device=dev, dtype=torch.bfloat16)
        if self.pool == 'mean':
            pm = torch.empty(B, D, device=dev, dtype=torch.float32)
            _lib.mean_pool(x, pm, B, N, D)
            _lib.layernorm(pm, g, b, out_bf16=pooled, eps=eps)
        else:                                          # LayerNorm is per token: normalise only the cls rows
            rows = cls_row_index(self.transformer.engine().rows, B, N, dev)
            _lib.layernorm(x, g, b, out_bf16=pooled, row_index=rows, eps=eps)
        return pooled

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        D = self.cls_token.shape[-1]
        pos = patch_engine(self).prepared(img.device)["pos"].view(-1, D)
        if transformer_is_hooked(self):                # Extractor (reference extractor.py:50-59): hook on .transformer
            x, B, N = patch_engine(self).run(img, pos=pos)
            out = hooked_transformer_tokens(self, x, B, N)
            x = out.reshape(B * N, D).float().contiguous()
        else:
            x, B, N = fused_encode(self, img, pos=pos)  # fp32 residual stream [B*N, D]
        return classify(self, self.mlp_head[1], self._pool(x, B, N))
