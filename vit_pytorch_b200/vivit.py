"""Drop-in `ViViT` for lucidrains/vit-pytorch's `vit_pytorch.vivit.ViViT` (the factorized video transformer, both its
`factorized_encoder` and `factorized_self_attention` variants), with `Transformer`, `FactorizedTransformer` and
`Attention` of the same file, and a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed): `to_patch_embedding[0..3]`, `pos_embedding` (1, F', n, dim), `spatial_cls_token`,
`temporal_cls_token` (None with pool='mean'), `spatial_transformer` / `temporal_transformer` or
`factorized_transformer`, `mlp_head`, `variant`, `global_average_pool` (reference vivit.py:154-219).  The PyTorch graph
below mirrors the reference module for module, so Recorder / Extractor hooks keep working there.

Fused forward (engine.py):
  * patch embedding: the 2-D patch kernels on the (B, C, F' * pf * H, W) view with a (pf * p1, p2) box, as
    simple_vit_3d.py does ('(pf p1 p2 c)' is the 2-D '(p1' p2 c)' order), then b200vit_embed_tokens_grouped assembles
    B*F' sequences: LayerNorm(dim), the positional row of frame f and patch t ((f, t) of the [F'max, n_max] table, the
    reference's pos_embedding[:, :frames, :seq]), and the spatial cls row without a position (vivit.py:224-231).
  * factorized_encoder: spatial blocks over the B*F' sequences -> final LayerNorm of the cls rows (or all rows and the
    mean over the n tokens) -> temporal cls + F' rows per clip -> temporal blocks (with a frame mask: the key-masked
    b200vit_attention_axial, G = 1) -> final LayerNorm -> cls row or mean -> head GEMM (vivit.py:244-272).
  * factorized_self_attention: every layer runs spatial attention over the B*F' sequences of n + 1 tokens and temporal
    attention over the B*(n + 1) strided sequences of F' tokens (b200vit_attention_axial, G = n + 1), then the
    feed-forward block (vivit.py:138-152) -> final LayerNorm -> x[:, 0, 0] or the mean over all F'(n + 1) rows.
  The frame mask is reduced over each frame patch with `all` (and padded for the temporal cls) on the device.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn
from torch.nn.attention import SDPBackend, sdpa_kernel

from . import _lib
from .engine import (AttnBlock, EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, _f32, classify, common_reason,
                     on_device, patch_engine)
from .simple_vit_3d import VideoPatchify
from .vit import FeedForward, FusedTransformer, pair

MAX_AXIAL_LEN = 64          # b200vit_attention_axial: a temporal sequence fits one 64-row tile


class Attention(nn.Module):
    """Pre-LN multi-head attention with an optional key mask, through scaled_dot_product_attention or the explicit
    softmax (reference vivit.py:39-100)."""

    def __init__(self, dim, heads=8, dim_head=64, dropout=0., use_flash_attn=True) -> None:
        super().__init__()
        self.use_flash_attn = use_flash_attn
        self.dropout_p = dropout
        inner_dim = dim_head * heads
        project_out = not (heads == 1 and dim_head == dim)
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.norm = nn.LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout)) if project_out else nn.Identity()

    def flash_attn(self, q, k, v, mask=None):
        with sdpa_kernel([SDPBackend.MATH, SDPBackend.EFFICIENT_ATTENTION, SDPBackend.FLASH_ATTENTION,
                          SDPBackend.CUDNN_ATTENTION]):
            return F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=self.dropout_p, is_causal=False,
                                                  scale=self.scale)

    def forward(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        b, n, _ = x.shape
        x = self.norm(x)
        q, k, v = (t.reshape(b, n, self.heads, -1).transpose(1, 2) for t in self.to_qkv(x).chunk(3, dim=-1))
        if mask is not None:
            mask = mask[:, None, None, :]
        if self.use_flash_attn:
            out = self.flash_attn(q, k, v, mask=mask)
        else:
            dots = torch.matmul(q, k.transpose(-1, -2)) * self.scale
            if mask is not None:
                dots = dots.masked_fill(~mask, -torch.finfo(dots.dtype).max)
            attn = self.dropout(self.attend(dots))
            out = torch.matmul(attn, v)
        return self.to_out(out.transpose(1, 2).reshape(b, n, -1))


def _out_proj(attn: Attention) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """(weight, bias) of to_out, (None, None) when it is the identity (heads == 1 and dim_head == dim)."""
    if isinstance(attn.to_out, nn.Identity):
        return None, None
    return attn.to_out[0].weight, attn.to_out[0].bias


def _encoder_layer(attn: Attention, ff: FeedForward, temporal: Optional[Attention] = None) -> EncoderLayer:
    fc1, fc2 = ff.net[1], ff.net[4]
    out_w, out_b = _out_proj(attn)
    block = None
    if temporal is not None:
        t_w, t_b = _out_proj(temporal)
        block = AttnBlock(ln=Norm.of(temporal.norm), qkv_w=temporal.to_qkv.weight, out_w=t_w, out_b=t_b)
    return EncoderLayer(ln1=Norm.of(attn.norm), qkv_w=attn.to_qkv.weight, out_w=out_w, out_b=out_b,
                        ln2=Norm.of(ff.net[0]), fc1_w=fc1.weight, fc1_b=fc1.bias, fc2_w=fc2.weight, fc2_b=fc2.bias,
                        heads=attn.heads, dim_head=attn.dim_head, scale=float(attn.scale), temporal=block)


def _flash_mode(transformer: nn.Module) -> Optional[bool]:
    """The use_flash_attn flag every Attention of the transformer shares, None if they differ."""
    flags = {m.use_flash_attn for m in transformer.modules() if isinstance(m, Attention)}
    return flags.pop() if len(flags) == 1 else None


def _attention_reason(transformer: nn.Module) -> Optional[str]:
    """Rules of the attention modules the generic dispatch does not know about."""
    flash = _flash_mode(transformer)
    if flash is None:
        return "the attention modules mix use_flash_attn settings"
    if flash and transformer.dropout_p > 0.0:
        # the reference passes dropout_p to scaled_dot_product_attention in eval mode too (vivit.py:65-71)
        return "dropout is active (scaled_dot_product_attention applies dropout_p in eval mode too)"
    return None


def _mask_reason(mask: Optional[torch.Tensor], x: torch.Tensor, shape: Tuple[int, int],
                 check_len: bool = True) -> Optional[str]:
    """None if `mask` (a per-token key mask of the given shape) can go to b200vit_attention_axial; `check_len`: the
    mask's second dim is the sequence length the kernel sees."""
    if mask is None:
        return None
    if mask.dtype != torch.bool:
        return f"mask dtype {mask.dtype} (the reference takes a boolean mask)"
    if tuple(mask.shape) != tuple(shape):
        return f"mask of shape {tuple(mask.shape)}, expected {tuple(shape)}"
    if mask.device != x.device:
        return "mask and input on different devices"
    if check_len and shape[1] > MAX_AXIAL_LEN:
        return f"masked sequences of {shape[1]} tokens (the masked attention kernel takes up to {MAX_AXIAL_LEN})"
    return None


class Transformer(FusedTransformer):
    """depth x (Attention, FeedForward) + final LayerNorm with an optional key mask (reference vivit.py:102-121).
    forward(x, mask) runs fused when eligible: without a mask through the usual attention kernels, with one through
    b200vit_attention_axial over the B sequences (G = 1)."""

    def __init__(self, dim, depth, heads, dim_head, mlp_dim, dropout=0., use_flash_attn=True) -> None:
        super().__init__()
        self.use_flash_attn = use_flash_attn
        self.dropout_p = float(dropout)
        self.norm = nn.LayerNorm(dim)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout, use_flash_attn=use_flash_attn),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        return [_encoder_layer(attn, ff) for attn, ff in self.layers], Norm.of(self.norm)

    def fused_reason(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> Optional[str]:
        r = super().fused_reason(x)
        if r is None:
            r = _attention_reason(self)
        if r is None:
            r = _mask_reason(mask, x, tuple(x.shape[:2]))
        return r

    def forward_eager(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        for attn, ff in self.layers:
            x = attn(x, mask=mask) + x
            x = ff(x) + x
        return self.norm(x)

    def forward(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self.fused_reason(x, mask) is None:
            axial = None if mask is None else (1, x.shape[1], mask.to(torch.uint8).contiguous(),
                                               bool(_flash_mode(self)))
            return self.engine().forward_tokens(x, axial=axial)
        return self.forward_eager(x, mask)


class FactorizedTransformer(FusedEncoder, FusedWeightsMixin, nn.Module):
    """depth x (spatial Attention, temporal Attention, FeedForward) + final LayerNorm over x [b, f, n, d]: attention
    over the n tokens of every frame, then over the f frames of every spatial position, with an optional per-frame
    mask shared by all positions (reference vivit.py:123-152)."""

    def __init__(self, dim, depth, heads, dim_head, mlp_dim, dropout=0., use_flash_attn=True) -> None:
        super().__init__()
        self.use_flash_attn = use_flash_attn
        self.dropout_p = float(dropout)
        self.norm = nn.LayerNorm(dim)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout, use_flash_attn=use_flash_attn),
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout, use_flash_attn=use_flash_attn),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        return [_encoder_layer(sa, ff, temporal=ta) for sa, ta, ff in self.layers], Norm.of(self.norm)

    def fused_reason(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> Optional[str]:
        r = common_reason(self, x, encoders=(self,), dropout_p=self.dropout_p, inside="transformer")
        if r is None and x.dim() != 4:
            r = "input is not (B, F, N, D)"
        if r is None:
            r = _attention_reason(self)
        if r is None and x.shape[1] > MAX_AXIAL_LEN:
            r = f"{x.shape[1]} frames (the temporal attention kernel takes up to {MAX_AXIAL_LEN})"
        if r is None:
            r = _mask_reason(mask, x, tuple(x.shape[:2]))
        if r is None:
            r = self.engine().unsupported_reason(x.shape[2])
        return r

    def forward_eager(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        batch, frames, seq, d = x.shape
        if mask is not None:
            mask = mask.repeat_interleave(seq, dim=0)          # 'b ... -> (b space) ...'
        for spatial_attn, temporal_attn, ff in self.layers:
            x = x.reshape(batch * frames, seq, d)
            x = spatial_attn(x) + x
            x = x.reshape(batch, frames, seq, d).transpose(1, 2).reshape(batch * seq, frames, d)
            x = temporal_attn(x, mask=mask) + x
            x = ff(x) + x
            x = x.reshape(batch, seq, frames, d).transpose(1, 2)
        return self.norm(x)

    def forward(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self.fused_reason(x, mask) is None:
            b, f, n, d = x.shape
            axial = (n, f, None if mask is None else mask.to(torch.uint8).contiguous(), bool(_flash_mode(self)))
            return self.engine().forward_tokens(x.reshape(b * f, n, d), axial=axial).view(b, f, n, d)
        return self.forward_eager(x, mask)


class ViViTPatchify(VideoPatchify):
    """`Rearrange('b c (f pf) (h p1) (w p2) -> b f (h w) (pf p1 p2 c)')` (reference vivit.py:196); parameter-free."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return super().forward(x).flatten(2, 3)


class ViViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, image_patch_size, frames, frame_patch_size, num_classes, dim, spatial_depth,
                 temporal_depth, heads, mlp_dim, pool='cls', channels=3, dim_head=64, dropout=0., emb_dropout=0.,
                 variant='factorized_encoder', use_flash_attn: bool = True) -> None:
        super().__init__()
        image_height, image_width = pair(image_size)
        self.patch_size = patch_height, patch_width = pair(image_patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, \
            'Image dimensions must be divisible by the patch size.'
        assert frames % frame_patch_size == 0, 'Frames must be divisible by frame patch size'
        assert variant in ('factorized_encoder', 'factorized_self_attention'), f'variant = {variant} is not implemented'
        num_image_patches = (image_height // patch_height) * (image_width // patch_width)
        num_frame_patches = frames // frame_patch_size
        patch_dim = channels * patch_height * patch_width * frame_patch_size
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'

        self.frame_patch_size = frame_patch_size
        self.global_average_pool = pool == 'mean'
        self.to_patch_embedding = nn.Sequential(
            ViViTPatchify(frame_patch_size, patch_height, patch_width),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.pos_embedding = nn.Parameter(torch.randn(1, num_frame_patches, num_image_patches, dim))
        self.dropout = nn.Dropout(emb_dropout)
        self.spatial_cls_token = nn.Parameter(torch.randn(1, 1, dim)) if not self.global_average_pool else None
        if variant == 'factorized_encoder':
            self.temporal_cls_token = nn.Parameter(torch.randn(1, 1, dim)) if not self.global_average_pool else None
            self.spatial_transformer = Transformer(dim, spatial_depth, heads, dim_head, mlp_dim, dropout,
                                                   use_flash_attn)
            self.temporal_transformer = Transformer(dim, temporal_depth, heads, dim_head, mlp_dim, dropout,
                                                    use_flash_attn)
        elif variant == 'factorized_self_attention':
            assert spatial_depth == temporal_depth, \
                'Spatial and temporal depth must be the same for factorized self-attention'
            self.factorized_transformer = FactorizedTransformer(dim, spatial_depth, heads, dim_head, mlp_dim, dropout,
                                                                use_flash_attn)
        self.pool = pool
        self.to_latent = nn.Identity()
        self.mlp_head = nn.Linear(dim, num_classes)
        self.variant = variant

        self._emb_dropout_p = float(emb_dropout)
        # the 2-D patch kernels see the video as (B, C, F' * pf * H, W) cut into (pf * p1, p2) boxes
        self.fused_patch_box: Tuple[int, int] = (frame_patch_size * patch_height, patch_width)

    def _transformers(self) -> List[nn.Module]:
        if self.variant == 'factorized_encoder':
            return [self.spatial_transformer, self.temporal_transformer]
        return [self.factorized_transformer]

    # ---------------------------------------------------------------------------------------------- dispatch
    def fused_reason(self, video: torch.Tensor, mask: Optional[torch.Tensor] = None) -> Optional[str]:
        """None if forward(video, mask) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if video.dim() != 5:
            return "input is not (B, C, F, H, W)"
        pf, (p1, p2) = self.frame_patch_size, self.patch_size
        if video.shape[1] * pf * p1 * p2 != self.to_patch_embedding[1].normalized_shape[0]:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        if video.shape[2] % pf or video.shape[3] % p1 or video.shape[4] % p2:
            return "video not divisible by the patch box"
        f, n = video.shape[2] // pf, (video.shape[3] // p1) * (video.shape[4] // p2)
        if f == 0 or n == 0:
            return "empty patch grid"
        if f > self.pos_embedding.shape[1] or n > self.pos_embedding.shape[2]:
            return (f"{f} frame patches x {n} patches exceed the positional table "
                    f"({self.pos_embedding.shape[1]} x {self.pos_embedding.shape[2]})")
        r = common_reason(self, video, encoders=self._transformers(),
                          dropout_p=max([self._emb_dropout_p] + [t.dropout_p for t in self._transformers()]),
                          skip=(self.to_latent,))
        for t in self._transformers():
            r = r or _attention_reason(t)
        if r is not None:
            return r
        ncls = 0 if self.global_average_pool else 1
        L = f + ncls if self.variant == 'factorized_encoder' else f
        if mask is not None:
            r = _mask_reason(mask, video, (video.shape[0], video.shape[2]), check_len=False)
            if r is None and L > MAX_AXIAL_LEN:
                r = f"masked temporal sequences of {L} tokens (the masked attention kernel takes up to {MAX_AXIAL_LEN})"
        if r is None and self.variant == 'factorized_self_attention' and L > MAX_AXIAL_LEN:
            r = f"{L} frame patches (the temporal attention kernel takes up to {MAX_AXIAL_LEN})"
        if r is None and self.fused_patch_box[0] * video.shape[4] * video.shape[1] * 2 > 200 * 1024:
            r = "one row of patch boxes exceeds the patch kernel's shared-memory slab"
        for t, N in zip(self._transformers(), (n + ncls, L)):
            r = r or t.engine().unsupported_reason(N)
        return r

    def forward(self, video: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self.fused_reason(video, mask) is None:
            with on_device(video):
                return self.forward_fused(video, mask)
        return self.forward_eager(video, mask)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, video: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        x = self.to_patch_embedding(video)
        batch, frames, seq, _ = x.shape
        x = x + self.pos_embedding[:, :frames, :seq]
        if self.spatial_cls_token is not None:
            spatial_cls_tokens = self.spatial_cls_token[None].expand(batch, frames, -1, -1)
            x = torch.cat((spatial_cls_tokens, x), dim=2)
        x = self.dropout(x)
        temporal_mask = None
        if mask is not None:
            temporal_mask = mask.reshape(mask.shape[0], -1, self.frame_patch_size).all(dim=-1)
        if self.variant == 'factorized_encoder':
            x = x.reshape(batch * frames, *x.shape[2:])
            x = self.spatial_transformer(x)
            x = x.reshape(batch, frames, *x.shape[1:])
            x = x[:, :, 0] if not self.global_average_pool else x.mean(dim=2)
            if self.temporal_cls_token is not None:
                temporal_cls_tokens = self.temporal_cls_token.expand(batch, -1, -1)
                x = torch.cat((temporal_cls_tokens, x), dim=1)
                if temporal_mask is not None:
                    temporal_mask = F.pad(temporal_mask, (1, 0), value=True)
            x = self.temporal_transformer(x, mask=temporal_mask)
            x = x[:, 0] if not self.global_average_pool else x.mean(dim=1)
        else:
            x = self.factorized_transformer(x, mask=temporal_mask)
            x = x[:, 0, 0] if not self.global_average_pool else x.mean(dim=(1, 2))
        x = self.to_latent(x)
        return self.mlp_head(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def forward_fused(self, video: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        b, c, ft, ht, wt = video.shape
        pf, (p1, p2) = self.frame_patch_size, self.patch_size
        f, n = ft // pf, (ht // p1) * (wt // p2)
        dev = video.device
        if pf == 1:
            img = video.contiguous().view(b, c, ft * ht, wt)
        else:
            # (f pf) (h p1) -> (f h pf p1): the pf frames of one box under each other; token order (f h w) unchanged
            img = video.reshape(b, c, f, pf, ht // p1, p1, wt).permute(0, 1, 2, 4, 3, 5, 6).reshape(b, c, ft * ht, wt)
        cls = not self.global_average_pool
        ncls = 1 if cls else 0
        N = n + ncls
        fe = self.variant == 'factorized_encoder'
        eng = (self.spatial_transformer if fe else self.factorized_transformer).engine()
        pe = patch_engine(self)
        y = pe.project(img, patch=self.fused_patch_box)            # [b*f*n, D], patches in (b, f, h, w) order
        t = pe.prepared(dev)
        D = y.shape[1]
        xb, stats = eng.entry_buffers(b * f * N, dev)
        x = torch.empty(b * f * N, D, device=dev, dtype=torch.float32)
        _lib.embed_tokens_grouped(y, t["ln2.w"], t["ln2.b"], _f32(self.spatial_cls_token.reshape(1, D)) if cls else None,
                                  t["pos"].view(-1, D), x, b * f, n, ncls, pos_period=f,
                                  pos_stride=self.pos_embedding.shape[2], cls_pos=False,
                                  eps=self.to_patch_embedding[3].eps, xb=xb, stats=stats)
        key_mask = None if mask is None else mask.reshape(b, f, pf).all(dim=-1)
        if fe:
            eng.run_blocks(x, b * f, N, primed=xb is not None)
            xs = eng.pool(x, b * f, N, mean=not cls, dtype=torch.float32)
            tr = self.temporal_transformer
            if cls:
                xt = torch.cat((self.temporal_cls_token.detach().float().expand(b, 1, D), xs.view(b, f, D)), dim=1)
                xt = xt.reshape(b * (f + 1), D)
                if key_mask is not None:
                    key_mask = F.pad(key_mask, (1, 0), value=True)
            else:
                xt = xs
            Lt = f + ncls
            axial = None if key_mask is None else (1, Lt, key_mask.to(torch.uint8).contiguous(),
                                                   bool(_flash_mode(tr)))
            teng = tr.engine()
            teng.run_blocks(xt, b, Lt, axial=axial)
            pooled = teng.pool(xt, b, Lt, mean=not cls)
        else:
            tr = self.factorized_transformer
            axial = (N, f, None if key_mask is None else key_mask.to(torch.uint8).contiguous(),
                     bool(_flash_mode(tr)))
            eng.run_blocks(x, b * f, N, primed=xb is not None, axial=axial)
            pooled = eng.pool(x, b, f * N, mean=not cls)
        return classify(self, self.mlp_head, pooled)
