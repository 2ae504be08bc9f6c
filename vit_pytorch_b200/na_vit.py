"""Drop-in `NaViT` for `vit_pytorch.na_vit.NaViT` (reference na_vit.py:195-402): host-side mirror.

Same constructor keywords, parameter / buffer names, shapes and registration order (bias-free `LayerNorm` with a
`gamma` parameter and a zero `beta` buffer, per-head q/k `RMSNorm`, factorised height / width positional tables,
attention pooling with one learned query, bias-free head), same `forward(List[Tensor] | List[List[Tensor]],
group_images=False, group_max_seq_len=2048) -> (num_images, num_classes)` and the same greedy packing helper.

Two executions of the same arithmetic:
  * PyTorch graph (CPU, fp32, training, autograd, hooks): packed rows + a boolean mask built from per-token image ids,
    like the reference.
  * fused sm_90a path (CUDA bf16, eval, no autograd): images never interact, so the packing and the O(B L^2) mask are
    dropped altogether -- all tokens of all images form ONE padding-free [T, D] matrix described by cu_seqlens, the
    encoder GEMMs run on it unchanged, attention is the varlen block-diagonal kernel (`b200vit_attention_varlen`,
    pipelined 64-key blocks, any image size), the q/k RMSNorm is an epilogue of the QKV GEMM and the attention pooling
    its own small kernel.  Patch extraction ('c (h p1) (w p2) -> (h w) (c p1 p2)' per image, na_vit.py:300) + the
    first LayerNorm is one kernel over the whole list of images (`b200vit_patchify_varlen_ln`), the positional rows
    are gathered by `b200vit_embed_varlen`; the host only builds the small index arrays (`_lib.VarlenIndex`).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from . import _lib
from .engine import (EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, _bf16_rows, _f32, cached, head_width_reason,
                     hooks_inside, on_device, why_not_fused)


def group_images_by_max_seq_len(images: Sequence[Tensor], patch_size: int,
                                calc_token_dropout: Union[None, float, Callable] = None,
                                max_seq_len: int = 2048) -> List[List[Tensor]]:
    """Greedy packing in arrival order: open a new row when the next image does not fit (reference na_vit.py:38-77)."""
    if calc_token_dropout is None:
        drop = lambda h, w: 0.0
    elif isinstance(calc_token_dropout, (float, int)):
        drop = lambda h, w, v=float(calc_token_dropout): v
    else:
        drop = calc_token_dropout
    rows: List[List[Tensor]] = []
    row: List[Tensor] = []
    used = 0
    for image in images:
        assert isinstance(image, Tensor)
        h, w = image.shape[-2:]
        n = int((h // patch_size) * (w // patch_size) * (1 - drop(h, w)))
        assert n <= max_seq_len, f'image with dimensions {(h, w)} exceeds maximum sequence length'
        if used + n > max_seq_len:
            rows.append(row)
            row, used = [], 0
        row.append(image)
        used += n
    if row:
        rows.append(row)
    return rows


class LayerNorm(nn.Module):
    """LayerNorm with learned scale and no learned shift (reference na_vit.py:82-89)."""

    def __init__(self, dim: int) -> None:
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(dim))
        self.register_buffer('beta', torch.zeros(dim))

    def forward(self, x: Tensor) -> Tensor:
        return F.layer_norm(x, x.shape[-1:], self.gamma, self.beta)


class RMSNorm(nn.Module):
    """Per-head query/key normalisation: unit L2 norm * sqrt(dim) * gamma[h, 1, d] (reference na_vit.py:93-101)."""

    def __init__(self, heads: int, dim: int) -> None:
        super().__init__()
        self.scale = dim ** 0.5
        self.gamma = nn.Parameter(torch.ones(heads, 1, dim))

    def forward(self, x: Tensor) -> Tensor:
        return F.normalize(x, dim=-1) * self.scale * self.gamma


def FeedForward(dim: int, hidden_dim: int, dropout: float = 0.) -> nn.Sequential:
    return nn.Sequential(LayerNorm(dim), nn.Linear(dim, hidden_dim), nn.GELU(), nn.Dropout(dropout),
                         nn.Linear(hidden_dim, dim), nn.Dropout(dropout))


class Attention(nn.Module):
    """Self / cross attention with q/k RMSNorm and softmax scale 1 (reference na_vit.py:115-169)."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, dropout: float = 0.) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.norm = LayerNorm(dim)
        self.q_norm = RMSNorm(heads, dim_head)
        self.k_norm = RMSNorm(heads, dim_head)
        self.dropout_p = dropout
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim, inner_dim * 2, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim, bias=False), nn.Dropout(dropout))

    def forward(self, x: Tensor, context: Optional[Tensor] = None, mask: Optional[Tensor] = None,
                attn_mask: Optional[Tensor] = None) -> Tensor:
        x = self.norm(x)
        src = x if context is None else context
        b, n, _ = x.shape
        h = self.heads
        q = self.to_q(x).reshape(b, n, h, -1).transpose(1, 2)
        kv = self.to_kv(src).reshape(b, src.shape[1], 2, h, -1).permute(2, 0, 3, 1, 4)
        q, k, v = self.q_norm(q), self.k_norm(kv[0]), kv[1]
        if mask is not None:
            key_mask = mask[:, None, None, :]
            attn_mask = key_mask if attn_mask is None else (attn_mask & key_mask)
        out = F.scaled_dot_product_attention(q, k, v, attn_mask=attn_mask,
                                             dropout_p=self.dropout_p if self.training else 0., scale=1.)
        return self.to_out(out.transpose(1, 2).reshape(b, n, -1))


def _norm(ln: LayerNorm) -> Norm:
    """beta = None: the fused path assumes the zero `beta` buffer the reference registers (NaViT._nonzero_beta checks
    it); eps is that of F.layer_norm, which LayerNorm.forward uses."""
    return Norm(ln.gamma, None, 1e-5)


class Transformer(FusedEncoder, nn.Module):
    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.) -> None:
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))
        self.norm = LayerNorm(dim)

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Norm]:
        layers = []
        for attn, ff in self.layers:
            layers.append(EncoderLayer(
                ln1=_norm(attn.norm), qkv_w=torch.cat([attn.to_q.weight, attn.to_kv.weight], dim=0),
                out_w=attn.to_out[0].weight, out_b=attn.to_out[0].bias,
                ln2=_norm(ff[0]), fc1_w=ff[1].weight, fc1_b=ff[1].bias, fc2_w=ff[4].weight, fc2_b=ff[4].bias,
                heads=attn.heads, dim_head=attn.to_q.weight.shape[0] // attn.heads, scale=1.0,
                qk_norm="rms", qk_gamma=(attn.q_norm.gamma, attn.k_norm.gamma)))
        return layers, _norm(self.norm)

    def forward(self, x: Tensor, mask: Optional[Tensor] = None, attn_mask: Optional[Tensor] = None) -> Tensor:
        for attn, ff in self.layers:
            x = attn(x, mask=mask, attn_mask=attn_mask) + x
            x = ff(x) + x
        return self.norm(x)


class NaViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, channels=3, dim_head=64,
                 dropout=0., emb_dropout=0., token_dropout_prob=None) -> None:
        super().__init__()
        image_height, image_width = image_size if isinstance(image_size, tuple) else (image_size, image_size)
        self.calc_token_dropout = None
        if callable(token_dropout_prob):
            self.calc_token_dropout = token_dropout_prob
        elif isinstance(token_dropout_prob, (float, int)):
            assert 0. <= token_dropout_prob < 1.
            token_dropout_prob = float(token_dropout_prob)
            self.calc_token_dropout = lambda height, width: token_dropout_prob
        assert image_height % patch_size == 0 and image_width % patch_size == 0, \
            'Image dimensions must be divisible by the patch size.'
        patch_dim = channels * (patch_size ** 2)
        self.channels = channels
        self.patch_size = patch_size
        self.to_patch_embedding = nn.Sequential(LayerNorm(patch_dim), nn.Linear(patch_dim, dim), LayerNorm(dim))
        self.pos_embed_height = nn.Parameter(torch.randn(image_height // patch_size, dim))
        self.pos_embed_width = nn.Parameter(torch.randn(image_width // patch_size, dim))
        self.dropout = nn.Dropout(emb_dropout)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim, dropout)
        self.attn_pool_queries = nn.Parameter(torch.randn(dim))
        self.attn_pool = Attention(dim=dim, dim_head=dim_head, heads=heads)
        self.to_latent = nn.Identity()
        self.mlp_head = nn.Sequential(LayerNorm(dim), nn.Linear(dim, num_classes, bias=False))

    @property
    def device(self):
        return next(self.parameters()).device

    # ------------------------------------------------------------------------------------------------------------
    # fused sm_90a path
    # ------------------------------------------------------------------------------------------------------------
    def fused_reason(self, batched_images=None) -> Optional[str]:
        """None if forward(batched_images) runs the hand-written kernels, else the reason for the PyTorch graph."""
        if batched_images is None:
            return "no input given"
        first = batched_images[0] if torch.is_tensor(batched_images[0]) else batched_images[0][0]
        attn0 = self.transformer.layers[0][0] if len(self.transformer.layers) else None
        if attn0 is None:
            return "depth == 0"
        p_drop = max(self.dropout.p, attn0.dropout_p)
        r = why_not_fused(list(self.parameters()), first, training=self.training, dropout_p=p_drop)
        if r is None:
            flat = batched_images if torch.is_tensor(batched_images[0]) else [im for row in batched_images for im in row]
            for im in flat:
                if not (torch.is_tensor(im) and im.is_cuda and im.device == first.device and im.dtype == first.dtype):
                    r = "images differ in device or dtype"
                    break
                if torch.is_grad_enabled() and im.requires_grad:
                    r = "autograd is recording (fused path is forward only)"
                    break
        if r is None and self._nonzero_beta():
            r = "a LayerNorm `beta` buffer is non-zero (the fused path folds beta = 0, as the reference registers it)"
        if r is None and self.training and self.calc_token_dropout is not None:
            r = "token dropout is active"
        if r is None and hooks_inside(self, skip=(self.to_latent,)):
            r = "forward hooks registered inside the model"
        if r is None:
            r = head_width_reason(attn0.to_q.weight.shape[0] // attn0.heads)
        if r is None and (self.pos_embed_height.shape[1] % 8 or (self.channels * self.patch_size ** 2) % 8):
            r = "dim / patch_dim not multiples of 8"
        return r

    def _nonzero_beta(self) -> bool:
        """The `beta` buffers are part of the state_dict; the fused path assumes the zeros the reference registers
        (checked once per buffer version, not per forward: the check synchronises)."""
        betas = [b for n, b in self.named_buffers() if n.endswith("beta")]
        return cached(self, "_beta_nonzero", betas, lambda: any(bool(b.any()) for b in betas))

    def _prepared(self) -> Dict[str, Tensor]:
        """Device copies of the patch-embedding, positional, pooling and head weights (the encoder layers are the
        transformer engine's)."""
        return cached(self, "_prep", [p for n, p in self.named_parameters() if not n.startswith("transformer.")],
                      self._build)

    def _build(self) -> Dict[str, Tensor]:
        t: Dict[str, Tensor] = {}
        pe = self.to_patch_embedding
        t["pe.ln1"], t["pe.w"], t["pe.b"] = _f32(pe[0].gamma), _bf16_rows(pe[1].weight), _f32(pe[1].bias)
        t["pe.ln2"] = _f32(pe[2].gamma)
        t["pos_h"], t["pos_w"] = _f32(self.pos_embed_height), _f32(self.pos_embed_width)
        # the pooling query is the same for every image: LayerNorm -> to_q -> per-head RMSNorm, once per weight version
        pool = self.attn_pool
        t["pool.kv"] = _bf16_rows(pool.to_kv.weight)
        t["pool.gk"] = _f32(pool.k_norm.gamma).reshape(-1).contiguous()
        t["pool.out"] = _bf16_rows(pool.to_out[0].weight)
        qv = self.attn_pool_queries.detach().float()
        qn = F.layer_norm(qv, qv.shape, pool.norm.gamma.detach().float(), None)
        qh = (pool.to_q.weight.detach().float() @ qn).reshape(pool.heads, -1)
        qh = F.normalize(qh, dim=-1) * pool.q_norm.scale * pool.q_norm.gamma.detach().float().reshape(pool.heads, -1)
        t["pool.qn"] = qh.reshape(-1).contiguous()
        t["pool.queries"] = qv.contiguous()
        t["head.ln"], t["head.w"] = _f32(self.mlp_head[0].gamma), _bf16_rows(self.mlp_head[1].weight)
        return t

    @torch.no_grad()
    def forward_fused(self, batched_images) -> Tensor:
        if torch.is_tensor(batched_images[0]):
            batched_images = [batched_images]
        images = [im for row in batched_images for im in row]        # output order of the reference: row major
        t = self._prepared()
        eng = self.transformer.engine()
        dev = images[0].device
        p, c = self.patch_size, self.channels
        heads = self.attn_pool.heads
        D = t["pos_h"].shape[1]
        I = t["pool.out"].shape[1]
        dh = I // heads
        max_gh, max_gw = self.pos_embed_height.shape[0], self.pos_embed_width.shape[0]
        for img in images:
            assert img.ndim == 3 and img.shape[0] == c
            hh, ww = img.shape[-2:]
            assert hh % p == 0 and ww % p == 0, f'height and width {(hh, ww)} of images must be divisible by patch size {p}'
            if hh < p or ww < p:
                raise ValueError(f"image of {(hh, ww)} pixels has no {p} x {p} patch")
            if hh // p > max_gh or ww // p > max_gw:     # the reference's table lookup raises here (na_vit.py:354-359)
                raise IndexError(f"image of {(hh // p, ww // p)} patches exceeds the positional tables {(max_gh, max_gw)}")
        images = [im.contiguous() for im in images]
        # ---- host-side bookkeeping only: per-image token counts / grid shapes -> one small index buffer on the device;
        #      patch pixels and positional rows are gathered by the kernels
        ix = _lib.VarlenIndex(images, p, dev)
        S, T = ix.S, ix.T
        bf16 = dict(device=dev, dtype=torch.bfloat16)
        f32 = dict(device=dev, dtype=torch.float32)
        # ---- patch embedding: patchify + LN(no bias) -> Linear -> LN(no bias) + pos_h + pos_w   (na_vit.py:300,350-359)
        pd = c * p * p
        a0 = torch.empty(T, pd, **bf16)
        _lib.patchify_varlen_ln(images, t["pe.ln1"], a0, ix.cu, p, index=ix)
        y = torch.empty(T, D, **f32)
        _lib.gemm(a0, t["pe.w"], out_f32=y, bias=t["pe.b"])
        x = torch.empty_like(y)
        xb, stats = eng.entry_buffers(T, dev)
        _lib.embed_varlen(y, t["pe.ln2"], t["pos_h"], t["pos_w"], ix, x, p, xb=xb, stats=stats)
        # ---- encoder layers on the packed [T, D] matrix                                     (na_vit.py:183-193)
        eng.run_blocks(x, primed=xb is not None, varlen=ix)
        xn = eng.workspace(T, dev)["xn"]
        eng.final_norm(x, out_bf16=xn)
        # ---- attention pooling: one query per image over that image's (un-normalised-again) tokens (na_vit.py:371-387)
        kv = torch.empty(T, 2 * I, **bf16)
        _lib.gemm_headnorm(xn, t["pool.kv"], out_bf16=kv, head_gamma=t["pool.gk"], norm_heads=heads,   # k half only
                           dh=dh)
        pooled = torch.empty(S, I, **bf16)
        _lib.attn_pool(kv, t["pool.qn"], ix.cu, pooled, heads, dh)
        z = t["pool.queries"][None, :].expand(S, -1).contiguous()
        _lib.gemm(pooled, t["pool.out"], out_f32=z, resid=z)                      # + queries
        zl = torch.empty(S, D, **bf16)
        _lib.layernorm(z, t["head.ln"], None, out_bf16=zl)
        zl = self.to_latent(zl)
        logits = torch.empty(S, t["head.w"].shape[0], **bf16)
        _lib.gemm(zl, t["head.w"], out_bf16=logits)
        return logits

    # ------------------------------------------------------------------------------------------------------------
    def _tokenise_row(self, images: Sequence[Tensor], training_dropout: bool):
        """One packed row: patch vectors in (c p1 p2) order, (h, w) grid positions and image ids per token."""
        p, c, dev = self.patch_size, self.channels, self.device
        seqs, poss, ids = [], [], []
        for i, img in enumerate(images):
            assert img.ndim == 3 and img.shape[0] == c
            hh, ww = img.shape[-2:]
            assert hh % p == 0 and ww % p == 0, f'height and width {(hh, ww)} of images must be divisible by patch size {p}'
            gh, gw = hh // p, ww // p
            seq = img.reshape(c, gh, p, gw, p).permute(1, 3, 0, 2, 4).reshape(gh * gw, c * p * p)
            pos = torch.stack([torch.arange(gh, device=dev).repeat_interleave(gw),
                               torch.arange(gw, device=dev).repeat(gh)], dim=-1)
            if training_dropout:
                rate = self.calc_token_dropout(hh, ww)
                keep = max(1, int(seq.shape[0] * (1 - rate)))
                idx = torch.randn((seq.shape[0],), device=dev).topk(keep, dim=-1).indices
                seq, pos = seq[idx], pos[idx]
            seqs.append(seq)
            poss.append(pos)
            ids.append(torch.full((seq.shape[0],), i, device=dev, dtype=torch.long))
        return torch.cat(seqs), torch.cat(poss), torch.cat(ids)

    def forward(self, batched_images: Union[List[Tensor], List[List[Tensor]]], group_images: bool = False,
                group_max_seq_len: int = 2048) -> Tensor:
        if self.fused_reason(batched_images) is None:
            # grouping only decides which images share a padded row; the padding-free path does not need it, and the
            # output order (input order) is the same either way -- except for the reference's size assertion
            if group_images:
                flat = batched_images if torch.is_tensor(batched_images[0]) else [im for r in batched_images for im in r]
                for im in flat:
                    n = (im.shape[-2] // self.patch_size) * (im.shape[-1] // self.patch_size)
                    assert n <= group_max_seq_len, \
                        f'image with dimensions {tuple(im.shape[-2:])} exceeds maximum sequence length'
            first = batched_images[0] if torch.is_tensor(batched_images[0]) else batched_images[0][0]
            with on_device(first):
                return self.forward_fused(batched_images)
        return self.forward_eager(batched_images, group_images, group_max_seq_len)

    def forward_eager(self, batched_images: Union[List[Tensor], List[List[Tensor]]], group_images: bool = False,
                      group_max_seq_len: int = 2048) -> Tensor:
        dev = self.device
        training_dropout = self.calc_token_dropout is not None and self.training
        if group_images:
            batched_images = group_images_by_max_seq_len(
                batched_images, patch_size=self.patch_size,
                calc_token_dropout=self.calc_token_dropout if self.training else None, max_seq_len=group_max_seq_len)
        if torch.is_tensor(batched_images[0]):
            batched_images = [batched_images]

        rows = [self._tokenise_row(images, training_dropout) for images in batched_images]
        counts = torch.tensor([len(images) for images in batched_images], device=dev)
        lengths = torch.tensor([r[0].shape[0] for r in rows], device=dev)
        L = int(lengths.max())
        B = len(rows)
        patches = torch.zeros(B, L, rows[0][0].shape[1], device=dev, dtype=rows[0][0].dtype)
        positions = torch.zeros(B, L, 2, device=dev, dtype=torch.long)
        image_ids = torch.zeros(B, L, device=dev, dtype=torch.long)      # padding carries id 0, like pad_sequence
        for b, (seq, pos, ids) in enumerate(rows):
            n = seq.shape[0]
            patches[b, :n], positions[b, :n], image_ids[b, :n] = seq, pos, ids
        valid = torch.arange(L, device=dev)[None, :] < lengths[:, None]                       # key padding mask
        attn_mask = (image_ids[:, None, :, None] == image_ids[:, None, None, :]) & valid[:, None, None, :]

        x = self.to_patch_embedding(patches)
        x = x + self.pos_embed_height[positions[..., 0]] + self.pos_embed_width[positions[..., 1]]
        x = self.dropout(x)
        x = self.transformer(x, attn_mask=attn_mask)

        # attention pooling: query i of a row attends to the tokens of image i of that row
        Q = int(counts.max())
        queries = self.attn_pool_queries[None, None, :].expand(B, Q, -1)
        slot = torch.arange(Q, device=dev)
        pool_mask = (slot[None, :, None] == image_ids[:, None, :]) & valid[:, None, :]
        x = self.attn_pool(queries, context=x, attn_mask=pool_mask[:, None]) + queries
        x = x.reshape(B * Q, -1)[(slot[None, :] < counts[:, None]).reshape(-1)]
        return self.mlp_head(self.to_latent(x))
