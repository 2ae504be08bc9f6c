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

from typing import Callable, Dict, List, Optional, Sequence, Union

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from . import _lib
from .engine import FusedWeightsMixin, _version_key, hooks_inside, ln_mode, on_device, why_not_fused


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


class Transformer(nn.Module):
    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.) -> None:
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))
        self.norm = LayerNorm(dim)

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
        if r is None and attn0.to_q.weight.shape[0] // attn0.heads != 64:
            r = "dim_head != 64 (the attention kernels are built for 64)"
        if r is None and (self.pos_embed_height.shape[1] % 8 or (self.channels * self.patch_size ** 2) % 8):
            r = "dim / patch_dim not multiples of 8"
        return r

    def _nonzero_beta(self) -> bool:
        """The `beta` buffers are part of the state_dict; the fused path assumes the zeros the reference registers
        (checked once per buffer version, not per forward: the check synchronises)."""
        betas = [b for n, b in self.named_buffers() if n.endswith("beta")]
        key = _version_key(betas)
        if getattr(self, "_beta_key", None) != key:
            self._beta_key, self._beta_nonzero = key, any(bool(b.any()) for b in betas)
        return self._beta_nonzero

    def _prepared(self) -> Dict[str, Tensor]:
        params = list(self.parameters())
        key = _version_key(params)
        if getattr(self, "_prep_key", None) == key:
            return self._prep
        f32 = lambda t: t.detach().float().contiguous()
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()
        t: Dict[str, Tensor] = {}
        pe = self.to_patch_embedding
        t["pe.ln1"], t["pe.w"], t["pe.b"], t["pe.ln2"] = f32(pe[0].gamma), bf(pe[1].weight), f32(pe[1].bias), f32(pe[2].gamma)
        t["pos_h"], t["pos_w"] = f32(self.pos_embed_height), f32(self.pos_embed_width)

        def attn_w(prefix: str, a: Attention) -> None:
            t[prefix + "ln"] = f32(a.norm.gamma)
            t[prefix + "qkv"] = bf(torch.cat([a.to_q.weight, a.to_kv.weight], dim=0))       # rows: q | k | v
            t[prefix + "kv"] = bf(a.to_kv.weight)
            t[prefix + "gqk"] = torch.cat([f32(a.q_norm.gamma).reshape(-1), f32(a.k_norm.gamma).reshape(-1)]).contiguous()
            t[prefix + "gk"] = f32(a.k_norm.gamma).reshape(-1).contiguous()
            t[prefix + "out"] = bf(a.to_out[0].weight)

        def fold(name: str, w: Tensor, gamma: Tensor) -> None:
            # LN(x; gamma, beta = 0) W^T == rstd * (x (gamma * W)^T - mu * colsum): see engine.TransformerEngine
            wg = (w.detach().float() * gamma.detach().float()[None, :]).to(torch.bfloat16).contiguous()
            t[name + "g"] = wg
            t[name + "s"] = wg.float().sum(dim=1).contiguous()       # from the ROUNDED weights the MMA sees

        for i, (attn, ff) in enumerate(self.transformer.layers):
            attn_w(f"{i}.a.", attn)
            fold(f"{i}.a.qkv", torch.cat([attn.to_q.weight, attn.to_kv.weight], dim=0), attn.norm.gamma)
            t[f"{i}.a.qkvt"] = torch.zeros(t[f"{i}.a.qkvs"].shape[0], device=t[f"{i}.a.qkvs"].device)
            fold(f"{i}.f.w1", ff[1].weight, ff[0].gamma)
            t[f"{i}.f.ln"] = f32(ff[0].gamma)
            t[f"{i}.f.w1"], t[f"{i}.f.b1"] = bf(ff[1].weight), f32(ff[1].bias)
            t[f"{i}.f.w2"], t[f"{i}.f.b2"] = bf(ff[4].weight), f32(ff[4].bias)
        t["norm"] = f32(self.transformer.norm.gamma)
        attn_w("pool.", self.attn_pool)
        # the pooling query is the same for every image: LayerNorm -> to_q -> per-head RMSNorm, once per weight version
        pool = self.attn_pool
        qv = self.attn_pool_queries.detach().float()
        qn = F.layer_norm(qv, qv.shape, pool.norm.gamma.detach().float(), None)
        qh = (pool.to_q.weight.detach().float() @ qn).reshape(pool.heads, -1)
        qh = F.normalize(qh, dim=-1) * pool.q_norm.scale * pool.q_norm.gamma.detach().float().reshape(pool.heads, -1)
        t["pool.qn"] = qh.reshape(-1).contiguous()
        t["pool.queries"] = qv.contiguous()
        t["head.ln"], t["head.w"] = f32(self.mlp_head[0].gamma), bf(self.mlp_head[1].weight)
        self._prep_key, self._prep = key, t
        return t

    @torch.no_grad()
    def forward_fused(self, batched_images) -> Tensor:
        if torch.is_tensor(batched_images[0]):
            batched_images = [batched_images]
        images = [im for row in batched_images for im in row]        # output order of the reference: row major
        t = self._prepared()
        dev = images[0].device
        p, c = self.patch_size, self.channels
        heads = self.attn_pool.heads
        D = t["pos_h"].shape[1]
        I = t["0.a.out"].shape[1]
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
        fold = ln_mode() == "fold"
        # ---- patch embedding: patchify + LN(no bias) -> Linear -> LN(no bias) + pos_h + pos_w   (na_vit.py:300,350-359)
        pd = c * p * p
        a0 = torch.empty(T, pd, **bf16)
        _lib.patchify_varlen_ln(images, t["pe.ln1"], a0, ix.cu, p, index=ix)
        y = torch.empty(T, D, **f32)
        _lib.gemm(a0, t["pe.w"], out_f32=y, bias=t["pe.b"])
        x = torch.empty_like(y)
        xn = torch.empty(T, D, **bf16)              # exact: LayerNorm output; fold: bf16 copy of the residual stream
        st_in = torch.empty(T, 1, 2, **f32) if fold else None
        _lib.embed_varlen(y, t["pe.ln2"], t["pos_h"], t["pos_w"], ix, x, p, xb=xn if fold else None, stats=st_in)
        # ---- encoder layers on the packed [T, D] matrix                                     (na_vit.py:183-193)
        qkv = torch.empty(T, 3 * I, **bf16)
        o = torch.empty(T, I, **bf16)
        hbuf = torch.empty(T, t["0.f.w1"].shape[0], **bf16)
        depth = len(self.transformer.layers)
        if fold:
            # LayerNorm folded into the QKV / FC1 GEMMs (engine.py): the residual GEMMs emit the bf16 copy of x and
            # the partial row statistics the next folded GEMM needs
            parts = _lib.stats_parts(D)
            sa, sb = torch.empty(T, parts, 2, **f32), torch.empty(T, parts, 2, **f32)
            for i in range(depth):
                _lib.gemm_headnorm(xn, t[f"{i}.a.qkvg"], out_bf16=qkv, bias=t[f"{i}.a.qkvt"],
                                   ln_sums=st_in if i == 0 else sa, col_s=t[f"{i}.a.qkvs"],
                                   head_gamma=t[f"{i}.a.gqk"], norm_heads=2 * heads)   # q / k RMSNorm in the epilogue
                _lib.attention_varlen(qkv, o, ix.cu, ix.tile_prefix, ix.total_tiles, heads, 64, 1.0)
                _lib.gemm(o, t[f"{i}.a.out"], out_f32=x, out_bf16=xn, resid=x, stats_out=sb)
                _lib.gemm(xn, t[f"{i}.f.w1g"], out_bf16=hbuf, bias=t[f"{i}.f.b1"], gelu=True, ln_sums=sb,
                          col_s=t[f"{i}.f.w1s"])
                _lib.gemm(hbuf, t[f"{i}.f.w2"], out_f32=x, out_bf16=xn, bias=t[f"{i}.f.b2"], resid=x, stats_out=sa)
        else:
            for i in range(depth):
                _lib.layernorm(x, t[f"{i}.a.ln"], None, out_bf16=xn)
                _lib.gemm_headnorm(xn, t[f"{i}.a.qkv"], out_bf16=qkv, head_gamma=t[f"{i}.a.gqk"], norm_heads=2 * heads)
                _lib.attention_varlen(qkv, o, ix.cu, ix.tile_prefix, ix.total_tiles, heads, 64, 1.0)
                _lib.gemm(o, t[f"{i}.a.out"], out_f32=x, resid=x)
                _lib.layernorm(x, t[f"{i}.f.ln"], None, out_bf16=xn)
                _lib.gemm(xn, t[f"{i}.f.w1"], out_bf16=hbuf, bias=t[f"{i}.f.b1"], gelu=True)
                _lib.gemm(hbuf, t[f"{i}.f.w2"], out_f32=x, bias=t[f"{i}.f.b2"], resid=x)
        _lib.layernorm(x, t["norm"], None, out_bf16=xn)
        # ---- attention pooling: one query per image over that image's (un-normalised-again) tokens (na_vit.py:371-387)
        kv = torch.empty(T, 2 * I, **bf16)
        _lib.gemm_headnorm(xn, t["pool.kv"], out_bf16=kv, head_gamma=t["pool.gk"], norm_heads=heads)   # k half only
        pooled = torch.empty(S, I, **bf16)
        _lib.attn_pool(kv, t["pool.qn"], ix.cu, pooled, heads, 64)
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
