"""Drop-in `NaViT` of `vit_pytorch.na_vit_nested_tensor` (reference na_vit_nested_tensor.py:134-301): the padding-free
NaViT front-end that hands a list of different-resolution images to the encoder as ONE jagged batch.

It differs from `na_vit.NaViT` in the module tree (so it is its own class, not a flag): separate `to_queries` /
`to_keys` / `to_values` projections, q / k normalised by `nn.LayerNorm(dim_head, bias=False)` (`qk_rmsnorm=True`) or not
at all, `nn.LayerNorm` (with bias) around the patch projection, bias-free LayerNorms everywhere else, default softmax
scale `dim_head ** -0.5`, and attention pooling WITHOUT the residual query (`forward(List[Tensor]) -> (n, classes)`).

Two executions of the same arithmetic:
  * PyTorch graph (CPU / fp32 / training / autograd / hooks): images never interact, so the reference's jagged batch is
    evaluated image by image with plain dense tensors -- no dependence on the prototype nested-tensor operators.
  * fused sm_90a path (CUDA bf16, eval): exactly `na_vit.NaViT`'s padding-free schedule -- all tokens in one [T, D]
    matrix described by `cu_seqlens`, `b200vit_patchify_varlen_ln`, `b200vit_embed_varlen`, LN-folded QKV GEMM with the
    per-head LayerNorm as its epilogue (`EPI_HEADLN`), `b200vit_attention_varlen`, dual-epilogue residual GEMMs,
    `b200vit_attn_pool`.  The LayerNorm biases of the patch embedding are folded on the host (beta_1 into the patch
    projection's bias, beta_2 into the height positional table), which is exact in real arithmetic.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from . import _lib
from .engine import FusedWeightsMixin, _version_key, hooks_inside, ln_mode, on_device, why_not_fused


def FeedForward(dim: int, hidden_dim: int, dropout: float = 0.) -> nn.Sequential:
    return nn.Sequential(nn.LayerNorm(dim, bias=False), nn.Linear(dim, hidden_dim), nn.GELU(), nn.Dropout(dropout),
                         nn.Linear(hidden_dim, dim), nn.Dropout(dropout))


class Attention(nn.Module):
    """reference na_vit_nested_tensor.py:42-119, on dense [n, dim] (one image) instead of a jagged batch."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, dropout: float = 0., qk_norm: bool = True) -> None:
        super().__init__()
        self.norm = nn.LayerNorm(dim, bias=False)
        dim_inner = heads * dim_head
        self.heads, self.dim_head = heads, dim_head
        self.to_queries = nn.Linear(dim, dim_inner, bias=False)
        self.to_keys = nn.Linear(dim, dim_inner, bias=False)
        self.to_values = nn.Linear(dim, dim_inner, bias=False)
        self.query_norm = nn.LayerNorm(dim_head, bias=False) if qk_norm else nn.Identity()
        self.key_norm = nn.LayerNorm(dim_head, bias=False) if qk_norm else nn.Identity()
        self.dropout = dropout
        self.to_out = nn.Linear(dim_inner, dim, bias=False)

    def forward(self, x: Tensor, context: Optional[Tensor] = None) -> Tensor:
        x = self.norm(x)
        context = x if context is None else context
        h, d = self.heads, self.dim_head
        q = self.query_norm(self.to_queries(x).unflatten(-1, (h, d))).transpose(-3, -2)
        k = self.key_norm(self.to_keys(context).unflatten(-1, (h, d))).transpose(-3, -2)
        v = self.to_values(context).unflatten(-1, (h, d)).transpose(-3, -2)
        out = F.scaled_dot_product_attention(q, k, v, dropout_p=self.dropout if self.training else 0.)
        return self.to_out(out.transpose(-3, -2).flatten(-2))


class Transformer(nn.Module):
    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.,
                 qk_norm: bool = True) -> None:
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout, qk_norm=qk_norm),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))
        self.norm = nn.LayerNorm(dim, bias=False)

    def forward(self, x: Tensor) -> Tensor:
        for attn, ff in self.layers:
            x = attn(x) + x
            x = ff(x) + x
        return self.norm(x)


class Patches(nn.Module):
    """'c (h p1) (w p2) -> h w (c p1 p2)' (reference :186)."""

    def __init__(self, p: int) -> None:
        super().__init__()
        self.p = p

    def forward(self, img: Tensor) -> Tensor:
        c, hh, ww = img.shape
        p = self.p
        return img.reshape(c, hh // p, p, ww // p, p).permute(1, 3, 0, 2, 4).reshape(hh // p, ww // p, c * p * p)


class NaViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, channels=3, dim_head=64,
                 dropout=0., emb_dropout=0., qk_rmsnorm=True, token_dropout_prob: Optional[float] = None) -> None:
        super().__init__()
        image_height, image_width = image_size if isinstance(image_size, tuple) else (image_size, image_size)
        self.token_dropout_prob = token_dropout_prob
        assert image_height % patch_size == 0 and image_width % patch_size == 0, \
            'Image dimensions must be divisible by the patch size.'
        patch_dim = channels * (patch_size ** 2)
        self.channels = channels
        self.patch_size = patch_size
        self.to_patches = Patches(patch_size)
        self.to_patch_embedding = nn.Sequential(nn.LayerNorm(patch_dim), nn.Linear(patch_dim, dim), nn.LayerNorm(dim))
        self.pos_embed_height = nn.Parameter(torch.randn(image_height // patch_size, dim))
        self.pos_embed_width = nn.Parameter(torch.randn(image_width // patch_size, dim))
        self.dropout = nn.Dropout(emb_dropout)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim, dropout, qk_rmsnorm)
        self.attn_pool_queries = nn.Parameter(torch.randn(dim))
        self.attn_pool = Attention(dim=dim, dim_head=dim_head, heads=heads)
        self.to_latent = nn.Identity()
        self.mlp_head = nn.Sequential(nn.LayerNorm(dim, bias=False), nn.Linear(dim, num_classes, bias=False))
        self._dropout_p = float(dropout)

    @property
    def device(self):
        return next(self.parameters()).device

    # ------------------------------------------------------------------------------------------------------------
    def _check(self, images: List[Tensor]) -> None:
        assert all(im.ndim == 3 and im.shape[0] == self.channels for im in images), \
            f'all images must have {self.channels} channels and number of dimensions of 3 (channels, height, width)'

    def forward(self, images: List[Tensor]) -> Tensor:
        if self.fused_reason(images) is None:
            with on_device(images[0]):
                return self.forward_fused(images)
        return self.forward_eager(images)

    def forward_eager(self, images: List[Tensor]) -> Tensor:
        self._check(images)
        dev = self.device
        out = []
        for img in images:
            patches = self.to_patches(img)
            gh, gw = patches.shape[:2]
            tokens = patches.reshape(gh * gw, -1)
            hi = torch.arange(gh, device=dev).repeat_interleave(gw)
            wi = torch.arange(gw, device=dev).repeat(gh)
            if self.training and self.token_dropout_prob is not None and self.token_dropout_prob > 0:
                keep = max(1, int((1. - self.token_dropout_prob) * tokens.shape[0]))
                idx = torch.randn((tokens.shape[0],), device=dev).topk(keep, dim=-1).indices
                tokens, hi, wi = tokens[idx], hi[idx], wi[idx]
            x = self.to_patch_embedding(tokens) + (self.pos_embed_height[hi] + self.pos_embed_width[wi])
            x = self.transformer(self.dropout(x))
            out.append(self.attn_pool(self.attn_pool_queries[None, :], x))
        logits = torch.cat(out, dim=0)
        return self.mlp_head(self.to_latent(logits))

    # ------------------------------------------------------------------------------------------------------------
    # fused sm_90a path
    # ------------------------------------------------------------------------------------------------------------
    def fused_reason(self, images=None) -> Optional[str]:
        if not images:
            return "no input given"
        if not all(torch.is_tensor(im) for im in images):
            return "input is not a list of tensors"
        first = images[0]
        if len(self.transformer.layers) == 0:
            return "depth == 0"
        r = why_not_fused(list(self.parameters()), first, training=self.training,
                          dropout_p=max(self.dropout.p, self._dropout_p))
        if r is None:
            for im in images:
                if not (im.is_cuda and im.device == first.device and im.dtype == first.dtype):
                    return "images differ in device or dtype"
                if torch.is_grad_enabled() and im.requires_grad:
                    return "autograd is recording (fused path is forward only)"
        if r is None and self.training and self.token_dropout_prob:
            r = "token dropout is active"
        if r is None and hooks_inside(self, skip=(self.to_latent,)):
            r = "forward hooks registered inside the model"
        if r is None and self.attn_pool.dim_head != 64:
            r = "dim_head != 64 (the attention kernels are built for 64)"
        if r is None and (self.pos_embed_height.shape[1] % 8 or (self.channels * self.patch_size ** 2) % 8):
            r = "dim / patch_dim not multiples of 8"
        return r

    def _prepared(self) -> Dict[str, Tensor]:
        params = list(self.parameters())
        key = _version_key(params)
        if getattr(self, "_prep_key", None) == key:
            return self._prep
        f32 = lambda t: t.detach().float().contiguous()
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()
        t: Dict[str, Tensor] = {}
        ln1, lin, ln2 = self.to_patch_embedding
        # LN(x; g1, b1) W^T + c == (x_hat g1) W^T + (W b1 + c): beta_1 moves into the projection's bias
        t["pe.ln1"], t["pe.w"] = f32(ln1.weight), bf(lin.weight)
        t["pe.b"] = (lin.weight.detach().float() @ ln1.bias.detach().float() + lin.bias.detach().float()).contiguous()
        # LN(y; g2, b2) + pos_h + pos_w == y_hat g2 + (pos_h + b2) + pos_w: beta_2 moves into the height table
        t["pe.ln2"] = f32(ln2.weight)
        t["pos_h"] = (self.pos_embed_height.detach().float() + ln2.bias.detach().float()[None, :]).contiguous()
        t["pos_w"] = f32(self.pos_embed_width)

        def fold(name: str, w: Tensor, gamma: Tensor) -> None:
            wg = (w.detach().float() * gamma.detach().float()[None, :]).to(torch.bfloat16).contiguous()
            t[name + "g"] = wg
            t[name + "s"] = wg.float().sum(dim=1).contiguous()

        def head_gamma(a: Attention, which) -> Optional[Tensor]:
            mods = [getattr(a, n) for n in which]
            if isinstance(mods[0], nn.Identity):
                return None
            return torch.cat([f32(m.weight).repeat(a.heads) for m in mods]).contiguous()   # same gamma for every head

        for i, (attn, ff) in enumerate(self.transformer.layers):
            w = torch.cat([attn.to_queries.weight, attn.to_keys.weight, attn.to_values.weight], dim=0)
            t[f"{i}.qkv"] = bf(w)
            fold(f"{i}.qkv", w, attn.norm.weight)
            t[f"{i}.qkvt"] = torch.zeros(w.shape[0], device=w.device)
            t[f"{i}.ln1"] = f32(attn.norm.weight)
            t[f"{i}.gqk"] = head_gamma(attn, ("query_norm", "key_norm"))
            t[f"{i}.out"] = bf(attn.to_out.weight)
            fold(f"{i}.w1", ff[1].weight, ff[0].weight)
            t[f"{i}.ln2"] = f32(ff[0].weight)
            t[f"{i}.w1"], t[f"{i}.b1"] = bf(ff[1].weight), f32(ff[1].bias)
            t[f"{i}.w2"], t[f"{i}.b2"] = bf(ff[4].weight), f32(ff[4].bias)
        t["norm"] = f32(self.transformer.norm.weight)
        pool = self.attn_pool
        t["pool.kv"] = bf(torch.cat([pool.to_keys.weight, pool.to_values.weight], dim=0))
        t["pool.gk"] = head_gamma(pool, ("key_norm",))
        t["pool.out"] = bf(pool.to_out.weight)
        # the pooling query is the same for every image: LayerNorm -> to_queries -> per-head LayerNorm, times the
        # softmax scale dim_head ** -0.5 (the pooling kernel uses scale 1)
        qv = self.attn_pool_queries.detach().float()
        qn = F.layer_norm(qv, qv.shape, pool.norm.weight.detach().float(), None)
        qh = (pool.to_queries.weight.detach().float() @ qn).reshape(pool.heads, -1)
        if not isinstance(pool.query_norm, nn.Identity):
            qh = F.layer_norm(qh, qh.shape[-1:], pool.query_norm.weight.detach().float(), None, pool.query_norm.eps)
        t["pool.qn"] = (qh * pool.dim_head ** -0.5).reshape(-1).contiguous()
        t["head.ln"], t["head.w"] = f32(self.mlp_head[0].weight), bf(self.mlp_head[1].weight)
        self._prep_key, self._prep = key, t
        return t

    @torch.no_grad()
    def forward_fused(self, images: List[Tensor]) -> Tensor:
        self._check(images)
        t = self._prepared()
        dev = images[0].device
        p, c = self.patch_size, self.channels
        pool = self.attn_pool
        heads, dh = pool.heads, pool.dim_head
        D = t["pos_h"].shape[1]
        I = heads * dh
        max_gh, max_gw = self.pos_embed_height.shape[0], self.pos_embed_width.shape[0]
        for img in images:
            hh, ww = img.shape[-2:]
            assert hh % p == 0 and ww % p == 0, f'height and width {(hh, ww)} of images must be divisible by patch size {p}'
            if hh < p or ww < p:
                raise ValueError(f"image of {(hh, ww)} pixels has no {p} x {p} patch")
            if hh // p > max_gh or ww // p > max_gw:      # the reference's table lookup raises here
                raise IndexError(f"image of {(hh // p, ww // p)} patches exceeds the positional tables {(max_gh, max_gw)}")
        images = [im.contiguous() for im in images]
        ix = _lib.VarlenIndex(images, p, dev)
        S, T = ix.S, ix.T
        bf16 = dict(device=dev, dtype=torch.bfloat16)
        f32 = dict(device=dev, dtype=torch.float32)
        fold = ln_mode() == "fold"
        scale = dh ** -0.5
        lyr = self.transformer.layers
        # ---- patch embedding (reference :186-192,226-262)
        a0 = torch.empty(T, c * p * p, **bf16)
        _lib.patchify_varlen_ln(images, t["pe.ln1"], a0, ix.cu, p, eps=self.to_patch_embedding[0].eps, index=ix)
        y = torch.empty(T, D, **f32)
        _lib.gemm(a0, t["pe.w"], out_f32=y, bias=t["pe.b"])
        x = torch.empty_like(y)
        xn = torch.empty(T, D, **bf16)
        st_in = torch.empty(T, 1, 2, **f32) if fold else None
        _lib.embed_varlen(y, t["pe.ln2"], t["pos_h"], t["pos_w"], ix, x, p, xb=xn if fold else None, stats=st_in,
                          eps=self.to_patch_embedding[2].eps)
        # ---- encoder layers on the packed [T, D] matrix (reference :121-132)
        qkv = torch.empty(T, 3 * I, **bf16)
        o = torch.empty(T, I, **bf16)
        hbuf = torch.empty(T, t["0.w1"].shape[0], **bf16)
        parts = _lib.stats_parts(D)
        sa, sb = (torch.empty(T, parts, 2, **f32), torch.empty(T, parts, 2, **f32)) if fold else (None, None)
        for i, (attn, ff) in enumerate(lyr):
            gqk = t[f"{i}.gqk"]
            hln = None if gqk is None else attn.query_norm.eps
            if fold:
                kw = dict(out_bf16=qkv, bias=t[f"{i}.qkvt"], ln_sums=st_in if i == 0 else sa, col_s=t[f"{i}.qkvs"],
                          ln_eps=attn.norm.eps)
                if gqk is None:
                    _lib.gemm(xn, t[f"{i}.qkvg"], **kw)
                else:
                    _lib.gemm_headnorm(xn, t[f"{i}.qkvg"], head_gamma=gqk, norm_heads=2 * heads,
                                       head_layernorm_eps=hln, **kw)
            else:
                _lib.layernorm(x, t[f"{i}.ln1"], None, out_bf16=xn, eps=attn.norm.eps)
                if gqk is None:
                    _lib.gemm(xn, t[f"{i}.qkv"], out_bf16=qkv)
                else:
                    _lib.gemm_headnorm(xn, t[f"{i}.qkv"], out_bf16=qkv, head_gamma=gqk, norm_heads=2 * heads,
                                       head_layernorm_eps=hln)
            _lib.attention_varlen(qkv, o, ix.cu, ix.tile_prefix, ix.total_tiles, heads, dh, scale)
            if fold:
                _lib.gemm(o, t[f"{i}.out"], out_f32=x, out_bf16=xn, resid=x, stats_out=sb)
                _lib.gemm(xn, t[f"{i}.w1g"], out_bf16=hbuf, bias=t[f"{i}.b1"], gelu=True, ln_sums=sb,
                          col_s=t[f"{i}.w1s"], ln_eps=ff[0].eps)
                _lib.gemm(hbuf, t[f"{i}.w2"], out_f32=x, out_bf16=xn, bias=t[f"{i}.b2"], resid=x, stats_out=sa)
            else:
                _lib.gemm(o, t[f"{i}.out"], out_f32=x, resid=x)
                _lib.layernorm(x, t[f"{i}.ln2"], None, out_bf16=xn, eps=ff[0].eps)
                _lib.gemm(xn, t[f"{i}.w1"], out_bf16=hbuf, bias=t[f"{i}.b1"], gelu=True)
                _lib.gemm(hbuf, t[f"{i}.w2"], out_f32=x, bias=t[f"{i}.b2"], resid=x)
        _lib.layernorm(x, t["norm"], None, out_bf16=xn, eps=self.transformer.norm.eps)
        # ---- attention pooling, one query per image, no residual (reference :284-296)
        kv = torch.empty(T, 2 * I, **bf16)
        if t["pool.gk"] is None:
            _lib.gemm(xn, t["pool.kv"], out_bf16=kv)
        else:
            _lib.gemm_headnorm(xn, t["pool.kv"], out_bf16=kv, head_gamma=t["pool.gk"], norm_heads=heads,
                               head_layernorm_eps=pool.key_norm.eps)
        pooled = torch.empty(S, I, **bf16)
        _lib.attn_pool(kv, t["pool.qn"], ix.cu, pooled, heads, dh)
        z = torch.empty(S, D, **f32)
        _lib.gemm(pooled, t["pool.out"], out_f32=z)
        zl = torch.empty(S, D, **bf16)
        _lib.cast_f32_bf16(z.view(-1), zl.view(-1))
        lat = self.to_latent(zl)                        # stays a called module
        if lat is not zl:
            z = lat.float().contiguous()
        zn = torch.empty(S, D, **bf16)
        _lib.layernorm(z, t["head.ln"], None, out_bf16=zn, eps=self.mlp_head[0].eps)
        logits = torch.empty(S, t["head.w"].shape[0], **bf16)
        _lib.gemm(zn, t["head.w"], out_bf16=logits)
        return logits
