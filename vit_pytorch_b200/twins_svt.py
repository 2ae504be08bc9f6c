"""Drop-in `TwinsSVT` for lucidrains/vit-pytorch's `vit_pytorch.twins_svt.TwinsSVT` (Twins-SVT: locally-grouped and
global sub-sampled attention over a 2-D token map), with `Transformer`, `LocalAttention`, `GlobalAttention`,
`FeedForward`, `PatchEmbedding`, `PEG`, `LayerNorm` and `Residual` of the same file, and a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed): `layers.{0..3}` the four stages, each `Sequential(PatchEmbedding, Transformer(depth
1), PEG, Transformer(depth s_depth))`, `layers.4` the average pool, `layers.5` the parameter-free squeeze, `layers.6`
the classifier (reference twins_svt.py:178-235).  Every Transformer runs 8 heads of 64 whatever its stage's width; the
last stage has no local attention (positions 0 and 1 of its layers are nn.Identity).  The PyTorch graph below mirrors
the reference module for module, so hooks on any submodule keep working there.

Fused forward, on the token-major map x fp32 [B*h*w, C] (token (b, y, x) at row (b*h + y)*w + x), per stage:
  * PatchEmbedding (twins_svt.py:59-75): stage 1 b200vit_patchify_ln on the NCHW image, later stages
    b200vit_merge_patches_ln on the previous stage's map -- both emit the merged features in (p1 p2 c) order, so the
    first LayerNorm's affine and the 1 x 1 convolution's weight columns are permuted from the reference's (c p1 p2) --
    then the convolution as one GEMM and b200vit_embed_tokens for the second LayerNorm, writing the stage's stream
    and, in fold mode, its bf16 copy and row statistics;
  * both Transformers through TransformerEngine.run_blocks with the stage's grid: a Twins layer is two pre-LN pairs,
    (LocalAttention, FeedForward) with b200vit_attention_window, then (GlobalAttention, FeedForward) with
    b200vit_attention_kv over the keys of the stride-k convolution (engine.py);
  * PEG between them (twins_svt.py:77-83): b200vit_peg into a second buffer, and in fold mode b200vit_rowstats_cast
    into the next Transformer's entry buffers;
  * head: b200vit_mean_pool over the last map, then the classifier GEMM.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import (PEG_KERNEL_SIZES, EncoderLayer, FusedEncoder, FusedWeightsMixin, Norm, StridedKV, Windows,
                     _bf16_rows, _f32, cached, common_reason, depthwise_peg_weights, head_engine, on_device)

__all__ = ["FeedForward", "GlobalAttention", "LayerNorm", "LocalAttention", "PEG", "PatchEmbedding", "Residual",
           "Transformer", "TwinsSVT", "group_by_key_prefix_and_remove_prefix", "group_dict_by_key", "merge_weights",
           "peg_weights"]


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


class Residual(nn.Module):
    def __init__(self, fn) -> None:
        super().__init__()
        self.fn = fn

    def forward(self, x, **kwargs):
        return self.fn(x, **kwargs) + x


class LayerNorm(nn.Module):
    """LayerNorm over the channel dim of an NCHW map: biased variance, eps inside the square root, affine `g` / `b` of
    shape (1, dim, 1, 1) (reference twins_svt.py:33-43)."""

    def __init__(self, dim, eps=1e-5) -> None:
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
    def __init__(self, dim, mult=4, dropout=0.) -> None:
        super().__init__()
        self.net = nn.Sequential(
            LayerNorm(dim),
            nn.Conv2d(dim, dim * mult, 1),
            nn.GELU(),
            nn.Dropout(dropout),
            nn.Conv2d(dim * mult, dim, 1),
            nn.Dropout(dropout),
        )

    def forward(self, x):
        return self.net(x)


class PatchEmbedding(nn.Module):
    """p x p patch merging with the features ordered (c p1 p2), LayerNorm over all of them, 1 x 1 convolution,
    LayerNorm (reference twins_svt.py:59-75)."""

    def __init__(self, *, dim, dim_out, patch_size) -> None:
        super().__init__()
        self.dim = dim
        self.dim_out = dim_out
        self.patch_size = patch_size
        self.proj = nn.Sequential(
            LayerNorm(patch_size ** 2 * dim),
            nn.Conv2d(patch_size ** 2 * dim, dim_out, 1),
            LayerNorm(dim_out),
        )

    def forward(self, fmap):
        p = self.patch_size
        b, c, H, W = fmap.shape
        if H % p or W % p:
            # what einops raises for 'b c (h p1) (w p2) -> b (c p1 p2) h w'
            raise RuntimeError(f"PatchEmbedding: a {H} x {W} map is not divisible by patch_size={p} (twins_svt.py:74)")
        fmap = fmap.reshape(b, c, H // p, p, W // p, p).permute(0, 1, 3, 5, 2, 4).reshape(b, c * p * p, H // p, W // p)
        return self.proj(fmap)


class PEG(nn.Module):
    def __init__(self, dim, kernel_size=3) -> None:
        super().__init__()
        self.proj = Residual(nn.Conv2d(dim, dim, kernel_size=kernel_size, padding=kernel_size // 2, groups=dim,
                                       stride=1))

    def forward(self, x):
        return self.proj(x)


def _heads(t: torch.Tensor, h: int) -> torch.Tensor:
    """(b, h*d, x, y) -> (b*h, x*y, d)"""
    b, c, x, y = t.shape
    return t.reshape(b * h, c // h, x * y).transpose(1, 2)


class LocalAttention(nn.Module):
    def __init__(self, dim, heads=8, dim_head=64, dropout=0., patch_size=7) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.patch_size = patch_size
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.norm = LayerNorm(dim)
        self.to_q = nn.Conv2d(dim, inner_dim, 1, bias=False)
        self.to_kv = nn.Conv2d(dim, inner_dim * 2, 1, bias=False)
        self.to_out = nn.Sequential(nn.Conv2d(inner_dim, dim, 1), nn.Dropout(dropout))

    def forward(self, fmap):
        fmap = self.norm(fmap)
        b, c, H, W = fmap.shape
        p, h = self.patch_size, self.heads
        if H % p or W % p:
            raise RuntimeError(f"LocalAttention: a {H} x {W} map is not divisible into {p} x {p} windows "
                               "(twins_svt.py:109)")
        x, y = H // p, W // p
        fmap = fmap.reshape(b, c, x, p, y, p).permute(0, 2, 4, 1, 3, 5).reshape(b * x * y, c, p, p)
        q, k, v = (self.to_q(fmap), *self.to_kv(fmap).chunk(2, dim=1))
        q, k, v = (_heads(t, h) for t in (q, k, v))
        dots = torch.einsum('b i d, b j d -> b i j', q, k) * self.scale
        attn = dots.softmax(dim=-1)
        out = torch.einsum('b i j, b j d -> b i d', attn, v)                      # (b x y h) (p1 p2) d
        out = out.reshape(b, x, y, h, p, p, -1).permute(0, 3, 6, 1, 4, 2, 5).reshape(b, -1, H, W)
        return self.to_out(out)


class GlobalAttention(nn.Module):
    def __init__(self, dim, heads=8, dim_head=64, dropout=0., k=7) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.norm = LayerNorm(dim)
        self.to_q = nn.Conv2d(dim, inner_dim, 1, bias=False)
        self.to_kv = nn.Conv2d(dim, inner_dim * 2, k, stride=k, bias=False)
        self.dropout = nn.Dropout(dropout)
        self.to_out = nn.Sequential(nn.Conv2d(inner_dim, dim, 1), nn.Dropout(dropout))

    def forward(self, x):
        x = self.norm(x)
        b, _, X, Y = x.shape
        h = self.heads
        q, k, v = (self.to_q(x), *self.to_kv(x).chunk(2, dim=1))
        q, k, v = (_heads(t, h) for t in (q, k, v))
        dots = torch.einsum('b i d, b j d -> b i j', q, k) * self.scale
        attn = self.dropout(dots.softmax(dim=-1))
        out = torch.einsum('b i j, b j d -> b i d', attn, v)
        out = out.reshape(b, h, X * Y, -1).permute(0, 1, 3, 2).reshape(b, -1, X, Y)
        return self.to_out(out)


class Transformer(FusedEncoder, nn.Module):
    """depth x (LocalAttention, FeedForward, GlobalAttention, FeedForward), each in a Residual; without `has_local`
    the first two are nn.Identity (reference twins_svt.py:159-176).  The fused forward runs it through engine()."""

    def __init__(self, dim, depth, heads=8, dim_head=64, mlp_mult=4, local_patch_size=7, global_k=7, dropout=0.,
                 has_local=True) -> None:
        super().__init__()
        self.dim_head = dim_head
        self.dropout_p = float(dropout)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Residual(LocalAttention(dim, heads=heads, dim_head=dim_head, dropout=dropout,
                                        patch_size=local_patch_size)) if has_local else nn.Identity(),
                Residual(FeedForward(dim, mlp_mult, dropout=dropout)) if has_local else nn.Identity(),
                Residual(GlobalAttention(dim, heads=heads, dim_head=dim_head, dropout=dropout, k=global_k)),
                Residual(FeedForward(dim, mlp_mult, dropout=dropout)),
            ]))

    def forward(self, x):
        for local_attn, ff1, global_attn, ff2 in self.layers:
            x = local_attn(x)
            x = ff1(x)
            x = global_attn(x)
            x = ff2(x)
        return x

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        """Two EncoderLayers per Twins layer: (local attention, FF) with Windows, then (global attention, FF) with
        StridedKV; only the second where the layer has no local attention."""
        layers = []
        for local_attn, ff1, global_attn, ff2 in self.layers:
            for attn, ff in ((local_attn, ff1), (global_attn, ff2)):
                if isinstance(attn, nn.Identity):
                    continue
                a, f = attn.fn, ff.fn.net
                I, D = a.to_q.weight.shape[:2]
                local = isinstance(a, LocalAttention)
                qkv_w = (torch.cat((a.to_q.weight.detach(), a.to_kv.weight.detach())).reshape(3 * I, D) if local
                         else a.to_q.weight.reshape(I, D))
                layers.append(EncoderLayer(
                    ln1=_norm(a.norm), qkv_w=qkv_w, out_w=a.to_out[0].weight.reshape(D, I), out_b=a.to_out[0].bias,
                    ln2=_norm(f[0]), fc1_w=f[1].weight.reshape(-1, D), fc1_b=f[1].bias,
                    fc2_w=f[4].weight.reshape(D, -1), fc2_b=f[4].bias, heads=a.heads, dim_head=I // a.heads,
                    scale=a.scale,
                    attention=Windows(a.patch_size) if local else StridedKV(a.to_kv.kernel_size[0], a.to_kv.weight)))
        return layers, None


def _to_p1p2c(t: torch.Tensor, C: int, p: int) -> torch.Tensor:
    """The last dim of t from the reference's (c p1 p2) feature order to (p1 p2 c)."""
    return t.reshape(*t.shape[:-1], C, p * p).transpose(-1, -2).reshape(*t.shape[:-1], C * p * p)


def merge_weights(pe: PatchEmbedding) -> dict:
    """The prepared weights of a PatchEmbedding for merged features in (p1 p2 c) order: 'g' / 'b' fp32 [p*p*C] (the
    first LayerNorm), 'w' bf16 [dim_out, kp] (the 1 x 1 convolution, K zero-padded to kp) and 'bias' fp32, 'g2' / 'b2'
    fp32 [dim_out] (the second LayerNorm)."""
    ln1, conv, ln2 = pe.proj
    C, p = pe.dim, pe.patch_size
    K = C * p * p
    kp = (K + 63) // 64 * 64
    w = _to_p1p2c(conv.weight.detach().reshape(pe.dim_out, K), C, p)
    return {"g": _to_p1p2c(ln1.g.detach().float().reshape(K), C, p).contiguous(),
            "b": _to_p1p2c(ln1.b.detach().float().reshape(K), C, p).contiguous(),
            "w": _bf16_rows(w, kp), "bias": _f32(conv.bias), "kp": kp,
            "g2": _f32(ln2.g.reshape(-1)), "b2": _f32(ln2.b.reshape(-1))}


def peg_weights(peg: PEG) -> dict:
    """'w' fp32 [k*k, C] (the depthwise weights tap major) and 'b' fp32 [C] of b200vit_peg."""
    return depthwise_peg_weights(peg.proj.fn)


class _Squeeze(nn.Module):
    """Rearrange('... () () -> ...') (reference twins_svt.py:230), without einops."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x.reshape(x.shape[:-2])


class TwinsSVT(FusedWeightsMixin, nn.Module):
    def __init__(
        self,
        *,
        num_classes,
        s1_emb_dim=64,
        s1_patch_size=4,
        s1_local_patch_size=7,
        s1_global_k=7,
        s1_depth=1,
        s2_emb_dim=128,
        s2_patch_size=2,
        s2_local_patch_size=7,
        s2_global_k=7,
        s2_depth=1,
        s3_emb_dim=256,
        s3_patch_size=2,
        s3_local_patch_size=7,
        s3_global_k=7,
        s3_depth=5,
        s4_emb_dim=512,
        s4_patch_size=2,
        s4_local_patch_size=7,
        s4_global_k=7,
        s4_depth=4,
        peg_kernel_size=3,
        dropout=0.
    ) -> None:
        super().__init__()
        kwargs = dict(locals())
        dim = 3
        layers = []
        for prefix in ('s1', 's2', 's3', 's4'):
            config, kwargs = group_by_key_prefix_and_remove_prefix(f'{prefix}_', kwargs)
            is_last = prefix == 's4'
            dim_next = config['emb_dim']
            layers.append(nn.Sequential(
                PatchEmbedding(dim=dim, dim_out=dim_next, patch_size=config['patch_size']),
                Transformer(dim=dim_next, depth=1, local_patch_size=config['local_patch_size'],
                            global_k=config['global_k'], dropout=dropout, has_local=not is_last),
                PEG(dim=dim_next, kernel_size=peg_kernel_size),
                Transformer(dim=dim_next, depth=config['depth'], local_patch_size=config['local_patch_size'],
                            global_k=config['global_k'], dropout=dropout, has_local=not is_last),
            ))
            dim = dim_next
        self.layers = nn.Sequential(*layers, nn.AdaptiveAvgPool2d(1), _Squeeze(), nn.Linear(dim, num_classes))
        self._dropout_p = float(dropout)

    def stages(self) -> List[nn.Sequential]:
        return list(self.layers[:4])

    # ---------------------------------------------------------------------------------------------- dispatch
    def stage_reason(self, H: int, W: int) -> Tuple[Optional[str], List[Tuple[int, int]]]:
        """(why the reference itself cannot process an H x W image, or None; the (h, w) token grid of every stage up
        to the one that fails)."""
        grids: List[Tuple[int, int]] = []
        for i, (pe, t1, peg, _) in enumerate(self.stages()):
            p = pe.patch_size
            if H % p or W % p or H < p or W < p:
                return f"stage {i + 1}: a {H} x {W} map is not divisible by patch_size={p}", grids
            H, W = H // p, W // p
            grids.append((H, W))
            local, _, glob, _ = t1.layers[0]
            if not isinstance(local, nn.Identity) and (H % local.fn.patch_size or W % local.fn.patch_size):
                return (f"stage {i + 1}: the {H} x {W} grid is not divisible by "
                        f"local_patch_size={local.fn.patch_size}"), grids
            k = glob.fn.to_kv.kernel_size[0]
            if min(H, W) < k:
                return f"stage {i + 1}: the {H} x {W} grid is smaller than global_k={k}", grids
            if peg.proj.fn.kernel_size[0] % 2 == 0:
                return f"peg_kernel_size={peg.proj.fn.kernel_size[0]} is even (the reference's residual add fails)", grids
        return None, grids

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4 or img.shape[1] != 3:
            return "input is not (B, 3, H, W)"
        encoders = [t for s in self.stages() for t in (s[1], s[3])]
        r = common_reason(self, img, encoders=encoders, dropout_p=self._dropout_p)
        if r is not None:
            return r
        r, grids = self.stage_reason(img.shape[2], img.shape[3])
        if r is not None:
            return r
        k = self.layers[0][2].proj.fn.kernel_size[0]
        if k not in PEG_KERNEL_SIZES:
            return f"peg_kernel_size={k} (the positional-encoding kernel is built for 1, 3, 5 and 7)"
        # a map has at most 16384 tokens (unsupported_reason) and never more keys than tokens, which is
        # b200vit_attention_kv's limit
        for (_, t1, _, t2), (h, w) in zip(self.stages(), grids):
            for t in (t1, t2):
                r = t.engine().unsupported_reason(h * w, grid=(h, w))
                if r is not None:
                    return r
        return None

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, x: torch.Tensor) -> torch.Tensor:
        return self.layers(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def _merge_weights(self, i: int, pe: PatchEmbedding) -> dict:
        return cached(self, f"_merge{i}", list(pe.parameters()), lambda: merge_weights(pe))

    def _peg_weights(self, i: int, peg: PEG) -> dict:
        return cached(self, f"_peg{i}", list(peg.parameters()), lambda: peg_weights(peg))

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev, bf = img.device, dict(device=img.device, dtype=torch.bfloat16)
        B, _, h, w = img.shape
        x = None
        for i, (pe, t1, peg, t2) in enumerate(self.stages()):
            # PatchEmbedding: merged and normalised patches -> 1 x 1 convolution GEMM -> LayerNorm into the stream
            m, p = self._merge_weights(i, pe), pe.patch_size
            h, w = h // p, w // p
            M, D = B * h * w, pe.dim_out
            a = torch.empty(M, m["kp"], **bf)
            if i == 0:
                _lib.patchify_ln(img.contiguous(), m["g"], m["b"], a, p, p, eps=pe.proj[0].eps)
            else:
                _lib.merge_patches_ln(x, m["g"], m["b"], a, B, h * p, w * p, p, eps=pe.proj[0].eps)
            y = torch.empty(M, D, device=dev, dtype=torch.float32)
            _lib.gemm(a, m["w"], out_f32=y, bias=m["bias"])
            t2.engine().share_workspace(t1.engine())      # same shapes, never running at the same time
            xb, stats = t1.engine().entry_buffers(M, dev)
            x = torch.empty(M, D, device=dev, dtype=torch.float32)
            _lib.embed_tokens(y, m["g2"], m["b2"], None, None, x, B, h * w, 0, eps=pe.proj[2].eps, xb=xb, stats=stats)
            t1.engine().run_blocks(x, B, h * w, primed=xb is not None, grid=(h, w))
            # PEG out of place (every token reads its neighbours), then the second Transformer's entry buffers
            pw = self._peg_weights(i, peg)
            x2 = torch.empty_like(x)
            _lib.peg(x, pw["w"], pw["b"], x2, B, h, w, peg.proj.fn.kernel_size[0])
            x = x2
            xb, stats = t2.engine().entry_buffers(M, dev)
            if xb is not None:
                _lib.rowstats_cast(x, xb, stats)
            t2.engine().run_blocks(x, B, h * w, primed=xb is not None, grid=(h, w))
        # head: mean over the last map, then the classifier GEMM
        D = x.shape[1]
        pm = torch.empty(B, D, device=dev, dtype=torch.float32)
        _lib.mean_pool(x, pm, B, h * w, D)
        pooled = torch.empty(B, D, **bf)
        _lib.cast_f32_bf16(pm, pooled)
        return head_engine(self, self.layers[6]).run(pooled)
