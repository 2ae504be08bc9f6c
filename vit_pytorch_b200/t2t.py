"""Drop-in `T2TViT` for lucidrains/vit-pytorch's `vit_pytorch.t2t.T2TViT` (Tokens-to-Token ViT), with `RearrangeImage`
and `conv_output_size` of the same file, and a fused sm_90a forward.

Same constructor keywords, parameter names / shapes / registration order (=> identical `state_dict` and identical
random init under the same seed): `to_patch_embedding` one nn.Sequential of four modules per soft split -- RearrangeImage
(nn.Identity in the first), nn.Unfold(k, stride=s, padding=s // 2), the transpose, and vit.Transformer(dim=w, heads=1,
depth=1, dim_head=w, mlp_dim=w) with w = channels * (k1 * ... * k)^2 (nn.Identity in the last) -- then
Linear(w_last, dim); `pos_embedding` (1, conv_output_size(...)^2 + 1, dim), `cls_token`, `transformer`, `mlp_head`
(reference t2t.py:26-62).  The PyTorch graph below mirrors the reference module for module, including RearrangeImage's
`int(sqrt(n))` rule, so hooks on any submodule keep working there.

Fused forward (no host synchronisation: graph.GraphedForward captures it):
  * per soft split: b200vit_t2t_unfold_image (first) or b200vit_t2t_unfold_tokens (later) writing the soft-split
    Transformer's fp32 residual stream x[B*n, round8(w)] (or, last, the bf16 A operand of the final Linear); then its
    one layer, driven from here (soft_split_layer): the shape occurs in no other family;
  * Linear(w_last, dim) as one GEMM (K = w_last, the padding of its rows never read), b200vit_embed_tokens without a
    LayerNorm (cls row, positional rows :n + 1), the main encoder through its TransformerEngine (run_blocks, pool) and
    the head GEMM (t2t.py:64-80).
A soft-split layer (vit.py Transformer, depth 1, then its final LayerNorm) on the stream x[M, W8], W8 = round8(w):
    xa  = LN1(x[:, :w])                     b200vit_layernorm (statistics over the true w)
    qkv = xa Wqkv'^T                         GEMM, K = w; q | k | v each padded to dp by zero rows of Wqkv'
    x  += bf16(softmax(q k^T w^-0.5) v)      dp <= 160: b200vit_attention_varlen at dp in (32, 64, 80, 128, 160), then
                                             the residual GEMM with an identity weight (to_out is nn.Identity);
                                             wider: b200vit_attention_wide, whose P V epilogue adds into x itself
    h   = GELU(LN2(x) W1'^T + b1)            b200vit_layernorm, GEMM (K = w, N = W8 with zero rows and bias)
    x  += h W2'^T + b2                       residual GEMM (K = w; rows past w and their bias zero: x's padding stays 0)
    y   = LN(x[:, :w])                       b200vit_layernorm -> the bf16 token rows the next soft split reads
B200VIT_LN_MODE applies to the main encoder only: the soft-split LayerNorms always run as b200vit_layernorm, since
their GEMMs' K is not the LayerNorm's width.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import FusedWeightsMixin, _bf16_rows, _f32, cached, classify, common_reason, on_device
from .pit import _Transpose, pool_grid
from .vit import Transformer

__all__ = ["RearrangeImage", "T2TViT", "conv_output_size", "soft_split_width"]

# the head widths b200vit_attention_varlen is built for; a soft-split head up to 160 wide runs at the next of them
NARROW_WIDTHS = (32, 64, 80, 128, 160)


def exists(val):
    return val is not None


def conv_output_size(image_size, kernel_size, stride, padding):
    return int(((image_size - kernel_size + (2 * padding)) / stride) + 1)


def round8(n: int) -> int:
    return (n + 7) // 8 * 8


def soft_split_width(w: int) -> int:
    """The attention width dp a soft-split head w wide runs at: the next built varlen width up to 160, else w rounded
    up to 64 (b200vit_attention_wide)."""
    for d in NARROW_WIDTHS:
        if w <= d:
            return d
    return (w + 63) // 64 * 64


class RearrangeImage(nn.Module):
    """rearrange(x, 'b (h w) c -> b c h w', h = int(sqrt(n))) (reference t2t.py:20-22), without einops; the map is
    PiT's Pool grid rule (pit.pool_grid).  The transpose after each Unfold (t2t.py:39) is pit._Transpose."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b, n, c = x.shape
        g = pool_grid(n)
        if g is None:
            # what einops raises for an h that does not divide n
            raise RuntimeError(f"RearrangeImage: {n} tokens cannot be read as a map of {int(math.sqrt(n))} rows "
                               "(t2t.py:22)")
        return x.reshape(b, g[0], g[1], c).permute(0, 3, 1, 2)


class T2TViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, num_classes, dim, depth=None, heads=None, mlp_dim=None, pool='cls', channels=3,
                 dim_head=64, dropout=0., emb_dropout=0., transformer=None, t2t_layers=((7, 4), (3, 2), (3, 2))
                 ) -> None:
        super().__init__()
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'

        layers = []
        layer_dim = channels
        output_image_size = image_size

        for i, (kernel_size, stride) in enumerate(t2t_layers):
            layer_dim *= kernel_size ** 2
            is_first = i == 0
            is_last = i == (len(t2t_layers) - 1)
            output_image_size = conv_output_size(output_image_size, kernel_size, stride, stride // 2)

            layers.extend([
                RearrangeImage() if not is_first else nn.Identity(),
                nn.Unfold(kernel_size=kernel_size, stride=stride, padding=stride // 2),
                _Transpose(),
                Transformer(dim=layer_dim, heads=1, depth=1, dim_head=layer_dim, mlp_dim=layer_dim,
                            dropout=dropout) if not is_last else nn.Identity(),
            ])

        layers.append(nn.Linear(layer_dim, dim))
        self.to_patch_embedding = nn.Sequential(*layers)

        self.pos_embedding = nn.Parameter(torch.randn(1, output_image_size ** 2 + 1, dim))
        self.cls_token = nn.Parameter(torch.randn(1, 1, dim))
        self.dropout = nn.Dropout(emb_dropout)

        if not exists(transformer):
            assert all([exists(depth), exists(heads), exists(mlp_dim)]), 'depth, heads, and mlp_dim must be supplied'
            self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim, dropout)
        else:
            self.transformer = transformer

        self.pool = pool
        self.to_latent = nn.Identity()

        self.mlp_head = nn.Linear(dim, num_classes)

        self.t2t_layers = tuple(tuple(kv) for kv in t2t_layers)
        self.channels = channels
        self._emb_dropout_p = float(emb_dropout)
        self._cu: dict = {}

    def soft_splits(self) -> List[Optional[Transformer]]:
        """The soft-split Transformer of every stage (None in the last, whose slot holds nn.Identity)."""
        mods = list(self.to_patch_embedding)
        return [mods[4 * i + 3] if isinstance(mods[4 * i + 3], Transformer) else None
                for i in range(len(self.t2t_layers))]

    # ---------------------------------------------------------------------------------------------- dispatch
    def stage_geometry(self, H: int, W: int) -> Optional[List[Tuple[int, int, int, int]]]:
        """(source map h, w, unfold grid oh, ow) of every soft split for an H x W image, in order; None where the
        reference raises: a map the int(sqrt(n)) rule cannot read, or one smaller than the unfold window."""
        out = []
        h, w = H, W
        for i, (k, s) in enumerate(self.t2t_layers):
            if i > 0:
                g = pool_grid(out[-1][2] * out[-1][3])
                if g is None:
                    return None
                h, w = g
            p = s // 2
            if h + 2 * p < k or w + 2 * p < k:
                return None
            out.append((h, w, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1))
        return out

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        if img.shape[1] != self.channels:
            return "channel count differs from the constructor's (the reference's Transformer raises)"
        if not isinstance(self.transformer, Transformer):
            return "transformer= is not this package's vit.Transformer"
        if any(s // 2 >= k for k, s in self.t2t_layers):
            return "a soft split whose padding stride // 2 is not below its kernel size"
        splits = [t for t in self.soft_splits() if t is not None]
        r = common_reason(self, img, encoders=[self.transformer] + splits,
                          dropout_p=max([self._emb_dropout_p, self.transformer.dropout_p] +
                                        [t.dropout_p for t in splits]))
        if r is not None:
            return r
        geo = self.stage_geometry(img.shape[2], img.shape[3])
        if geo is None:
            return "a soft split's token map cannot be read by the reference's int(sqrt(n)) rule or is smaller " \
                   "than its window"
        n = geo[-1][2] * geo[-1][3]
        if n + 1 > self.pos_embedding.shape[1]:
            return f"{n + 1} tokens exceed the positional table ({self.pos_embedding.shape[1]})"
        for t, (_, _, oh, ow) in zip(self.soft_splits(), geo):
            if t is None:
                continue
            w = t.layers[0][0].to_qkv.in_features
            dp = soft_split_width(w)
            if dp > 160 and oh * ow > _lib.ATTN_WIDE_MAX_TOKENS:
                return f"a soft split {w} wide over {oh * ow} tokens (the wide attention kernel takes at most " \
                       f"{_lib.ATTN_WIDE_MAX_TOKENS})"
            if dp > _lib.ATTN_WIDE_MAX_WIDTH:
                return f"a soft split {w} wide (the wide attention kernel takes at most {_lib.ATTN_WIDE_MAX_WIDTH})"
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
        x += self.pos_embedding[:, :n + 1]
        x = self.dropout(x)

        x = self.transformer(x)

        x = x.mean(dim=1) if self.pool == 'mean' else x[:, 0]

        x = self.to_latent(x)
        return self.mlp_head(x)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def _split_weights(self, i: int, t: Transformer) -> dict:
        return cached(self, f"_split{i}", list(t.parameters()), lambda: split_weights(t))

    def _embed_weights(self) -> dict:
        lin = self.to_patch_embedding[-1]
        params = [lin.weight, lin.bias, self.pos_embedding, self.cls_token]

        def build():
            D = lin.out_features
            return {"w": _bf16_rows(lin.weight, round8(lin.in_features)), "b": _f32(lin.bias),
                    "pos": self.pos_embedding.detach().float().reshape(-1, D).contiguous(),
                    "cls": self.cls_token.detach().float().reshape(1, D).contiguous()}
        return cached(self, "_embed", params, build)

    def _varlen(self, B: int, n: int, device: torch.device):
        """(cu_seqlens, tile_prefix, total_tiles) of B images of n tokens, made once per shape (no host-to-device copy
        inside a captured forward)."""
        key = (B, n, str(device))
        if key not in self._cu:
            self._cu[key] = _lib.varlen_index([n] * B, device)
        return self._cu[key]

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        dev = img.device
        B, C = img.shape[0], img.shape[1]
        geo = self.stage_geometry(img.shape[2], img.shape[3])
        splits = self.soft_splits()
        src, width = img.contiguous(), C
        for i, ((k, s), t, (mh, mw, oh, ow)) in enumerate(zip(self.t2t_layers, splits, geo)):
            w = width * k * k
            n = oh * ow
            out = torch.empty(B * n, round8(w), device=dev, dtype=torch.float32 if t is not None else torch.bfloat16)
            if i == 0:
                _lib.t2t_unfold_image(src, out, k, s, s // 2)
            else:
                _lib.t2t_unfold_tokens(src[:, :width], (mh, mw), out, k, s, s // 2)
            if t is not None:
                src = soft_split_layer(self._split_weights(i, t), out, B, n, self._varlen(B, n, dev))
            else:
                src = out
            width = w
        # Linear(w_last, dim) -> cls row and positions -> main encoder -> pool -> head
        e = self._embed_weights()
        D = e["w"].shape[0]
        y = torch.empty(B * n, D, device=dev, dtype=torch.float32)
        _lib.gemm(src, e["w"], out_f32=y, bias=e["b"], k=width)
        N = n + 1
        eng = self.transformer.engine()
        xb, stats = eng.entry_buffers(B * N, dev)
        x = torch.empty(B * N, D, device=dev, dtype=torch.float32)
        _lib.embed_tokens(y, None, None, e["cls"], e["pos"], x, B, n, 1, xb=xb, stats=stats)
        eng.run_blocks(x, B, N, primed=xb is not None)
        return classify(self, self.mlp_head, eng.pool(x, B, N, mean=self.pool == 'mean'))


def split_weights(t: Transformer) -> dict:
    """The prepared weights of a soft-split Transformer (vit.Transformer, depth 1, heads 1, dim_head = mlp_dim = dim
    = w), padded for soft_split_layer: W8 = round8(w) columns everywhere, the attention width dp = soft_split_width(w).
    'qkv' bf16 [3 dp, W8] (q | k | v, rows w .. dp of each zero), 'eye' bf16 [W8, W8] (dp <= 160 only: identity on the first
    w rows, the identity to_out as a residual GEMM), 'w1' / 'w2' bf16 [W8, W8] and 'b1' / 'b2' fp32 [W8] (rows and bias past w
    zero), the LayerNorm affines 'ln1', 'ln2', 'norm' as (gamma, beta, eps), 'w', 'dp', 'scale'."""
    attn, ff = t.layers[0]
    w = attn.to_qkv.in_features
    dp, W8 = soft_split_width(w), round8(w)
    dev = attn.to_qkv.weight.device
    qkv = torch.zeros(3 * dp, W8, device=dev, dtype=torch.bfloat16)
    wq = attn.to_qkv.weight.detach()
    for j in range(3):
        qkv[j * dp:j * dp + w, :w] = wq[j * w:(j + 1) * w]
    fc1, fc2 = [m for m in ff.net if isinstance(m, nn.Linear)]

    def square(lin: nn.Linear) -> Tuple[torch.Tensor, torch.Tensor]:
        m = torch.zeros(W8, W8, device=dev, dtype=torch.bfloat16)
        m[:w, :w] = lin.weight.detach()
        b = torch.zeros(W8, device=dev, dtype=torch.float32)
        b[:w] = lin.bias.detach().float()
        return m, b

    w1, b1 = square(fc1)
    w2, b2 = square(fc2)
    ln = lambda m: (_f32(m.weight), _f32(m.bias), float(m.eps))      # noqa: E731
    out = {"qkv": qkv, "w1": w1, "b1": b1, "w2": w2, "b2": b2, "ln1": ln(attn.norm),
            "ln2": ln(ff.net[0]), "norm": ln(t.norm), "w": w, "dp": dp, "scale": float(attn.scale)}
    if dp <= NARROW_WIDTHS[-1]:
        out["eye"] = torch.zeros(W8, W8, device=dev, dtype=torch.bfloat16)
        out["eye"][:w, :w] = torch.eye(w, device=dev, dtype=torch.bfloat16)
    return out


def soft_split_layer(t: dict, x: torch.Tensor, B: int, n: int, varlen) -> torch.Tensor:
    """One soft-split Transformer (t: split_weights) on its fp32 stream x[B*n, W8] (columns past w zero), in place;
    returns the bf16 rows [B*n, W8] of its final LayerNorm (columns past w unwritten: every reader takes w).
    Every GEMM here runs at K = w, which need not be a multiple of 8: b200vit_gemm_bf16 reads a K tail through TMA's
    zero fill (include/b200vit.h), so the padding columns of its operands are never read."""
    w, dp = t["w"], t["dp"]
    M, W8 = x.shape
    dev, bf = x.device, dict(device=x.device, dtype=torch.bfloat16)
    xt = x[:, :w]
    xa = torch.empty(M, W8, **bf)
    g, b, eps = t["ln1"]
    _lib.layernorm(xt, g, b, out_bf16=xa[:, :w], eps=eps)
    qkv = torch.empty(M, 3 * dp, **bf)
    _lib.gemm(xa, t["qkv"], out_bf16=qkv, k=w)
    if dp <= NARROW_WIDTHS[-1]:
        o = torch.empty(M, dp, **bf)
        cu, tp, tiles = varlen
        _lib.attention_varlen(qkv, o, cu, tp, tiles, 1, dp, t["scale"])
        _lib.gemm(o, t["eye"], out_f32=x, resid=x, k=w)
    else:
        images = max(1, min(B, (256 << 20) // _lib.attention_wide_workspace(n, dp, 1)))
        ws = torch.empty(_lib.attention_wide_workspace(n, dp, images), device=dev, dtype=torch.uint8)
        _lib.attention_wide(qkv, B, n, dp, t["scale"], ws, x=x, n_resid=w)
    g, b, eps = t["ln2"]
    _lib.layernorm(xt, g, b, out_bf16=xa[:, :w], eps=eps)
    h = torch.empty(M, W8, **bf)
    _lib.gemm(xa, t["w1"], out_bf16=h, bias=t["b1"], gelu=True, k=w)
    _lib.gemm(h, t["w2"], out_f32=x, resid=x, bias=t["b2"], k=w)
    y = torch.empty(M, W8, **bf)
    g, b, eps = t["norm"]
    _lib.layernorm(xt, g, b, out_bf16=y[:, :w], eps=eps)
    return y
