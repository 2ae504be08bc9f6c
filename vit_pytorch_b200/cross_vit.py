"""Drop-in `CrossViT` for lucidrains/vit-pytorch's `vit_pytorch.cross_vit.CrossViT`, with `ImageEmbedder`,
`MultiScaleEncoder`, `CrossTransformer`, `ProjectInOut`, `Transformer`, `Attention` and `FeedForward` of the same
file, and a fused sm_90a forward.

Same constructor keywords and defaults, parameter names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed): `sm_image_embedder.{to_patch_embedding.{1,2,3}, pos_embedding (1, n + 1,
dim), cls_token (1, 1, dim)}`, `multi_scale_encoder.layers.i.{0,1}` (branch Transformers: `layers` before `norm`),
`multi_scale_encoder.layers.i.2.layers.j.{0,1}.{fn, project_in, project_out}`, `sm_mlp_head`, `lg_mlp_head` (reference
cross_vit.py:18-270).  The PyTorch graph below mirrors the reference module for module, so hooks on any submodule keep
working there.

Fused forward (engine.py):
  * both ImageEmbedders: PatchEmbedEngine (16 x 16 patches: b200vit_patch_embed_tma; other sizes: patchify_ln + GEMM),
    then b200vit_embed_tokens with the cls row and the first n + 1 rows of the positional table (cross_vit.py:192-200);
  * every multi-scale block: each branch's encoder layers (TransformerEngine; the stages of one branch share one
    workspace), its final LayerNorm written back as the new stream, then both class-token cross-attention directions
    (CrossAttentionEngine, b200vit_attention_cls; cross_vit.py:121-130,157-162);
  * heads: LayerNorm of each stream's cls rows (row_index), sm head GEMM to fp32 logits, lg head GEMM adding them as
    its residual (cross_vit.py:265-270).
A hook on `multi_scale_encoder` itself (Extractor(v, layer_name='multi_scale_encoder')) keeps the call fused: the
embedded bf16 tokens then pass through that module call.  Hooks strictly inside the model run the PyTorch graph.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .engine import (CrossAttentionEngine, CrossLayer, FusedWeightsMixin, Norm, _bf16_rows, _f32, _has_hooks, cached,
                     cls_row_index, common_reason, fused_two_streams, head_width_reason, hooks_inside, on_device,
                     patch_engine, why_not_fused)
from .vit import FeedForward, FusedTransformer, Patchify

__all__ = ["Attention", "CrossTransformer", "CrossViT", "FeedForward", "ImageEmbedder", "MultiScaleEncoder",
           "ProjectInOut", "Transformer"]


class Attention(nn.Module):
    """Pre-LN multi-head attention with separate to_q / to_kv; cross attention when `context` is given, the normalised
    query tokens prepended to it with kv_include_self (reference cross_vit.py:34-71)."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, dropout: float = 0.) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.norm = nn.LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim, inner_dim * 2, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout))

    def forward(self, x: torch.Tensor, context: Optional[torch.Tensor] = None,
                kv_include_self: bool = False) -> torch.Tensor:
        b, n, _ = x.shape
        h = self.heads
        x = self.norm(x)
        context = x if context is None else context
        if kv_include_self:
            context = torch.cat((x, context), dim=1)
        k, v = self.to_kv(context).chunk(2, dim=-1)
        q, k, v = (t.reshape(b, t.shape[1], h, -1).transpose(1, 2) for t in (self.to_q(x), k, v))
        dots = torch.matmul(q, k.transpose(-1, -2)) * self.scale
        attn = self.dropout(self.attend(dots))
        out = torch.matmul(attn, v).transpose(1, 2).reshape(b, n, -1)
        return self.to_out(out)


class Transformer(FusedTransformer):
    """depth x (Attention, FeedForward) residual blocks + final LayerNorm (reference cross_vit.py:75-90): one branch
    encoder of a multi-scale block.  Callable on arbitrary (B, N, D) tokens; runs fused when eligible."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.) -> None:
        super().__init__()
        self.dropout_p = float(dropout)
        self.layers = nn.ModuleList([])
        self.norm = nn.LayerNorm(dim)
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))

    @staticmethod
    def qkv_weight(attn: nn.Module) -> torch.Tensor:
        return torch.cat([attn.to_q.weight, attn.to_kv.weight], dim=0)     # rows q | k | v


class ProjectInOut(nn.Module):
    """fn between Linear projections into and back out of another width, Identity when the widths match (reference
    cross_vit.py:94-107)."""

    def __init__(self, dim_in: int, dim_out: int, fn: nn.Module) -> None:
        super().__init__()
        self.fn = fn
        need_projection = dim_in != dim_out
        self.project_in = nn.Linear(dim_in, dim_out) if need_projection else nn.Identity()
        self.project_out = nn.Linear(dim_out, dim_in) if need_projection else nn.Identity()

    def forward(self, x: torch.Tensor, *args, **kwargs) -> torch.Tensor:
        x = self.project_in(x)
        x = self.fn(x, *args, **kwargs)
        return self.project_out(x)


def _linear(m: nn.Module) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
    return None if isinstance(m, nn.Identity) else (m.weight, m.bias)


class CrossTransformer(nn.Module):
    """depth x (sm cls attends to lg patches, lg cls attends to sm patches) (reference cross_vit.py:111-130)."""

    def __init__(self, sm_dim: int, lg_dim: int, depth: int, heads: int, dim_head: int, dropout: float) -> None:
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                ProjectInOut(sm_dim, lg_dim, Attention(lg_dim, heads=heads, dim_head=dim_head, dropout=dropout)),
                ProjectInOut(lg_dim, sm_dim, Attention(sm_dim, heads=heads, dim_head=dim_head, dropout=dropout)),
            ]))
        self._cross_engines: Optional[Tuple[CrossAttentionEngine, CrossAttentionEngine]] = None

    def forward(self, sm_tokens: torch.Tensor, lg_tokens: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        (sm_cls, sm_patch_tokens), (lg_cls, lg_patch_tokens) = ((t[:, :1], t[:, 1:]) for t in (sm_tokens, lg_tokens))
        for sm_attend_lg, lg_attend_sm in self.layers:
            sm_cls = sm_attend_lg(sm_cls, context=lg_patch_tokens, kv_include_self=True) + sm_cls
            lg_cls = lg_attend_sm(lg_cls, context=sm_patch_tokens, kv_include_self=True) + lg_cls
        sm_tokens = torch.cat((sm_cls, sm_patch_tokens), dim=1)
        lg_tokens = torch.cat((lg_cls, lg_patch_tokens), dim=1)
        return sm_tokens, lg_tokens

    # ---------------------------------------------------------------------------------------------- fused kernels
    def cross_params(self, direction: int) -> List[torch.Tensor]:
        """Parameters of direction 0 (sm cls attends to lg) or 1 (lg cls attends to sm)."""
        return [p for layer in self.layers for p in layer[direction].parameters()]

    def cross_layers(self, direction: int) -> List[CrossLayer]:
        out = []
        for layer in self.layers:
            pio = layer[direction]
            a = pio.fn
            out.append(CrossLayer(
                proj_in=_linear(pio.project_in), ln=Norm.of(a.norm), q_w=a.to_q.weight, kv_w=a.to_kv.weight,
                out_w=a.to_out[0].weight, out_b=a.to_out[0].bias, proj_out=_linear(pio.project_out),
                heads=a.heads, dim_head=a.dim_head, scale=float(a.scale)))
        return out

    def engines(self) -> Tuple[CrossAttentionEngine, CrossAttentionEngine]:
        if self._cross_engines is None:
            self._cross_engines = (CrossAttentionEngine(self, 0), CrossAttentionEngine(self, 1))
        return self._cross_engines


class MultiScaleEncoder(nn.Module):
    """depth x (sm Transformer, lg Transformer, CrossTransformer) on two token streams (reference cross_vit.py:134-162).
    Callable on bf16 CUDA tokens (B, N_sm, sm_dim), (B, N_lg, lg_dim); runs fused when eligible."""

    def __init__(self, *, depth, sm_dim, lg_dim, sm_enc_params, lg_enc_params, cross_attn_heads, cross_attn_depth,
                 cross_attn_dim_head=64, dropout=0.) -> None:
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Transformer(dim=sm_dim, dropout=dropout, **sm_enc_params),
                Transformer(dim=lg_dim, dropout=dropout, **lg_enc_params),
                CrossTransformer(sm_dim=sm_dim, lg_dim=lg_dim, depth=cross_attn_depth, heads=cross_attn_heads,
                                 dim_head=cross_attn_dim_head, dropout=dropout),
            ]))
        self.dropout_p = float(dropout)
        self._rows: dict = {}

    def forward_eager(self, sm_tokens: torch.Tensor, lg_tokens: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        for sm_enc, lg_enc, cross_attend in self.layers:
            sm_tokens, lg_tokens = sm_enc(sm_tokens), lg_enc(lg_tokens)
            sm_tokens, lg_tokens = cross_attend(sm_tokens, lg_tokens)
        return sm_tokens, lg_tokens

    def forward(self, sm_tokens: torch.Tensor, lg_tokens: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        if self.fused_reason(sm_tokens, lg_tokens) is None:
            with on_device(sm_tokens):
                return self.forward_fused(sm_tokens, lg_tokens)
        return self.forward_eager(sm_tokens, lg_tokens)

    # ---------------------------------------------------------------------------------------------- dispatch
    def shape_reason(self, n_sm: int, n_lg: int) -> Optional[str]:
        """None if the kernels cover streams of n_sm and n_lg tokens (cls included) through this encoder."""
        if len(self.layers) == 0:
            return "depth == 0"
        sm_enc, lg_enc, cross = self.layers[0]
        if len(sm_enc.layers) == 0 or len(lg_enc.layers) == 0 or len(cross.layers) == 0:
            return "an encoder or cross-attention depth of 0"
        r = head_width_reason(cross.layers[0][0].fn.dim_head)
        if r is not None:
            return "cross attention " + r
        for name, enc, n in (("sm", sm_enc, n_sm), ("lg", lg_enc, n_lg)):
            r = enc.engine().unsupported_reason(n)
            if r is not None:
                return f"{name} encoder: {r}"
        return None

    def fused_reason(self, sm_tokens: torch.Tensor, lg_tokens: torch.Tensor) -> Optional[str]:
        """None if forward(sm_tokens, lg_tokens) will run the fused kernels, else why not."""
        r = why_not_fused(list(self.parameters()), sm_tokens, training=self.training, dropout_p=self.dropout_p)
        if r is None:
            r = why_not_fused([], lg_tokens, training=self.training, dropout_p=self.dropout_p)
        if r is None and (lg_tokens.device != sm_tokens.device):
            r = "sm and lg tokens on different devices"
        if r is None and hooks_inside(self):
            r = "forward hooks registered inside the model"
        if r is not None:
            return r
        if sm_tokens.dim() != 3 or lg_tokens.dim() != 3 or sm_tokens.shape[0] != lg_tokens.shape[0]:
            return "tokens are not (B, N, D) with one batch size"
        sm_enc, lg_enc, _ = self.layers[0] if len(self.layers) else (None, None, None)
        if sm_enc is not None and (sm_tokens.shape[2] != sm_enc.norm.normalized_shape[0]
                                   or lg_tokens.shape[2] != lg_enc.norm.normalized_shape[0]):
            return "token width differs from the encoder's"
        if sm_tokens.shape[1] < 1 or lg_tokens.shape[1] < 1:
            return "a stream without a cls token"
        return self.shape_reason(sm_tokens.shape[1], lg_tokens.shape[1])

    # ---------------------------------------------------------------------------------------------- fused kernels
    def stages(self) -> list:
        """(sm TransformerEngine, lg TransformerEngine, sm->lg and lg->sm CrossAttentionEngine) per block; the branch
        engines of later blocks run on the first block's workspaces (one per branch, not one per block)."""
        out = []
        for sm_enc, lg_enc, cross in self.layers:
            es, el = sm_enc.engine(), lg_enc.engine()
            if out:
                es.share_workspace(out[0][0])
                el.share_workspace(out[0][1])
            out.append((es, el) + cross.engines())
        return out

    def cls_rows(self, B: int, n_sm: int, n_lg: int, device) -> Tuple[torch.Tensor, torch.Tensor]:
        return cls_row_index(self._rows, B, n_sm, device), cls_row_index(self._rows, B, n_lg, device)

    def run_streams(self, xs: torch.Tensor, xl: torch.Tensor, B: int, n_sm: int, n_lg: int, primed: bool):
        """The whole encoder on fp32 streams xs [B*n_sm, sm_dim], xl [B*n_lg, lg_dim] (engine.fused_two_streams)."""
        return fused_two_streams(self.stages(), xs, xl, B, n_sm, n_lg, primed,
                                 self.cls_rows(B, n_sm, n_lg, xs.device))

    def forward_fused(self, sm_tokens: torch.Tensor, lg_tokens: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        B, Ns, Ds = sm_tokens.shape
        Nl, Dl = lg_tokens.shape[1:]
        xs = sm_tokens.reshape(B * Ns, Ds).float().contiguous()
        xl = lg_tokens.reshape(B * Nl, Dl).float().contiguous()
        x, _ = self.run_streams(xs, xl, B, Ns, Nl, primed=False)
        outs = []
        for xf, n, d in ((x[0], Ns, Ds), (x[1], Nl, Dl)):
            o = torch.empty(B, n, d, device=xf.device, dtype=torch.bfloat16)
            _lib.cast_f32_bf16(xf.view(-1), o.view(-1))
            outs.append(o)
        return outs[0], outs[1]


class ImageEmbedder(nn.Module):
    """'(p1 p2 c)' patches -> LayerNorm -> Linear -> LayerNorm, cls token, positional table (reference
    cross_vit.py:166-200)."""

    def __init__(self, *, dim, image_size, patch_size, dropout=0., channels=3) -> None:
        super().__init__()
        assert image_size % patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        num_patches = (image_size // patch_size) ** 2
        patch_dim = channels * patch_size ** 2
        self.patch_size = (patch_size, patch_size)
        self.to_patch_embedding = nn.Sequential(
            Patchify(patch_size, patch_size),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.pos_embedding = nn.Parameter(torch.randn(1, num_patches + 1, dim))
        self.cls_token = nn.Parameter(torch.randn(1, 1, dim))
        self.dropout = nn.Dropout(dropout)

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        x = self.to_patch_embedding(img)
        b, n, _ = x.shape
        cls_tokens = self.cls_token.expand(b, -1, -1)
        x = torch.cat((cls_tokens, x), dim=1)
        x += self.pos_embedding[:, :(n + 1)]
        return self.dropout(x)

    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """The shape checks of the fused embedding (device, dtype and dropout are the caller's)."""
        p = self.patch_size[0]
        if img.shape[1] * p * p != self.to_patch_embedding[1].normalized_shape[0]:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        if img.shape[2] % p or img.shape[3] % p:
            return "image not divisible by the patch size"
        n = (img.shape[2] // p) * (img.shape[3] // p)
        if n + 1 > self.pos_embedding.shape[1]:
            return f"{n + 1} tokens exceed the positional table ({self.pos_embedding.shape[1]})"
        return None

    def tokens(self, img: torch.Tensor) -> int:
        return (img.shape[2] // self.patch_size[0]) * (img.shape[3] // self.patch_size[1]) + 1

    def embed_fused(self, img: torch.Tensor, xb: Optional[torch.Tensor] = None,
                    stats: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, int, int]:
        """img bf16 [B, C, H, W] -> (x fp32 [B*(n+1), dim], B, n + 1); optionally also the bf16 copy and row sums."""
        pe = patch_engine(self)
        pos = pe.prepared(img.device)["pos"].view(-1, self.pos_embedding.shape[-1])
        return pe.run(img, xb=xb, stats=stats, pos=pos)


class CrossViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, num_classes, sm_dim, lg_dim, sm_patch_size=12, sm_enc_depth=1, sm_enc_heads=8,
                 sm_enc_mlp_dim=2048, sm_enc_dim_head=64, lg_patch_size=16, lg_enc_depth=4, lg_enc_heads=8,
                 lg_enc_mlp_dim=2048, lg_enc_dim_head=64, cross_attn_depth=2, cross_attn_heads=8,
                 cross_attn_dim_head=64, depth=3, dropout=0.1, emb_dropout=0.1, channels=3) -> None:
        super().__init__()
        self.sm_image_embedder = ImageEmbedder(dim=sm_dim, channels=channels, image_size=image_size,
                                               patch_size=sm_patch_size, dropout=emb_dropout)
        self.lg_image_embedder = ImageEmbedder(dim=lg_dim, channels=channels, image_size=image_size,
                                               patch_size=lg_patch_size, dropout=emb_dropout)
        self.multi_scale_encoder = MultiScaleEncoder(
            depth=depth,
            sm_dim=sm_dim,
            lg_dim=lg_dim,
            cross_attn_heads=cross_attn_heads,
            cross_attn_dim_head=cross_attn_dim_head,
            cross_attn_depth=cross_attn_depth,
            sm_enc_params=dict(depth=sm_enc_depth, heads=sm_enc_heads, mlp_dim=sm_enc_mlp_dim,
                               dim_head=sm_enc_dim_head),
            lg_enc_params=dict(depth=lg_enc_depth, heads=lg_enc_heads, mlp_dim=lg_enc_mlp_dim,
                               dim_head=lg_enc_dim_head),
            dropout=dropout,
        )
        self.sm_mlp_head = nn.Sequential(nn.LayerNorm(sm_dim), nn.Linear(sm_dim, num_classes))
        self.lg_mlp_head = nn.Sequential(nn.LayerNorm(lg_dim), nn.Linear(lg_dim, num_classes))

        self._emb_dropout_p = float(emb_dropout)

    # ---------------------------------------------------------------------------------------------- dispatch
    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        se, le, mse = self.sm_image_embedder, self.lg_image_embedder, self.multi_scale_encoder
        r = common_reason(self, img, dropout_p=max(self._emb_dropout_p, mse.dropout_p), skip=(mse,))
        for name, emb in (("sm", se), ("lg", le)):
            if r is None:
                r = emb.fused_reason(img)
                r = None if r is None else f"{name} embedder: {r}"
        if r is None:
            r = mse.shape_reason(se.tokens(img), le.tokens(img))
        return r

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        if self.fused_reason(img) is None:
            with on_device(img):
                return self.forward_fused(img)
        return self.forward_eager(img)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, img: torch.Tensor) -> torch.Tensor:
        sm_tokens = self.sm_image_embedder(img)
        lg_tokens = self.lg_image_embedder(img)
        sm_tokens, lg_tokens = self.multi_scale_encoder(sm_tokens, lg_tokens)
        sm_cls, lg_cls = (t[:, 0] for t in (sm_tokens, lg_tokens))
        sm_logits = self.sm_mlp_head(sm_cls)
        lg_logits = self.lg_mlp_head(lg_cls)
        return sm_logits + lg_logits

    # ---------------------------------------------------------------------------------------------- fused kernels
    def _head_weights(self) -> dict:
        heads = (("sm", self.sm_mlp_head), ("lg", self.lg_mlp_head))
        build = lambda: {name: (_f32(h[0].weight), _f32(h[0].bias), h[0].eps, _bf16_rows(h[1].weight),   # noqa: E731
                                _f32(h[1].bias)) for name, h in heads}
        return cached(self, "_heads", [p for _, h in heads for p in h.parameters()], build)

    def forward_fused(self, img: torch.Tensor) -> torch.Tensor:
        se, le, mse = self.sm_image_embedder, self.lg_image_embedder, self.multi_scale_encoder
        B, dev = img.shape[0], img.device
        if _has_hooks(mse):                            # Extractor(v, layer_name='multi_scale_encoder')
            streams = []
            for emb in (se, le):
                x, _, N = emb.embed_fused(img)
                tok = torch.empty(B, N, x.shape[1], device=dev, dtype=torch.bfloat16)
                _lib.cast_f32_bf16(x.view(-1), tok.view(-1))
                streams.append(tok)
            outs = mse(*streams)
            x = [o.reshape(-1, o.shape[-1]).float().contiguous() for o in outs]
            rows = mse.cls_rows(B, outs[0].shape[1], outs[1].shape[1], dev)
        else:
            stages = mse.stages()
            Ns, Nl = se.tokens(img), le.tokens(img)
            xbs, sts = stages[0][0].entry_buffers(B * Ns, dev)
            xbl, stl = stages[0][1].entry_buffers(B * Nl, dev)
            xs, _, _ = se.embed_fused(img, xb=xbs, stats=sts)
            xl, _, _ = le.embed_fused(img, xb=xbl, stats=stl)
            rows = mse.cls_rows(B, Ns, Nl, dev)
            x, _ = fused_two_streams(stages, xs, xl, B, Ns, Nl, xbs is not None, rows)
        heads = self._head_weights()
        nc = heads["sm"][3].shape[0]
        ncp = (nc + 7) // 8 * 8                        # residual row stride: a multiple of 4 (and of 8 for bf16)
        logits = torch.empty(B, ncp, device=dev, dtype=torch.float32)
        out = torch.empty(B, ncp, device=dev, dtype=torch.bfloat16)
        for i, name in enumerate(("sm", "lg")):
            g, b, eps, w, bias = heads[name]
            pooled = torch.empty(B, x[i].shape[1], device=dev, dtype=torch.bfloat16)
            _lib.layernorm(x[i], g, b, out_bf16=pooled, row_index=rows[i], eps=eps)
            if i == 0:
                _lib.gemm(pooled, w, out_f32=logits, bias=bias)
            else:                                      # sm_logits + lg_logits, added in fp32
                _lib.gemm(pooled, w, out_f32=logits, out_bf16=out, bias=bias, resid=logits)
        return out[:, :nc]
