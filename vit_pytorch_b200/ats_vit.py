"""Drop-in `ViT` for lucidrains/vit-pytorch's `vit_pytorch.ats_vit.ViT` (Adaptive Token Sampling), with
`AdaptiveTokenSampling`, `Attention`, `FeedForward`, `Transformer`, `sample_gumbel` and `batched_index_select` of the same
file, and a fused sm_90a forward.

Same constructor keywords and asserts, parameter names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed): `to_patch_embedding` (Rearrange, LayerNorm(patch), Linear, LayerNorm(dim)),
`pos_embedding` (1, n + 1, dim), `cls_token` (1, 1, dim), `transformer.layers[i]` = (Attention with norm / attend /
dropout / to_qkv / ats / to_out, FeedForward), `mlp_head` (LayerNorm, Linear) (reference ats_vit.py:111-240).  The
PyTorch graph below mirrors the reference module for module, including its draws from torch's generator, so hooks on
any submodule keep working there.  `forward(img, return_sampled_token_ids=True)` returns (logits, ids[B, L_max - 1]):
each image's kept token indices (cls excluded), -1 for padding.

Fused forward (no host synchronisation unless the token ids are asked for: graph.GraphedForward captures it).  Every
image keeps a slot of S_l rows, S_0 = n + 1 and S_l = min(S_{l-1}, 1 + K_l) with K_l = max_tokens_per_depth[l]; its
valid length L_b and the token index of every row live on the device.
  * patch embedding and token assembly (PatchEmbedEngine);
  * the layers before the first that may sample (K_l < S_{l-1} - 1): plain ViT layers through the TransformerEngine;
  * a layer that may sample: LN1 + QKV on B*S_{l-1} rows; b200vit_ats_select (the device decides whether the layer
    samples, from the batch's padded length max_b L_b, as ats_vit.py:169 does) -> row map, new lengths and ids;
    b200vit_ats_gather of the kept rows' q and fp32 residual rows into the other stream buffer; b200vit_attention_kv_lens
    of the kept queries over each image's old valid keys; out-projection onto the new stream; feed-forward;
  * a later layer that cannot sample: the same without the selection, queries read in place;
  * LayerNorm + Linear of every image's row 0.
The engine's workspace is allocated once for B*(n + 1) rows; later layers run on row-prefix views of it.

Two deliberate differences from the reference in the fused path (the PyTorch graph has neither):
  * the uniforms are drawn (`draw_uniform`) at every layer that MIGHT sample, shaped (B, K_l, S_{l-1} - 1) from the
    slot rather than the padded length.  So once tokens have been dropped, a seeded run consumes torch's generator
    differently from the reference;
  * the scores, pseudo-logits and Gumbel noise are computed in fp32 from the bf16 qkv, so where the bf16 reference
    graph rounds two candidates to a tie the fused path need not pick the same one.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn
from torch.nn.utils.rnn import pad_sequence

from . import _lib
from .engine import (BlocksCall, EncoderLayer, FusedWeightsMixin, Norm, TransformerEngine, common_reason,
                     head_engine, head_ln_pool, ln_mode, on_device, patch_engine)
from .vit import Patchify

__all__ = ["AdaptiveTokenSampling", "Attention", "FeedForward", "Transformer", "ViT", "batched_index_select",
           "draw_uniform", "sample_gumbel", "sampling_layers", "slot_plan"]


def exists(val):
    return val is not None


def pair(t):
    return t if isinstance(t, tuple) else (t, t)


def log(t, eps=1e-6):
    return torch.log(t + eps)


def sample_gumbel(shape, device, dtype, eps=1e-6):
    """Gumbel noise -log(-log(u + eps) + eps) of uniforms u drawn like the reference (ats_vit.py:21-23)."""
    u = torch.empty(shape, device=device, dtype=dtype).uniform_(0, 1)
    return -log(-log(u, eps), eps)


def draw_uniform(shape, device, dtype, layer: int) -> torch.Tensor:
    """The uniforms the fused path's select kernel turns into Gumbel noise at encoder layer `layer`: drawn as
    sample_gumbel draws them.  Module-level so that a caller (a test replaying recorded draws) can replace it; a
    replacement may return fp32 or bf16 of `shape`."""
    return torch.empty(shape, device=device, dtype=dtype).uniform_(0, 1)


def batched_index_select(values, indices, dim=1):
    """Per batch element, the entries of `values` along `dim` at `indices`: indices holds values.shape[:dim] leading
    dims, then any index dims; the result is indices.shape + values.shape[dim + 1:] (ats_vit.py:27-42)."""
    lead, rest = indices.shape[:dim], values.shape[dim + 1:]
    flat = indices.reshape(*lead, -1)
    flat = flat.reshape(*flat.shape, *([1] * len(rest))).expand(*flat.shape, *rest)
    return values.gather(dim, flat).reshape(*indices.shape, *rest)


def slot_plan(n_tokens: int, max_tokens_per_depth) -> List[Tuple[int, int, bool]]:
    """(S_in, S_out, may_sample) of every layer of the fused path for sequences of n_tokens (cls included): a layer may
    sample when K < S_in - 1, and then keeps S_out = K + 1 rows per image."""
    out, S = [], n_tokens
    for K in max_tokens_per_depth:
        if K < S - 1:
            out.append((S, K + 1, True))
            S = K + 1
        else:
            out.append((S, S, False))
    return out


class AdaptiveTokenSampling(nn.Module):
    def __init__(self, output_num_tokens, eps=1e-6):
        super().__init__()
        self.eps = eps
        self.output_num_tokens = output_num_tokens

    def forward(self, attn, value, mask):
        heads, K, eps = attn.shape[1], self.output_num_tokens, self.eps
        # the cls query's attention to every other token, weighted by the value norms and summed over the heads
        scores = torch.einsum('b h n, b h n -> b n', attn[..., 0, 1:], value[..., 1:, :].norm(dim=-1))
        pseudo_logits = log(scores / (scores.sum(dim=-1, keepdim=True) + eps))
        pseudo_logits = pseudo_logits.masked_fill(~mask[:, 1:], -torch.finfo(attn.dtype).max / 2)
        # K Gumbel-max draws per image (the softmax inverted to logits); + 1 keeps 0 for the cls token / padding
        pseudo_logits = pseudo_logits.unsqueeze(1).repeat(1, K, 1)
        pseudo_logits = pseudo_logits + sample_gumbel(pseudo_logits.shape, device=attn.device, dtype=attn.dtype)
        drawn = pseudo_logits.argmax(dim=-1) + 1
        # every drawn token once, in order, right-padded with 0 to the longest image of the batch
        kept = pad_sequence([torch.unique(t, sorted=True) for t in torch.unbind(drawn)], batch_first=True)
        new_mask = F.pad(kept != 0, (1, 0), value=True)
        kept = F.pad(kept, (1, 0), value=0)
        new_attn = batched_index_select(attn, kept.unsqueeze(1).expand(-1, heads, -1), dim=2)
        return new_attn, new_mask, kept


class FeedForward(nn.Module):
    def __init__(self, dim, hidden_dim, dropout=0.):
        super().__init__()
        self.net = nn.Sequential(
            nn.LayerNorm(dim),
            nn.Linear(dim, hidden_dim),
            nn.GELU(),
            nn.Dropout(dropout),
            nn.Linear(hidden_dim, dim),
            nn.Dropout(dropout),
        )

    def forward(self, x):
        return self.net(x)


class Attention(nn.Module):
    def __init__(self, dim, heads=8, dim_head=64, dropout=0., output_num_tokens=None):
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5

        self.norm = nn.LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)

        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)

        self.output_num_tokens = output_num_tokens
        self.ats = AdaptiveTokenSampling(output_num_tokens) if exists(output_num_tokens) else None

        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout))

    def forward(self, x, *, mask):
        b, num_tokens, _ = x.shape
        x = self.norm(x)
        q, k, v = (t.reshape(b, num_tokens, self.heads, -1).transpose(1, 2) for t in self.to_qkv(x).chunk(3, dim=-1))
        dots = torch.matmul(q, k.transpose(-1, -2)) * self.scale
        if exists(mask):
            pairs = mask[:, None, :, None] * mask[:, None, None, :]
            dots = dots.masked_fill(~pairs, -torch.finfo(dots.dtype).max)
        attn = self.dropout(self.attend(dots))

        sampled_token_ids = None
        if exists(self.output_num_tokens) and (num_tokens - 1) > self.output_num_tokens:
            attn, mask, sampled_token_ids = self.ats(attn, v, mask=mask)

        out = torch.matmul(attn, v).transpose(1, 2)
        out = out.reshape(b, out.shape[1], -1)
        return self.to_out(out), mask, sampled_token_ids


class Transformer(FusedWeightsMixin, nn.Module):
    """depth x (attention with token sampling, feed-forward) residual blocks, no final LayerNorm (ats_vit.py:153-192).
    forward(x) -> (x, token_ids) always runs the PyTorch graph: the fused layers need the slot bookkeeping that only
    ViT.forward_fused keeps, and run through engine() there."""

    def engine(self) -> TransformerEngine:
        """The TransformerEngine over encoder_layers(), made on first use, kept with the module."""
        eng = self.__dict__.get("_engine")
        if eng is None:
            eng = self._engine = TransformerEngine(self)
        return eng

    def __init__(self, dim, depth, max_tokens_per_depth, heads, dim_head, mlp_dim, dropout=0.):
        super().__init__()
        assert len(max_tokens_per_depth) == depth, \
            'max_tokens_per_depth must be a tuple of length that is equal to the depth of the transformer'
        assert sorted(max_tokens_per_depth, reverse=True) == list(max_tokens_per_depth), \
            'max_tokens_per_depth must be in decreasing order'
        assert min(max_tokens_per_depth) > 0, 'max_tokens_per_depth must have at least 1 token at any layer'

        self.dropout_p = float(dropout)
        self.layers = nn.ModuleList([])
        for _, output_num_tokens in zip(range(depth), max_tokens_per_depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, output_num_tokens=output_num_tokens, heads=heads, dim_head=dim_head, dropout=dropout),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))

    def encoder_layers(self) -> Tuple[List[EncoderLayer], Optional[Norm]]:
        layers = []
        for attn, ff in self.layers:
            out, fc1, fc2 = attn.to_out[0], ff.net[1], ff.net[4]
            layers.append(EncoderLayer(
                ln1=Norm.of(attn.norm), qkv_w=attn.to_qkv.weight, out_w=out.weight, out_b=out.bias,
                ln2=Norm.of(ff.net[0]), fc1_w=fc1.weight, fc1_b=fc1.bias, fc2_w=fc2.weight, fc2_b=fc2.bias,
                heads=attn.heads, dim_head=attn.dim_head, scale=float(attn.scale)))
        return layers, None

    def forward(self, x):
        b, n, device = *x.shape[:2], x.device
        # the mask tracks each image's padding once tokens have been dropped
        mask = torch.ones((b, n), device=device, dtype=torch.bool)
        token_ids = torch.arange(n, device=device).unsqueeze(0).repeat(b, 1)
        for attn, ff in self.layers:
            attn_out, mask, sampled_token_ids = attn(x, mask=mask)
            if exists(sampled_token_ids):
                # the residual follows the kept tokens
                x = batched_index_select(x, sampled_token_ids, dim=1)
                token_ids = batched_index_select(token_ids, sampled_token_ids, dim=1)
            x = x + attn_out
            x = ff(x) + x
        return x, token_ids


class ViT(FusedWeightsMixin, nn.Module):
    def __init__(self, *, image_size, patch_size, num_classes, dim, depth, max_tokens_per_depth, heads, mlp_dim,
                 channels=3, dim_head=64, dropout=0., emb_dropout=0.):
        super().__init__()
        image_height, image_width = pair(image_size)
        patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, \
            'Image dimensions must be divisible by the patch size.'
        num_patches = (image_height // patch_height) * (image_width // patch_width)
        patch_dim = channels * patch_height * patch_width
        self.patch_size = (patch_height, patch_width)

        self.to_patch_embedding = nn.Sequential(
            Patchify(patch_height, patch_width),
            nn.LayerNorm(patch_dim),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )

        self.pos_embedding = nn.Parameter(torch.randn(1, num_patches + 1, dim))
        self.cls_token = nn.Parameter(torch.randn(1, 1, dim))
        self.dropout = nn.Dropout(emb_dropout)

        self.transformer = Transformer(dim, depth, max_tokens_per_depth, heads, dim_head, mlp_dim, dropout)

        self.mlp_head = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, num_classes))

        self.max_tokens_per_depth = tuple(max_tokens_per_depth)
        self._emb_dropout_p = float(emb_dropout)
        self._cu: dict = {}

    # ---------------------------------------------------------------------------------------------- dispatch
    def fused_reason(self, img: torch.Tensor) -> Optional[str]:
        """None if forward(img) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        if img.dim() != 4:
            return "input is not (B, C, H, W)"
        ph, pw = self.patch_size
        if img.shape[1] * ph * pw != self.to_patch_embedding[1].normalized_shape[0]:
            return "channel count differs from the constructor's (the reference's LayerNorm raises)"
        r = common_reason(self, img, encoders=(self.transformer,),
                          dropout_p=max(self._emb_dropout_p, self.transformer.dropout_p))
        if r is not None:
            return r
        if img.shape[2] % ph or img.shape[3] % pw:
            return "image not divisible by the patch size"
        n = (img.shape[2] // ph) * (img.shape[3] // pw)
        if n + 1 > self.pos_embedding.shape[1]:
            return f"{n + 1} tokens exceed the positional table ({self.pos_embedding.shape[1]})"
        r = self.transformer.engine().unsupported_reason(n + 1)
        if r is not None:
            return r
        sampling = [S for S, _, may in slot_plan(n + 1, self.max_tokens_per_depth) if may]
        if sampling:
            S, H = sampling[0], self.transformer.layers[0][0].heads
            if S > _lib.ATS_MAX_TOKENS:
                return f"{S} tokens at a sampling layer (the select kernel takes at most {_lib.ATS_MAX_TOKENS})"
            if H * S > _lib.ATS_MAX_HEAD_TOKENS:
                return f"{H} heads x {S} tokens at a sampling layer (the select kernel holds at most " \
                       f"{_lib.ATS_MAX_HEAD_TOKENS})"
        return None

    def forward(self, img, return_sampled_token_ids=False):
        if self.fused_reason(img) is None:
            with on_device(img):
                logits, ids, lens = self.forward_fused(img)
                if not return_sampled_token_ids:
                    return logits
                # ids[:, 1:] - 1 up to the batch's padded length (a host synchronisation, only when asked for)
                width = int(lens.max()) - 1
                return logits, ids[:, 1:1 + width].long() - 1
        return self.forward_eager(img, return_sampled_token_ids)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, img, return_sampled_token_ids=False):
        x = self.to_patch_embedding(img)
        b, n, _ = x.shape

        cls_tokens = self.cls_token.expand(b, -1, -1)
        x = torch.cat((cls_tokens, x), dim=1)
        x += self.pos_embedding[:, :(n + 1)]
        x = self.dropout(x)

        x, token_ids = self.transformer(x)

        logits = self.mlp_head(x[:, 0])

        if return_sampled_token_ids:
            # without the cls token, and -1 for padding
            return logits, token_ids[:, 1:] - 1
        return logits

    # ---------------------------------------------------------------------------------------------- fused kernels
    def _start(self, B: int, N: int, device: torch.device) -> Tuple[torch.Tensor, torch.Tensor]:
        """(lengths int32 [B] = N, token ids int32 [B*N] = 0 .. N-1 per image), made once per shape (read only)."""
        key = (B, N, str(device))
        if key not in self._cu:
            self._cu[key] = (torch.full((B,), N, device=device, dtype=torch.int32),
                             torch.arange(N, device=device, dtype=torch.int32).repeat(B))
        return self._cu[key]

    def _scratch(self, B: int, S: int, D: int, I: int, device: torch.device) -> dict:
        """The buffers of sampling_layers for B images whose first sampling layer keeps S rows each: every later slot is
        at most S rows.  Made once per (shape, device, stream), as the engine's workspace is: two streams running the
        model must not share them."""
        key = ("scratch", B, S, D, I, str(device), torch.cuda.current_stream(device).cuda_stream)
        if key not in self._cu:
            i32 = dict(device=device, dtype=torch.int32)
            self._cu[key] = {
                "x": torch.empty(B * S, D, device=device, dtype=torch.float32),     # the other stream of the ping-pong
                "q": torch.empty(B * S, I, device=device, dtype=torch.bfloat16),    # the kept rows' queries
                "src": torch.empty(B * S, **i32),
                "lens": [torch.empty(B, **i32) for _ in range(2)],
                "ids": [torch.empty(B * S, **i32) for _ in range(2)],
            }
        return self._cu[key]

    def forward_fused(self, img: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """(logits [B, classes] bf16, token ids int32 [B, S_last] with 0 on padding rows, lengths int32 [B]); must run
        inside on_device(img)."""
        dev = img.device
        D = self.cls_token.shape[-1]
        pe, eng = patch_engine(self), self.transformer.engine()
        pos = pe.prepared(dev)["pos"].view(-1, D)
        B, N = pe.geometry(img)
        ws = eng.workspace(B * N, dev)
        xb, stats = eng.entry_buffers(B * N, dev)
        x, B, N = pe.run(img, xb=xb, stats=stats, pos=pos)
        plan = slot_plan(N, self.max_tokens_per_depth)
        first = next((i for i, (_, _, may) in enumerate(plan) if may), len(plan))
        if first:
            eng.run_blocks(x, B, N, primed=xb is not None, layers=None if first == len(plan) else range(first))
        lens, ids = self._start(B, N, dev)
        if first < len(plan):
            # the LN-fold row sums of ws['xn'] the next folded GEMM reads: the embedding's, or the last fc2's
            L0 = eng.layers[0]
            scratch = self._scratch(B, plan[first][1], D, L0.heads * L0.dim_head, dev)
            x, lens, ids = sampling_layers(eng, x, B, plan, first, self.max_tokens_per_depth, lens, ids,
                                           ws["stats_in"] if first == 0 else ws["stats_a"], img.dtype, scratch)
        S = plan[-1][1]
        pooled = head_ln_pool(self, self.mlp_head[0], x, B, S, mean=False)
        return head_engine(self, self.mlp_head[1]).run(pooled), ids.view(B, S), lens


def sampling_layers(eng: TransformerEngine, x: torch.Tensor, B: int, plan, first: int, max_tokens, lens: torch.Tensor,
                    ids: torch.Tensor, sums: torch.Tensor, dtype: torch.dtype, scratch: dict
                    ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The encoder layers first .. of the fused path (module docstring) on the fp32 stream x[B*S_first, D] whose
    workspace rows eng.workspace(B*N) holds; lens int32 [B] and ids int32 [B*S_first] the valid lengths and token ids
    entering them, `sums` the LN-fold row sums of the workspace's bf16 copy of x (fold mode).  Returns the final stream
    [B*S_last, D] and the lengths and ids after the last layer.  `scratch` (ViT._scratch) holds the other stream, the
    kept queries, the row map and the ping-pong lengths and ids, each for the rows of the first sampling layer's slot."""
    dev = x.device
    t = eng.prepared()
    ws = eng.workspace(x.shape[0], dev)
    fold = ln_mode() == "fold"
    if not fold:
        sums = None
    L0 = eng.layers[0]
    I = L0.heads * L0.dim_head
    streams = [x, scratch["x"]]                 # ping-pong: a compaction in place would race across CTAs
    qc, src, lens_buf, ids_buf = scratch["q"], scratch["src"], scratch["lens"], scratch["ids"]
    rows = lambda m: {k: v[:m] for k, v in ws.items()}       # noqa: E731  row-prefix views of the workspace
    cur = nsel = 0
    for i in range(first, len(plan)):
        S_in, S_out, may = plan[i]
        L, K = eng.layers[i], max_tokens[i]
        x = streams[cur][:B * S_in]
        c = BlocksCall(t, rows(B * S_in), x, B, S_in, None, None, None, None, None, None, fold, False)
        c.sums = sums
        c.project(L, i)                                          # qkv = LN1(x) Wqkv^T on B*S_in rows
        qkv = c.qkv
        keys = lens
        if may:
            u = draw_uniform((B, K, S_in - 1), dev, dtype=dtype, layer=i)
            j, nsel = nsel % 2, nsel + 1
            _lib.ats_select(qkv, lens, ids, u, src[:B * S_out], lens_buf[j], ids_buf[j][:B * S_out], B, S_in,
                            K, L.heads, L.dim_head, L.scale)
            cur ^= 1
            x = streams[cur][:B * S_out]
            _lib.ats_gather(src[:B * S_out], x=streams[cur ^ 1][:B * S_in], x_out=x, a=qkv,
                            a_out=qc[:B * S_out], ncols=I)
            q, lens, ids = qc[:B * S_out], lens_buf[j], ids_buf[j][:B * S_out]
        else:
            q = qkv[:, :I]
        c = BlocksCall(t, rows(B * S_out), x, B, S_out, None, None, None, None, None, None, fold, False)
        o = c.o[:, :I]
        _lib.attention_kv_lens(q, qkv[:, I:3 * I], o, keys, B, S_out, S_in, L.heads, L.dim_head, L.scale)
        c.residual(o, f"{i}.out", x, "stats_b")
        c.normed(x, f"{i}.ln2", L.ln2, f"{i}.fc1", c.h, gelu=True)
        c.residual(c.h, f"{i}.fc2", x, "stats_a")
        sums = c.sums
    return x, lens, ids
