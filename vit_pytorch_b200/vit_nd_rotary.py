"""Drop-in `ViTND` for lucidrains/vit-pytorch's `vit_pytorch.vit_nd_rotary.ViTND`: the N-dimensional ViT (inputs of
rank 1..7) with golden-gate N-d rotary position embeddings instead of a learned table, with a fused sm_90a forward.

Same constructor keywords, parameter and buffer names / shapes / registration order (=> identical `state_dict` and
identical random init under the same seed; reference vit_nd_rotary.py:28-302).  The one `rotary_emb` module is shared
by every attention layer, so its persistent `freqs` buffer appears under each of them in the state_dict, as in the
reference.

Fused forward (engine.py): b200vit_patchify_nd -> patch GEMM + bias -> b200vit_embed_tokens (LayerNorm(dim), no
positional term) -> encoder blocks with b200vit_rope_qk after every QKV GEMM -> final LayerNorm -> mean over the tokens
(or the tokens themselves with return_embed=True) -> head GEMM.  The (cos, sin) table is built on the device with the
reference's own torch expression from the module's CURRENT `freqs` buffer (bf16 after `.to(torch.bfloat16)`, as the
reference multiplies it) and cached per patch grid.  Anything the fused path does not cover runs the PyTorch graph
below, which mirrors the reference module for module.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from .engine import _WEIGHT_EPOCH, FusedWeightsMixin, classify, on_device
from .vit import FeedForward, FusedTransformer
from .vit_nd import NdPatchEngine, PatchifyND, ensure_tuple, nd_encode, nd_fused_reason


# ------------------------------------------------------------------------------------------------------------------
# golden-gate N-d rotary embedding (Jerry Xiong, https://jerryxio.ng/posts/nd-rope/; reference vit_nd_rotary.py:28-96)
# ------------------------------------------------------------------------------------------------------------------
def _golden_ratio(m: int) -> float:
    """The fixed point of x = (1 + x)^(1 / (m + 1)) (10 iterations from 2): the generalised golden ratio of dim m."""
    x = 2.0
    for _ in range(10):
        x = (1 + x) ** (1.0 / (m + 1.0))
    return x


def _directions(n: int, d: int) -> torch.Tensor:
    """n unit vectors in R^d from the golden-ratio low-discrepancy sequence mapped through the inverse normal CDF."""
    alpha = (1.0 / _golden_ratio(d)) ** torch.arange(1, d + 1, dtype=torch.float64)
    i = torch.arange(1, n + 1, dtype=torch.float64).unsqueeze(1)
    u = torch.fmod(i * alpha, 1.0)
    return F.normalize(torch.erfinv(2.0 * u - 1.0), dim=-1, p=2).float()


class GoldenGateRoPENd(nn.Module):
    """freqs[h, f, :] = omega_f * direction_(h, f): each (head, frequency) pair rotates along its own direction of the
    position space; theta = freqs . pos."""

    def __init__(self, dim_pos: int, heads: int, dim_head: int, rope_min_freq: float = 1.0,
                 rope_max_freq: float = 10000.0, rope_p_zero_freqs: float = 0.0) -> None:
        super().__init__()
        n_freqs = dim_head // 2
        n_zero = round(rope_p_zero_freqs * n_freqs)
        omega = torch.cat((torch.zeros(n_zero),
                           rope_min_freq * (rope_max_freq / rope_min_freq) ** torch.linspace(0, 1, n_freqs - n_zero)))
        directions = _directions(heads * n_freqs, dim_pos).reshape(heads, n_freqs, dim_pos)
        self.register_buffer('freqs', directions * omega[:, None])     # (h, f, p)

    def forward(self, input: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
        # input (b, h, n, d), pos (b, n, p)
        x, y = input.float().chunk(2, dim=-1)
        cos, sin = _cos_sin(self.freqs, pos)
        x_out = x * cos - y * sin
        y_out = x * sin + y * cos
        return torch.cat((x_out, y_out), dim=-1).type_as(input)


def _cos_sin(freqs: torch.Tensor, pos: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """cos / sin of theta (b, h, n, f) = sum_p freqs (1, h, 1, f, p) * pos (b, 1, n, 1, p): the reference's
    expression (vit_nd_rotary.py:82-89), so the fused table holds the very values its eager forward uses."""
    theta = (freqs[None, :, None] * pos.float()[:, None, :, None, :]).sum(dim=-1)
    return torch.cos(theta), torch.sin(theta)


def rope_table(freqs: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
    """pos (b, n, p) -> the b200vit_rope_qk table: fp32 [b*n, h, f, 2] = (cos, sin), contiguous."""
    cos, sin = _cos_sin(freqs, pos)                                    # (b, h, n, f)
    cs = torch.stack((cos, sin), dim=-1).permute(0, 2, 1, 3, 4)        # (b, n, h, f, 2)
    return cs.reshape(-1, *cs.shape[2:]).contiguous()


def grid_positions(grid, device) -> torch.Tensor:
    """(n, ndim) fp32 coordinates of a patch grid in row-major order (vit_nd_rotary.py:278-284)."""
    axes = [torch.arange(d, device=device, dtype=torch.float32) for d in grid]
    return torch.stack(torch.meshgrid(*axes, indexing='ij'), dim=-1).reshape(-1, len(grid))


# ------------------------------------------------------------------------------------------------------------------
# encoder (reference vit_nd_rotary.py:100-173)
# ------------------------------------------------------------------------------------------------------------------
class Attention(nn.Module):
    """Pre-LN attention with separate to_qk / to_v projections and rotary q / k (vit_nd_rotary.py:115-156)."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64, dropout: float = 0.,
                 rotary_emb: Optional[GoldenGateRoPENd] = None) -> None:
        super().__init__()
        inner_dim = dim_head * heads
        project_out = not (heads == 1 and dim_head == dim)
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.rotary_emb = rotary_emb
        self.norm = nn.LayerNorm(dim)
        self.attend = nn.Softmax(dim=-1)
        self.dropout = nn.Dropout(dropout)
        self.to_qk = nn.Linear(dim, inner_dim * 2, bias=False)
        self.to_v = nn.Linear(dim, inner_dim, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout)) if project_out else nn.Identity()

    def forward(self, x: torch.Tensor, pos: Optional[torch.Tensor] = None) -> torch.Tensor:
        x = self.norm(x)
        b, n, _ = x.shape
        q, k = self.to_qk(x).chunk(2, dim=-1)
        q, k, v = (t.reshape(b, n, self.heads, -1).transpose(1, 2) for t in (q, k, self.to_v(x)))
        if self.rotary_emb is not None:
            assert pos is not None
            q = self.rotary_emb(q, pos)
            k = self.rotary_emb(k, pos)
        dots = torch.matmul(q, k.transpose(-1, -2)) * self.scale
        attn = self.dropout(self.attend(dots))
        out = torch.matmul(attn, v).transpose(1, 2).reshape(b, n, -1)
        return self.to_out(out)


class Transformer(FusedTransformer):
    """depth x (rotary attention, feed-forward) + final LayerNorm; callable as transformer(tokens, pos) like the
    reference (vit_nd_rotary.py:158-173).  The fused call takes a per-token rope table (rows = B*N)."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int, dropout: float = 0.,
                 rotary_emb: Optional[GoldenGateRoPENd] = None) -> None:
        super().__init__()
        self.dropout_p = float(dropout)
        self.norm = nn.LayerNorm(dim)
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                Attention(dim, heads=heads, dim_head=dim_head, dropout=dropout, rotary_emb=rotary_emb),
                FeedForward(dim, mlp_dim, dropout=dropout),
            ]))

    @staticmethod
    def qkv_weight(attn: nn.Module) -> torch.Tensor:
        return torch.cat((attn.to_qk.weight, attn.to_v.weight), dim=0)        # q | k | v rows

    def shared_rotary(self) -> Tuple[Optional[GoldenGateRoPENd], Optional[str]]:
        """(the rotary module every attention holds, None) or (None, why the layers cannot share one table)."""
        mods = {id(attn.rotary_emb): attn.rotary_emb for attn, _ in self.layers}
        if len(mods) > 1:
            return None, "the attention layers hold different rotary_emb modules"
        return next(iter(mods.values()), None), None

    def fused_reason(self, x: torch.Tensor, pos: Optional[torch.Tensor] = None) -> Optional[str]:
        r = super().fused_reason(x)
        if r is not None:
            return r
        rot, r = self.shared_rotary()
        if r is not None or rot is None:
            return r
        if pos is None:
            return "no positions given (the reference asserts)"
        if pos.dim() != 3 or tuple(pos.shape) != (x.shape[0], x.shape[1], rot.freqs.shape[-1]):
            return f"positions of shape {tuple(pos.shape)} for tokens {tuple(x.shape)}"
        if pos.device != x.device:
            return "positions and tokens on different devices"
        return None

    def forward_eager(self, x: torch.Tensor, pos: Optional[torch.Tensor] = None) -> torch.Tensor:
        for attn, ff in self.layers:
            x = attn(x, pos) + x
            x = ff(x) + x
        return self.norm(x)

    def forward(self, x: torch.Tensor, pos: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self.fused_reason(x, pos) is None:
            rot = self.shared_rotary()[0]
            rope = None if rot is None else (rope_table(rot.freqs, pos), x.shape[0] * x.shape[1])
            return self.engine().forward_tokens(x, rope=rope)
        return self.forward_eager(x, pos)


class ViTND(FusedWeightsMixin, nn.Module):
    def __init__(self, *, ndim: int, input_shape, patch_size, num_classes: int, dim: int, depth: int, heads: int,
                 mlp_dim: int, channels: int = 3, dim_head: int = 64, dropout: float = 0., emb_dropout: float = 0.,
                 rope_min_freq: float = 1.0, rope_max_freq: float = 10000.0, rope_p_zero_freqs: float = 0.0) -> None:
        super().__init__()
        assert 1 <= ndim <= 7, 'ndim must be between 1 and 7'
        self.ndim = ndim
        input_shape = ensure_tuple(input_shape, ndim)
        patch_size = ensure_tuple(patch_size, ndim)
        for i, (s, p) in enumerate(zip(input_shape, patch_size)):
            assert s % p == 0, f'Input dimension {i} ({s}) must be divisible by patch size ({p})'
        patch_dim = channels * math.prod(patch_size)

        self.to_patch_embedding = nn.Sequential(
            PatchifyND(patch_size, flatten=False),
            nn.Linear(patch_dim, dim),
            nn.LayerNorm(dim),
        )
        self.dropout = nn.Dropout(emb_dropout)
        self.rotary_emb = GoldenGateRoPENd(dim_pos=ndim, heads=heads, dim_head=dim_head, rope_min_freq=rope_min_freq,
                                           rope_max_freq=rope_max_freq, rope_p_zero_freqs=rope_p_zero_freqs)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim, dropout, rotary_emb=self.rotary_emb)
        self.to_latent = nn.Identity()
        self.mlp_head = nn.Linear(dim, num_classes)

        self._nd_patch = tuple(patch_size)
        self._emb_dropout_p = float(emb_dropout)
        self._nd_engine = NdPatchEngine(self, self._nd_patch)
        self._rope_cache: Dict[tuple, torch.Tensor] = {}

    def muon_parameters(self) -> List[nn.Parameter]:
        params = []
        for m in self.modules():
            if isinstance(m, Attention):
                params.extend([m.to_v.weight, m.to_out[0].weight])
            elif isinstance(m, FeedForward):
                params.extend([m.net[1].weight, m.net[-2].weight])
        return params

    # ---------------------------------------------------------------------------------------------- dispatch
    def fused_reason(self, x: torch.Tensor) -> Optional[str]:
        """None if forward(x) will run the fused sm_90a kernels, else the reason for the PyTorch graph."""
        r = nd_fused_reason(self, x, self._nd_patch, max(self._emb_dropout_p, self.transformer.dropout_p))
        if r is None:
            rot, r = self.transformer.shared_rotary()
            if r is None and rot is not self.rotary_emb:
                r = "the attention layers do not hold the model's rotary_emb"
        if r is None:
            r = self.transformer.engine().unsupported_reason(self._nd_engine.tokens(x)[1])
        return r

    def forward(self, x: torch.Tensor, return_embed: bool = False) -> torch.Tensor:
        if self.fused_reason(x) is None:
            with on_device(x):
                return self.forward_fused(x, return_embed)
        return self.forward_eager(x, return_embed)

    # ---------------------------------------------------------------------------------------------- PyTorch graph
    def forward_eager(self, x: torch.Tensor, return_embed: bool = False) -> torch.Tensor:
        x = self.to_patch_embedding(x)                                  # (b, *grid, dim)
        batch, *grid, dim = x.shape
        pos = grid_positions(grid, x.device).expand(batch, -1, -1)
        x = self.dropout(x.reshape(batch, -1, dim))
        embed = self.transformer(x, pos)
        if return_embed:
            return embed.reshape(batch, *grid, dim)
        pooled = embed.mean(dim=1)
        pooled = self.to_latent(pooled)
        return self.mlp_head(pooled)

    # ---------------------------------------------------------------------------------------------- fused kernels
    def grid_table(self, grid: Tuple[int, ...], device: torch.device) -> torch.Tensor:
        """The rope_qk table [n, h, f, 2] of one patch grid, cached per (grid, device) and the freqs buffer's
        version."""
        f = self.rotary_emb.freqs
        key = (grid, str(device), _WEIGHT_EPOCH[0], f.data_ptr(), f._version, f.dtype)
        t = self._rope_cache.get(key)
        if t is None:
            self._rope_cache = {k: v for k, v in self._rope_cache.items() if k[:2] != key[:2]}
            t = self._rope_cache[key] = rope_table(f.to(device), grid_positions(grid, device)[None])
        return t

    def forward_fused(self, img: torch.Tensor, return_embed: bool = False) -> torch.Tensor:
        grid = tuple(s // p for s, p in zip(img.shape[2:], self._nd_patch))
        cs = self.grid_table(grid, img.device)
        x, B, N = nd_encode(self, self._nd_engine, img, rope=(cs, cs.shape[0]))      # table rows = N
        D = x.shape[1]
        eng = self.transformer.engine()
        if return_embed:
            out = torch.empty(B * N, D, device=img.device, dtype=torch.bfloat16)
            eng.final_norm(x, out_bf16=out)
            return out.view(B, *grid, D)
        return classify(self, self.mlp_head, eng.pool(x, B, N, mean=True))
