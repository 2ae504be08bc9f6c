"""fp64 references with a per-element error bound for the row kernels of rowops.cu  --  TEST INFRASTRUCTURE.

The conventions are those of oracle/bounds.py: every function returns `(ref, bound)`, fp64 tensors on the inputs'
device; the reference takes the kernel's own inputs, and the bound counts only the rounding the kernel itself does,
in its order, at the depth its fp32 sums really have.  u = 2^-24; there is no fast-math in build.py, so fp32 `/` and
`sqrtf` are correctly rounded (u relative) and `rsqrtf` is within 2 ulp (4 u relative).

Depth.  A warp sums a row in two stages: each lane runs a chain over its own elements, then a butterfly of 5 shuffle
levels (log2(LPH) levels inside an LPH-lane head group).  An element that passes through d roundings on its way to
the total contributes at most d u |element| to the error (first order), so a sum of depth d is off by at most
d u sum|element|.  The depths:
  - ln_row_stats (layernorm, embed_tokens, embed_varlen): D % 4 == 0 reads float4 and adds (v.x + v.y) + (v.z + v.w)
    into the lane's chain, depth 2 + ceil(D / 128) + 5; otherwise one element per step, ceil(D / 32) + 5.  The sum of
    squares has the same shape.  With this depth the LayerNorm is bounds.layernorm_e32 (its derivation is in
    bounds.py): E32 bounds the fp32 value (v - mean) rstd gamma + beta.
  - the row statistics (emit_row_stats, common.cuh) of the kernel's bf16 copy x^: D % 4 == 0: sum depth 2 +
    ceil(D / 128) + 5, sum of squares a chain of 4 fmas per float4, 4 ceil(D / 128) + 5; otherwise ceil(D / 32) + 5
    for both.  The squares of bf16 values are exact in fp32, so the bound is d u sum|x^| and d u sum x^2.  Statistics
    of the unrounded fp32 values differ from those of x^ by about 2^-9 sum|x| / sqrt(D) -- at D = 768, 50 times this
    bound, where the generic D u sum|x| bound of bounds.stats_reference is of the same size as the difference.
  - head norms (rmsnorm_heads_kernel): each lane holds 8 values of a head; the sum of squares is a chain of 8 fmas
    (exact products of bf16 values), the sum of values 4 adds of pairs (depth 5), the two-pass sum of (v - mean)^2 a
    chain of 8 fmas; then log2(LPH) butterfly levels, LPH = 4 / 8 / 16 / 16 lanes for dh = 32 / 64 / 80 / 128.

Output arithmetic after the statistics, each operation u relative unless noted:
  - token assembly (embed_tokens): patch row ((LN gamma + beta) + pos): E32 + u (|ref| + E32); a class row with a
    position cls + pos: u |ref|; class rows without a position, register-token rows and rows without LayerNorm or
    position are copies (bound 0).  embed_varlen: ((LN gamma + pos_h[row]) + pos_w[col]), two adds after E32.
  - RMS norm: v * (SQRT_DH / max(sqrtf(ss), 1e-12)) * gamma.  rel(inv) = d u / 2 + u (sqrtf) + u (division) + c,
    where c = |fl32(sqrt(dh)) - sqrt(dh)| / sqrt(dh) is the rounding of the kernel's constant (0 for dh = 64); two
    more products give E32 = (rel(inv) + 2 u) |ref|.  An all-zero head gives exactly 0.
  - head LayerNorm (no bias): mean = s1 * fl32(1 / dh) is off by d_mu = ((d1 + 2) u + k) mean|v| (k: the rounding
    of 1 / dh, nonzero for dh = 80); the two-pass q = sum (v - mean^)^2 = dh (var + (mean - mean^)^2) with relative
    error (d2 + 2) u, times fl32(1 / dh) (u + k), + eps (u): rel(var + eps) = (d2 + 4) u + k + d_mu^2 / (var + eps),
    rstd = rsqrtf(.) adds 4 u to half of it.  Then (v - mean^) rstd gamma: E32 = |gamma| rstd (|v - mean| (rel(rstd)
    + 3 u) + d_mu).  A one-pass E[v^2] - mean^2 has no such bound: its error is u E[v^2], not u var.
  - mean_pool: a sequential fp32 sum of the first n_pool rows then one division: (n_pool - 1) u mean|x| + u |ref|.
bf16 outputs: bound = bf16_ulp(ref) + (1 + 2^-8) E32 (bounds.layernorm_reference).
"""
from __future__ import annotations

import math
from typing import Optional, Sequence, Tuple

import torch

from oracle.bounds import U, U_BF16, bf16_bound, bf16_ulp, check, excess, layernorm_e32  # noqa: F401 (re-exported)

Tensor = torch.Tensor
HEAD_LANES = {32: 4, 64: 8, 80: 16, 128: 16}     # HeadLanes<DH>::LPH


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def ln_depth(D: int) -> int:
    """Deepest fp32 sum of ln_row_stats over a row of D values (one warp)."""
    return (2 + _cdiv(D, 128) if D % 4 == 0 else _cdiv(D, 32)) + 5


def stats_depths(D: int) -> Tuple[int, int]:
    """Deepest fp32 sums (sum, sum of squares) of emit_row_stats over a row of D values."""
    if D % 4 == 0:
        return 2 + _cdiv(D, 128) + 5, 4 * _cdiv(D, 128) + 5
    return _cdiv(D, 32) + 5, _cdiv(D, 32) + 5


def _bf16_out(ref: Tensor, e32: Tensor) -> Tensor:
    return bf16_ulp(ref) + (1 + U_BF16) * e32


def layernorm_reference(x: Tensor, gamma: Tensor, beta: Optional[Tensor] = None, eps: float = 1e-5,
                        row_index: Optional[Tensor] = None, bf16_out: bool = False) -> Tuple[Tensor, Tensor]:
    """(ref, bound) of b200vit_layernorm on the fp32 rows x[:, :D] (D = gamma.numel(); a wider x is read with its own
    stride, as the kernel's ldx).  row_index: output row r normalises x[row_index[r]].  bf16_out: bound the bf16
    output instead of the fp32 one."""
    D = gamma.numel()
    xs = x[:, :D] if row_index is None else x[row_index.long(), :D]
    ref, e32 = layernorm_e32(xs, gamma, beta, eps, ln_depth(D))
    return (ref, _bf16_out(ref, e32)) if bf16_out else (ref, e32)


def embed_tokens_reference(y: Tensor, gamma: Optional[Tensor], beta: Optional[Tensor], cls: Optional[Tensor],
                           pos: Optional[Tensor], groups: int, n: int, ncls: int, tail: Optional[Tensor] = None,
                           eps: float = 1e-5, pos_period: int = 1, pos_stride: int = 0,
                           cls_pos: bool = True) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [groups * (ncls + n + ntail), D] of the fp32 token rows of b200vit_embed_tokens_grouped.

    Group b reads the positional block at row (b % pos_period) * pos_stride: patch t takes row ncls + t of it when
    cls_pos (the class rows its first ncls rows), else row t (the class rows no position).  gamma None: no
    LayerNorm; pos None: no position; tail rows (register tokens) carry no position."""
    D = y.shape[1]
    dev = y.device
    ntail = 0 if tail is None else tail.shape[0]
    N = ncls + n + ntail
    y64 = y.double().view(groups, n, D)
    if gamma is not None:
        ln, e32 = layernorm_e32(y.view(-1, D), gamma, beta, eps, ln_depth(D))
        ln, e32 = ln.view(groups, n, D), e32.view(groups, n, D)
    else:
        ln, e32 = y64, torch.zeros_like(y64)
    ref = torch.zeros(groups, N, D, dtype=torch.float64, device=dev)
    bound = torch.zeros_like(ref)
    if pos is not None:
        base = (torch.arange(groups, device=dev) % pos_period) * pos_stride
        p64 = pos.double()
        prow = base[:, None] + torch.arange(n, device=dev)[None] + (ncls if cls_pos else 0)
        pp = p64[prow]                                                   # [groups, n, D]
        ref[:, ncls:ncls + n] = ln + pp
        bound[:, ncls:ncls + n] = e32 + U * (ref[:, ncls:ncls + n].abs() + e32)
    else:
        ref[:, ncls:ncls + n] = ln
        bound[:, ncls:ncls + n] = e32
    if ncls:
        c64 = cls.double()[None].expand(groups, -1, -1)
        if pos is not None and cls_pos:
            crow = base[:, None] + torch.arange(ncls, device=dev)[None]
            ref[:, :ncls] = c64 + p64[crow]
            bound[:, :ncls] = U * ref[:, :ncls].abs()
        else:
            ref[:, :ncls] = c64
    if ntail:
        ref[:, ncls + n:] = tail.double()[None]
    return ref.view(-1, D), bound.view(-1, D)


def varlen_grid(lengths: Sequence[int], dims: Sequence[Tuple[int, int]], p: int, device) -> Tuple[Tensor, Tensor]:
    """(row, col) of every packed token in its own image's patch grid (grid width max(W // p, 1))."""
    rows, cols = [], []
    for L, (_, w) in zip(lengths, dims):
        gw = max(w // p, 1)
        i = torch.arange(L)
        rows.append(i // gw)
        cols.append(i % gw)
    return torch.cat(rows).to(device), torch.cat(cols).to(device)


def embed_varlen_reference(y: Tensor, gamma: Tensor, pos_h: Tensor, pos_w: Tensor, lengths: Sequence[int],
                           dims: Sequence[Tuple[int, int]], p: int, eps: float = 1e-5) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [T, D] of b200vit_embed_varlen: ((LN(y) gamma + pos_h[row]) + pos_w[col]), LayerNorm without
    bias, (row, col) the token's place in its own image's patch grid."""
    D = y.shape[1]
    ln, e = layernorm_e32(y, gamma, None, eps, ln_depth(D))
    r, c = varlen_grid(lengths, dims, p, y.device)
    h = ln + pos_h.double()[r]
    e = e + U * (h.abs() + e)
    ref = h + pos_w.double()[c]
    return ref, e + U * (ref.abs() + e)


def row_stats_reference(xb: Tensor) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [M, 2] of the (sum, sum of squares) emit_row_stats writes for the rows of its bf16 copy xb[M, D]."""
    x = xb.double()
    d1, d2 = stats_depths(x.shape[1])
    ref = torch.stack([x.sum(1), (x * x).sum(1)], 1)
    bound = torch.stack([d1 * U * x.abs().sum(1), d2 * U * (x * x).sum(1)], 1)
    return ref, bound * (1 + 2 * max(d1, d2) * U)


def _head_depths(dh: int) -> Tuple[int, int]:
    """(depth of the sum of squares / second pass, depth of the sum of values) of a head."""
    L = int(math.log2(HEAD_LANES[dh]))
    return 8 + L, 5 + L


def _const_rel(v: float) -> float:
    """Relative rounding error of the fp32 constant nearest to v."""
    return abs(float(torch.tensor(v, dtype=torch.float32).item()) - v) / v


def rmsnorm_heads_reference(x: Tensor, gamma: Tensor) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [T, H, dh] of the bf16 per-head RMS norm v / max(||v||, 1e-12) sqrt(dh) gamma[h] of the bf16 heads
    x[T, H, dh], gamma [H, dh] (rmsnorm_heads, qk_rmsnorm, the norm half of gemm_headnorm)."""
    v = x.double()
    dh = v.shape[-1]
    d, _ = _head_depths(dh)
    nrm = torch.linalg.vector_norm(v, dim=-1, keepdim=True)
    ref = v / nrm.clamp_min(1e-12) * math.sqrt(dh) * gamma.double()
    rel = d * U / 2 + 2 * U + _const_rel(math.sqrt(dh)) + 2 * U
    return ref, _bf16_out(ref, rel * (1 + 1e-3) * ref.abs())


def layernorm_heads_reference(x: Tensor, gamma: Tensor, eps: float = 1e-5) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [T, H, dh] of the bf16 per-head LayerNorm without bias (v - mean) / sqrt(var + eps) gamma[h] with
    the two-pass variance (layernorm_heads, the norm half of gemm_headnorm with EPI_HEADLN)."""
    v = x.double()
    dh = v.shape[-1]
    d2, d1 = _head_depths(dh)
    k = _const_rel(1.0 / dh)
    mu = v.mean(-1, keepdim=True)
    var = ((v - mu) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    c = v - mu
    g = gamma.double()
    ref = c * rstd * g
    d_mu = ((d1 + 2) * U + k) * v.abs().mean(-1, keepdim=True)
    rel = ((d2 + 4) * U + k + d_mu * d_mu / (var + eps)) / 2 + 4 * U
    e32 = g.abs() * rstd * (c.abs() * (rel + 3 * U) + d_mu)
    return ref, _bf16_out(ref, e32 * (1 + 1e-3))


def mean_pool_reference(x: Tensor, n_pool: int) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [B, D] of b200vit_mean_pool: the mean of the first n_pool token rows of x[B, N, D]."""
    xs = x[:, :n_pool].double()
    ref = xs.mean(1)
    e = (n_pool - 1) * U * xs.abs().mean(1)
    return ref, e + U * (ref.abs() + e)
