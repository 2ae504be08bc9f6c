"""fp64 references with a per-element error bound for the GEMM and the patch kernels  --  TEST INFRASTRUCTURE.

Every function returns `(ref, bound)`: fp64 tensors of the kernel output's shape, on the device of the inputs.  A
kernel output `got` is correct when |got - ref| <= bound for every element (`check`).  The reference takes the
kernel's own inputs (the bf16 operands, the fp32 LayerNorm sums, col_s, the bias), so the bound counts only the
rounding the kernel itself does, never the conditioning of its inputs.

Notation: u = 2^-24 is the unit roundoff of fp32.  A bf16 result is round-to-nearest with an 8-bit significand, so
|bf16(v) - v| <= 2^-8 |v| (half an ulp, and the ulp of v is at most 2^-7 |v|).

GEMM accumulation.  acc = A W^T and abs = |A| |W|^T in fp64.  The bf16 products are exact in fp32; a chain of K fp32
additions is off by at most K u abs (first order), a worst case that random data stays far below.  wgmma's
accumulator need not round like IEEE fp32 (it may truncate the aligned addends), so the term is
E = (C_ACC K + 2) u abs: C_ACC K u abs for the growth along K, measured on the H100 (see C_ACC), and 2 u abs >= 2 u |acc|
for the last rounding of the accumulator, which a truncating accumulator can make at any K.

Epilogue, in the kernel's order (gemm.cu):
  - bias only:       v = fma(acc, 1, b)                       E + u (|acc| + |b| + E)
  - LN fold:         mu = s1/K, var = max(s2/K - mu^2, 0), rstd = rsqrtf(var + eps)  (s1, s2: the fp32 parts added
                     up in order), k = -rstd mu, c = fma(k, col_s, b), v = fma(acc, rstd, c).  The reference computes
                     mu, var and rstd in fp64 from the same fp32 parts.  Error terms: the sum of P parts and the
                     division (P + 2) u sum|part| / K for mu and E[x^2]; var = s2/K - mu^2 adds 2 |mu| d_mu and
                     3 u (s2/K + mu^2); rsqrtf is within 2 ulp (4 u relative) after the rounding of var + eps; then
                     rstd E + rstd rel (|acc| + |mu col_s|) + rstd d_mu |col_s| for the propagated errors and
                     u (|k col_s| + |b|) + u (|c|) + u |v| for the two fmas.
  - GELU:            1.13 E + 1.2e-5 + 4 u |gelu(v)|: 1.13 bounds the derivative of the erf GELU, 1.2e-5 is the
                     absolute accuracy of the epilogue's GELU (tests/test_gpu_kernels.py::test_gelu_epilogue_accuracy).
  - residual:        v + r in fp32: + u (|ref| + E).
  - bf16 output:     + 2^-8 (|ref| + E).
Statistics (EPI_STATS): part p of a row is the (sum, sum of squares) of the kernel's own bf16 output over columns
[p w, (p + 1) w) of that row, w = 128 if N > 128 else 64.  No fp32 sum in the kernel is deeper than the part's column
count, so the bound is ncols u sum|.|; a part wholly past N must be exactly zero.

Patch kernels (patchify_ln, patchify_spt_ln, patchify_varlen_ln): one warp per patch computes, in fp32, the mean
(one sum over the patch: each lane adds ceil(pd / 32) values, then a 5-level shuffle tree, depth d), the variance as
a second pass over (x - mean)^2, rsqrtf, then (x - mean) rstd gamma + beta rounded to bf16.  With d_mu = (d + 2) u
mean|x|, rel = (d + 3) u / 2 + d_mu^2 / (2 (var + eps)) + 5 u for rstd:
    E32 = |gamma| (|xhat| (rel + 3 u) + rstd d_mu) + u (|xhat gamma| + |beta|),
and the bf16 rounding of a value within E32 of ref is within one bf16 ulp of ref plus E32 (bound = ulp(ref) + E32).
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

Tensor = torch.Tensor

U = 2.0 ** -24          # fp32 unit roundoff
U_BF16 = 2.0 ** -8      # largest relative rounding error of a bf16 result (half an ulp)
# Growth of the wgmma fp32 accumulation error along K, in units of K u abs.  On an H100 80GB HBM3 the worst
# |got - ref| / (K u abs) of every fp32 output without the LayerNorm fold in tests/test_gpu_persistent.py (K from 40 to
# 832, every kernel instance, after the fp32 adds of bias and residual) was 0.034; C_ACC keeps a margin of about 7.
C_ACC = 0.25
GELU_SLOPE = 1.13
GELU_ABS = 1.2e-5
HARDSWISH_SLOPE = 1.5


def gemm_reference(a: Tensor, w: Tensor, *, bias: Optional[Tensor] = None, resid: Optional[Tensor] = None,
                   ln_sums: Optional[Tensor] = None, col_s: Optional[Tensor] = None, ln_eps: float = 1e-5,
                   gelu: bool = False, hardswish: bool = False, bf16_out: bool = False) -> Tuple[Tensor, Tensor]:
    """(ref, bound) of epilogue(a[m, K] @ w[N, K]^T) as b200vit_gemm_bf16 computes it.

    a, w: the bf16 operands (K = a.shape[1] exactly: slice off any row padding first).  ln_sums: [m, parts, 2] or
    [m, 2] fp32 partial row sums; resid: [m, N] fp32.  hardswish: EPI_HARDSWISH, y clamp(y + 3, 0, 6) / 6 (slope at
    most 1.5, then its add, clamp, product and division).  bf16_out: bound the bf16 output instead of the fp32 one."""
    a64, w64 = a.double(), w.double()
    K = a.shape[1]
    acc = a64 @ w64.t()
    e = (C_ACC * K + 2) * U * (a64.abs() @ w64.abs().t())
    b = None if bias is None else bias.double()
    if ln_sums is not None:
        s = ln_sums.double().reshape(a.shape[0], -1, 2)
        parts = s.shape[1]
        cs = col_s.double()[None]
        s1, s2 = s[..., 0].sum(1, keepdim=True), s[..., 1].sum(1, keepdim=True)
        mu, ex2 = s1 / K, s2 / K
        var = (ex2 - mu * mu).clamp_min(0.0)
        rstd = 1.0 / torch.sqrt(var + ln_eps)
        d_mu = (parts + 2) * U * s[..., 0].abs().sum(1, keepdim=True) / K
        d_ex2 = (parts + 2) * U * s[..., 1].abs().sum(1, keepdim=True) / K
        d_var = d_ex2 + 2 * mu.abs() * d_mu + 3 * U * (ex2 + mu * mu)
        x = (d_var + U * (var + ln_eps)) / (var + ln_eps)
        # relative error of rstd: exact for the perturbed argument (not first order), then rsqrtf's 2 ulp
        rel = (1.0 / torch.sqrt((1.0 - x).clamp_min(1e-300)) - 1.0) + 4 * U
        bb = b if b is not None else torch.zeros_like(cs)
        k = -rstd * mu
        c = k * cs + bb
        ref = rstd * acc + c
        d_k = rstd * (1 + rel) * (mu.abs() * (rel + 2 * U) + d_mu)
        d_c = d_k * cs.abs() + U * ((k * cs).abs() + bb.abs() + c.abs() + d_k * cs.abs())
        e = rstd * (1 + rel) * e + rstd * rel * acc.abs() + d_c
        e = e + U * (ref.abs() + e)
    elif b is not None:
        ref = acc + b[None]
        e = e + U * (acc.abs() + b.abs()[None] + e)
    else:
        ref = acc
    if gelu:
        ref = 0.5 * ref * (1.0 + torch.erf(ref / math.sqrt(2.0)))
        e = GELU_SLOPE * e + GELU_ABS + 4 * U * ref.abs()
    if hardswish:
        ref = ref * (ref + 3).clamp(0, 6) / 6
        e = HARDSWISH_SLOPE * e + 4 * U * ref.abs() + 1e-30
    if resid is not None:
        ref = ref + resid.double()
        e = e + U * (ref.abs() + e)
    return (ref, bf16_bound(ref, e)) if bf16_out else (ref, e)


def bf16_bound(ref: Tensor, bound: Tensor) -> Tensor:
    """The bound of a value within `bound` of `ref` after its rounding to bf16."""
    return bound + U_BF16 * (ref.abs() + bound)


def gemm_inputs(M: int, N: int, K: int, *, parts: int = 1, lda: Optional[int] = None, ldw: Optional[int] = None,
                ldo: Optional[int] = None, seed: int = 0, device="cpu") -> dict:
    """Seeded GEMM operands in the distributions the layer chain sees: A [M, lda] bf16 rows with a nonzero mean (the
    LayerNorm fold has something to subtract), W [N, ldw] bf16 of scale 1/sqrt(K), a bias and an fp32 residual
    [M, ldo] of unit scale, col_s = the fp32 row sums of W and ln_sums [M, parts, 2] = fp32 (sum, sum of squares) of
    A over `parts` contiguous column ranges (the statistics parts of the GEMM that wrote A)."""
    g = torch.Generator(device=device).manual_seed(seed)
    lda, ldw, ldo = lda or K, ldw or K, ldo or N
    a = (torch.randn(M, lda, generator=g, device=device) * 2 + 0.3).bfloat16()
    w = (torch.randn(N, ldw, generator=g, device=device) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, generator=g, device=device)
    resid = torch.randn(M, ldo, generator=g, device=device)
    af = a[:, :K].float()
    part = torch.arange(K, device=device) * parts // K
    s1 = torch.zeros(M, parts, device=device).index_add_(1, part, af)
    s2 = torch.zeros(M, parts, device=device).index_add_(1, part, af * af)
    return dict(a=a, w=w, bias=bias, resid=resid, col_s=w[:, :K].float().sum(1).contiguous(),
                ln_sums=torch.stack([s1, s2], 2).contiguous())


def stats_width(N: int) -> int:
    """Output columns per statistics part (gemm.cu: launch_gemm)."""
    return 128 if N > 128 else 64


def stats_reference(out_bf16: Tensor, parts: int) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [m, parts, 2] of EPI_STATS, from the kernel's own bf16 output rows out_bf16[m, N]."""
    x = out_bf16.double()
    N = x.shape[1]
    wd = stats_width(N)
    ref = torch.zeros(x.shape[0], parts, 2, dtype=torch.float64, device=x.device)
    bound = torch.zeros_like(ref)
    for p in range(parts):
        seg = x[:, p * wd:min((p + 1) * wd, N)]
        if seg.shape[1] == 0:
            continue
        ref[:, p, 0], ref[:, p, 1] = seg.sum(1), (seg * seg).sum(1)
        bound[:, p, 0] = seg.shape[1] * U * seg.abs().sum(1)
        bound[:, p, 1] = seg.shape[1] * U * (seg * seg).sum(1)
    return ref, bound


def bf16_ulp(x: Tensor) -> Tensor:
    """The spacing of bf16 numbers at |x| (8-bit significand): 2^(floor(log2 |x|) - 7); 0 at x = 0."""
    _, ex = torch.frexp(x.abs())
    return torch.where(x == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), ex - 8))


def layernorm_reference(x: Tensor, gamma: Tensor, beta: Optional[Tensor] = None, eps: float = 1e-5,
                        depth: Optional[int] = None) -> Tuple[Tensor, Tensor]:
    """(ref, bound) of the bf16 LayerNorm of the rows x[m, pd] (the patch pixels, in the output's column order) as
    the patch kernels compute it.  depth: the deepest fp32 sum of a row (default ceil(pd / 32) + 5, one warp)."""
    ref, e32 = layernorm_e32(x, gamma, beta, eps, depth)
    # the rounding of y32 is within half its ulp: at most one ulp of ref plus 2^-8 E32
    return ref, bf16_ulp(ref) + (1 + U_BF16) * e32


def layernorm_e32(x: Tensor, gamma: Tensor, beta: Optional[Tensor] = None, eps: float = 1e-5,
                  depth: Optional[int] = None) -> Tuple[Tensor, Tensor]:
    """(ref, E32): the fp64 LayerNorm of the rows x[m, pd] and the bound E32 of the fp32 value a one-warp two-pass
    LayerNorm computes before any output rounding (module docstring).  depth as in layernorm_reference."""
    x = x.double()
    pd = x.shape[1]
    d = depth if depth is not None else -(-pd // 32) + 5
    g = gamma.double()[None]
    bt = beta.double()[None] if beta is not None else torch.zeros_like(g)
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xh = (x - mu) * rstd
    ref = xh * g + bt
    d_mu = (d + 2) * U * x.abs().mean(1, keepdim=True)
    rel = (d + 3) * U / 2 + d_mu * d_mu / (2 * (var + eps)) + 5 * U
    e32 = g.abs() * (xh.abs() * (rel + 3 * U) + rstd * d_mu) + U * ((xh * g).abs() + bt.abs())
    return ref, e32


def excess(got: Tensor, ref: Tensor, bound: Tensor) -> float:
    """max |got - ref| / bound (inf where a NaN or an error against a zero bound is found)."""
    d = (got.double() - ref).abs()
    r = torch.where(d == 0, torch.zeros_like(d), d / bound)
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    return r.max().item() if r.numel() else 0.0


def check(got: Tensor, ref: Tensor, bound: Tensor, what: str = "") -> float:
    """Assert |got - ref| <= bound everywhere; returns the worst ratio (excess)."""
    d = (got.double() - ref).abs()
    bad = ~(d <= bound)
    if bad.any():
        idx = bad.nonzero()[0].tolist()
        i = tuple(idx)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound, first at {i}: "
                             f"got {got[i].item()!r} ref {ref[i].item()!r} bound {bound[i].item():.3e}")
    return excess(got, ref, bound)
