"""fp64 references with a per-element error bound for the attention kernels whose softmax is fp32 throughout
(b200vit_attn_pool and b200vit_attention_cls: attn_pool_kernel in rowops.cu; b200vit_attention_cls_headmix:
cls_headmix.cu; b200vit_attention_xca: xca.cu)  --  TEST INFRASTRUCTURE.

Every function returns `(ref, bound)`: fp64 tensors of the kernel output's shape, on the device of the inputs, to be
checked with oracle.bounds.check.  The reference takes the kernel's own bf16 / fp32 inputs, so the bound counts only the
rounding the kernel does.  u = 2^-24; every term is first order in u (the second-order terms are below 2^-40 relative
at every size these kernels accept).  None of these kernels rounds a probability to bf16, so no rounding of P is
replayed: every weight carries a relative error of a few fp32 ulps, and the bound is built from that.

Weighted averages.  attn_pool_kernel and the xca softmax compute y = sum_j w~_j v_j / sum_j w~_j.  If the kernel's weight
of key j is w~_j = W_j (1 + a_j), |a_j| <= ab_j, with W_j the exact weights and p_j = W_j / sum W, then
    y~ - y = sum_j p_j a_j (v_j - y) / (1 + sum_j p_j a_j),
so the error is at most sum_j p_j ab_j |v_j - y| / (1 - sum_j p_j ab_j): it charges each key's weight error against
|v_j - y|, not |v_j|, and a common factor of all weights (the running max, the merge factors of one warp) cancels.

attn_pool_kernel (rowops.cu).  One CTA of 8 warps per (image, head); warp w walks the 4-token groups w, w + 8, ...;
scores in natural-log units, q fp32 (NaViT: qn as given; CLS: fl(q scale)).
  - Score.  Lane l holds the element pairs l + 32 c (NP = ceil(dh / 64) of them): q.x k.x + q.y k.y (a product and an
    fma) added to the lane's sum, then a 5-level butterfly: depth 3 NP + 5, plus u for fl(q scale) (CLS):
    ds_j = (3 NP + 6) u sum|q||k_j|.
  - Exponentials.  __expf(x) is ex2.approx.ftz(fl(x log2e_f)): EX2_REL, plus |x| (u + dL) from the product and the fp32
    log2(e) (dL its relative error), plus u |x| for x = fl(s - m).  A key's weight passes its own exponential, the
    corr of every later group of its warp and the warp's merge factor __expf(m_w - M).  Their arguments telescope to
    at most 2 (M - s_j) (M the final max), so the log error of w~_j is
        d_j = ds_j + 2 (2 u + dL) (M - s_j + 2 max ds) + R EX2_REL,   R = G_w + 2 exponentials,
    G_w = ceil(n / 32) 4-token groups per warp (+ 1 for the query's own key under CLS), and ab_j = e^d_j - 1.
  - Sums.  Numerator and l: per group one rescale and four adds, then the fma chain over the 8 warps' partials:
    D = 5 (G_w + 1) + 8 roundings.  |dN| <= D u sum p (1 + ab) |v|, |dl| <= D u sum p (1 + ab), and flushed
    exponentials (ftz, below 2^-126, l >= 1 in the kernel's units) at most 2 n 2^-126 relative.
  - Output.  y = fl(A fl(1 / L)): two roundings, then bf16:
        E = (sum p ab |v - y| + D u sum p (1 + ab) |v| + |y| (D u sum p (1 + ab) + f)) / (1 - sum p ab - D u sum p (1 + ab) - f)
        bound = E32 + ulp_bf16(|y| + E32) / 2,   E32 = E + 2 u (|y| + E),   f = 2 n 2^-126.

cls_headmix.cu.  Per image all heads: q~ = fl(q c) with c = fl(scale log2e) (log2 units), s_h = q~_h . k_h as a chain
of dh fp32 fmas; s'_g = sum_h pre[h][g] s_h (a chain of H fmas; the zero-padded heads add exact zeros).
  - Scores.  A chain of fmas is off by at most u times the sum of its partial sums' magnitudes (each rounding is at
    most u |partial|), and the partial sums are replayed in the kernel's order in fp64: ds_h = u (sum_d |q~ k|_d +
    sum_d |partial_d|) (the first sum for fl(q c)); ds'_g = sum_h |pre_hg| ds_h + u sum_h |partial of the pre-mix|.
    Against the worst case dh u sum|q||k| this is about sqrt(dh) times smaller on random-sign products.
  - Both passes call the same `scores`, so they see the same fp32 scores s~'.  Write lse* = log2 sum_j 2^s~'_j.  Then
    the kernel's p~_gj = q_gj (1 + eps_gj) K_g, with q = softmax(s~') (the exact softmax of the kernel's scores),
    eps the error of pass 2's own ex2 and argument rounding, and K_g = 2^(lse* - lse~) the error of the lse.  The score
    errors move q only through the softmax, which is invariant to a common shift, so they are charged against
    |v_j - z_g| (z_g = sum_j p_gj v_j, the exact average of head g's weights over the output head's values):
        |sum_j q_gj v_j - z_g| <= sum_j p_gj sig_gj |v_j - z_g| / (1 - sum_j p_gj sig_gj),  sig = 2^ds' - 1.
  - Pass 1 (lse~).  Lane = key: K_l = ceil(nk / 256) keys per lane with an online max / sum, 5 shuffle merges, the
    8-warp merge.  A term of L passes its own ex2, up to K_l corrs, 5 + 1 merge factors: R = K_l + 7 ex2.approx
    (EX2_REL each) whose fp32 arguments (u |.| each, log2 units) telescope to at most 2 (M - s'_j + 2 max ds').  With the
    sums' roundings (2 per lane step, 2 per shuffle level, 2 per warp: D_L = 2 K_l + 26) the relative error of L
    against sum_j 2^(s~'_j - M) is
        rho = sum_j p_j (2^(2 u (M - s'_j + 2 max ds')) (1 + EX2_REL)^R - 1) + D_L u + nk 2^-126,
    and lse~ = fl(M + log2f(L)) is off from lse* by dlse = -log2(1 - rho) + 2 u |log2 L| (log2f: 1 ulp) + u |lse|:
    |K_g - 1| <= kap = 2^dlse - 1.
  - Pass 2.  p_g = ex2(fl(s'_g - lse_g)): eps_gj <= 2^(u (|s'_gj - lse_g| + 2 max ds' + dlse)) (1 + EX2_REL) - 1, plus
    2^-126 for a flushed result.  p is never normalised again.  Per (mixed head g, output head f):
        e_gf = (1 + kap) (sum_j p sig |v_j - z| + sum_j p (1 + sig) eps |v_j|) / (1 - sum p sig) + kap |z| + 2^-126 sum|v|.
  - Post-mix p'_f = sum_g post[g][f] p_g (H fmas, H u sum_g |post_gf| p~_g) and P V: each warp's chain over its at
    most K_w = 32 ceil(nk / 256) keys, then the sum of the 8 warps' partials ((K_w + 8) u sum_j |p~'_fj| |v_j|):
        E = sum_g |post_gf| e_gf + H u sum_j sum_g |post_gf| p~_gj |v_j| + (K_w + 8) u sum_j |p~'_fj| |v_j|,
    p~ bounded above by p (1 + sig) (1 + eps) (1 + kap) / (1 - sum p sig);  bound = E + ulp_bf16(|y| + E) / 2.

xca.cu.  Per (image, head), q, k, v the [N, dh] slices:
  - G_ij = sum_n q_ni k_nj and ss_i = sum_n q_ni^2 are fp32 fma chains over n = 0 .. N-1 in order (the zero rows of a
    partial tile add exact zeros).  As for cls_headmix, each chain is off by at most u times the sum of its partial
    sums' magnitudes, replayed in fp64: |dG_ij| <= u PG_ij, PG_ij = sum_n |sum_{m<=n} q_mi k_mj|, and |dss_i| <= u PS_i,
    PS_i = sum_n sum_{m<=n} q_mi^2.  r_i = 1 / max(sqrtf(ss_i), 1e-12f): relative rel_i = u PS_i / (2 ss_i) + 2 u.
  - x_ij = fl(fl(fl(tau r_i) G_ij) r_j): dx_ij = tau r_i r_j u PG_ij + |x_ij| (rel_i + rel_j + 3 u).  PG_ij <= N A_ij
    with A = |q|^T |k|, and by Cauchy-Schwarz A_ij r_i r_j <= 1: the first term is at most tau N u even where q_i and
    k_j are nearly orthogonal (G_ij ~ 0), which a bound relative to |G_ij| would miss.  On random-sign products the
    partial sums grow like sqrt(n), so PG is about sqrt(N) times below that worst case.  The norms' partial sums are
    positive and grow linearly, so PS_i is about N ss_i / 2 and the |x| term is about |x_ij| N u / 2.  Where a score
    comes near tau (columns nearly parallel) that is tau N u / 2, about 1.9e-3 at N = 3136 and tau = e^3, the order of
    the output's bf16 half ulp; on random columns |x_ij| is about tau / sqrt(N) and the term stays small.
  - Softmax over the dh channels: expf (2 ulp: 4 u) of fl(x - m) (u |x - m|): ab_j = e^(dx_j + u (|x_j - m| + 2 max dx)
    + 4 u) - 1; l is a chain of dh / 16 adds and a 4-level butterfly (D_l = dh / 16 + 4); A = fl(e fl(1 / l)).  So
    A~_ij = A_ij (1 + t_ij), |t_ij| <= (ab_j + sum_k A_ik ab_k + D_l u) / (1 - sum_k A_ik ab_k - D_l u) + 3 u.
  - O = V A^T: a chain of dh fmas.  E = sum_j A_ij |t_ij| |v_nj| + dh u sum_j A_ij (1 + |t_ij|) |v_nj|, then the bf16
    rounding as above.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from oracle.attention_bounds import EX2_REL, FTZ, LOG2E, scale_log2e
from oracle.bounds import U, bf16_ulp

Tensor = torch.Tensor

LOG2E_F = torch.tensor(LOG2E, dtype=torch.float32).item()      # the fp32 log2(e) of __expf
DL = abs(LOG2E_F / LOG2E - 1.0)
EXPF_REL = 4 * U                                               # expf: 2 ulp (CUDA C++ Programming Guide)
NORM_EPS_F = torch.tensor(1e-12, dtype=torch.float32).item()   # xca.cu: fmaxf(sqrtf(ss), 1e-12f)


def _out_bound(ref: Tensor, e32: Tensor) -> Tensor:
    """The bound of the bf16 rounding of a value within e32 of ref."""
    return e32 + 0.5 * bf16_ulp(ref.abs() + e32)


def cls_operands(qkv_self: Tensor, ctx: Optional[Tensor], rows: int, first: int, n: int, H: int,
                 dh: int) -> Tuple[Tensor, Tensor, Tensor]:
    """q [B, H, dh] and k, v [B, n + 1, H, dh] (key 0 the query token's own) of the class-token kernels' C ABI:
    row b of qkv_self[B, 3 H dh] is q | k | v of image b, its context rows b rows + first + j (j < n) of ctx [k | v]."""
    B, I = qkv_self.shape[0], H * dh
    q, ks, vs = qkv_self.view(B, 3, H, dh).unbind(1)
    if n == 0:
        return q, ks[:, None], vs[:, None]
    c = ctx[:B * rows].reshape(B, rows, ctx.shape[1])[:, first:first + n, :2 * I]
    k = torch.cat([ks[:, None], c[..., :I].reshape(B, n, H, dh)], 1)
    v = torch.cat([vs[:, None], c[..., I:].reshape(B, n, H, dh)], 1)
    return q, k, v


def pool_reference(q: Tensor, k: Tensor, v: Tensor, *, cls: bool, scale: float = 1.0) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [G, dh] of attn_pool_kernel: softmax_j(scale q . k_j) v_j for G independent queries q [G, dh]
    (fp32 for NaViT, bf16 for CLS) over k, v [G, nk, dh] (bf16).  cls: the CLS instance, whose key 0 is the query
    token's own key (taken by warp 0 before its groups) and whose q is rounded after the scale; nk = n + 1."""
    G, nk, dh = k.shape
    s32 = torch.tensor(scale, dtype=torch.float32).item()
    q64 = q.double() * s32
    k64, v64 = k.double(), v.double()
    s = torch.einsum('gd,gjd->gj', q64, k64)
    NP = -(-dh // 64)
    ds = (3 * NP + 6) * U * torch.einsum('gd,gjd->gj', q64.abs(), k64.abs())
    n_ctx = nk - 1 if cls else nk
    gw = -(-n_ctx // 32) + (1 if cls else 0)
    M = s.amax(-1, keepdim=True)
    d = ds + 2 * (2 * U + DL) * (M - s + 2 * ds.amax(-1, keepdim=True)) + (gw + 2) * EX2_REL
    p = torch.softmax(s, -1)
    y = torch.einsum('gj,gjd->gd', p, v64)
    ab = torch.expm1(d)
    D = 5 * (gw + 1) + 8
    f = 2 * nk * FTZ
    sa = (p * ab).sum(-1, keepdim=True)
    s3 = (p * (1 + ab)).sum(-1, keepdim=True)
    num = (torch.einsum('gj,gjd->gd', p * ab, (v64 - y[:, None]).abs())
           + D * U * torch.einsum('gj,gjd->gd', p * (1 + ab), v64.abs()) + y.abs() * (D * U * s3 + f)
           + f * v64.abs().amax(1))
    e = num / (1 - sa - D * U * s3 - f)
    e32 = e + 2 * U * (y.abs() + e)
    return y, _out_bound(y, e32)


def navit_pool_reference(kv: Tensor, qn: Tensor, lengths, H: int, dh: int) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [S, H dh] of b200vit_attn_pool on kv[T, 2 H dh] (k | v, bf16), qn[H dh] fp32, images of
    `lengths` consecutive tokens."""
    I = H * dh
    ref = torch.empty(len(lengths), I, dtype=torch.float64, device=kv.device)
    bound = torch.empty_like(ref)
    o = 0
    for i, n in enumerate(lengths):
        k = kv[o:o + n, :I].reshape(n, H, dh).transpose(0, 1)
        v = kv[o:o + n, I:2 * I].reshape(n, H, dh).transpose(0, 1)
        r, b = pool_reference(qn.view(H, dh), k, v, cls=False)
        ref[i], bound[i] = r.reshape(I), b.reshape(I)
        o += n
    return ref, bound


def cls_reference(qkv_self: Tensor, ctx: Optional[Tensor], rows: int, first: int, n: int, H: int, dh: int,
                  scale: float) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [B, H dh] of b200vit_attention_cls (the C ABI's arguments, see cls_operands)."""
    q, k, v = cls_operands(qkv_self, ctx, rows, first, n, H, dh)
    B = q.shape[0]
    r, b = pool_reference(q.reshape(B * H, dh), k.permute(0, 2, 1, 3).reshape(B * H, n + 1, dh),
                          v.permute(0, 2, 1, 3).reshape(B * H, n + 1, dh), cls=True, scale=scale)
    return r.view(B, H * dh), b.view(B, H * dh)


def cls_headmix_reference(qkv_self: Tensor, ctx: Optional[Tensor], rows: int, first: int, n: int, H: int, dh: int,
                          scale: float, pre: Tensor, post: Tensor) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [B, H dh] of b200vit_attention_cls_headmix: softmax over the keys of the pre-mixed scores, post-mixed,
    times v (pre, post fp32 [H, H], [input head, output head])."""
    q, k, v = cls_operands(qkv_self, ctx, rows, first, n, H, dh)
    B, nk = k.shape[0], k.shape[1]
    c = scale_log2e(scale)
    q64, k64, v64 = q.double() * c, k.double(), v.double()
    pre64, post64 = pre.double(), post.double()
    prod = q64[:, None] * k64                                           # [B, nk, H, dh]
    part = prod.cumsum(-1)                                              # the fma chain's partial sums, in order
    s = part[..., -1].transpose(1, 2)                                   # [B, H, nk]
    ds = U * (part.abs().sum(-1) + prod.abs().sum(-1)).transpose(1, 2)
    mix = (pre64[None, :, :, None] * s[:, :, None]).cumsum(1)           # [B, h, g, nk]: the pre-mix chain over h
    sm = mix[:, -1]
    dsm = torch.einsum('bhj,hg->bgj', ds, pre64.abs()) + U * mix.abs().sum(1)
    M = sm.amax(-1, keepdim=True)
    lse = torch.logsumexp(sm * math.log(2), -1, keepdim=True) / math.log(2)
    p = torch.exp2(sm - lse)
    dsmax = dsm.amax(-1, keepdim=True)
    sig = torch.expm1(dsm * math.log(2))
    sa = (p * sig).sum(-1, keepdim=True)
    kl = -(-nk // 256)
    rho = ((p * (torch.exp2(2 * U * (M - sm + 2 * dsmax)) * (1 + EX2_REL) ** (kl + 7) - 1)).sum(-1, keepdim=True)
           + (2 * kl + 26) * U + nk * FTZ)
    dlse = -torch.log2(1 - rho) + 2 * U * (lse - M).abs() + U * lse.abs()
    kap = torch.expm1(dlse * math.log(2))
    eps = torch.exp2(U * ((sm - lse).abs() + 2 * dsmax + dlse)) * (1 + EX2_REL) - 1
    pmax = p * (1 + sig) * (1 + eps) * (1 + kap) / (1 - sa) + FTZ             # >= the kernel's p_g
    kw = 32 * kl
    y = torch.empty(B, H, dh, dtype=torch.float64, device=q.device)
    e32 = torch.empty_like(y)
    for f in range(H):
        vf = v64[:, :, f]                                                # [B, nk, dh]
        z = torch.einsum('bgj,bjd->bgd', p, vf)
        e1 = torch.einsum('bgj,bgjd->bgd', p * sig, (vf[:, None] - z[:, :, None]).abs())
        e2 = torch.einsum('bgj,bjd->bgd', p * (1 + sig) * eps, vf.abs())
        eg = (1 + kap) * (e1 + e2) / (1 - sa) + kap * z.abs() + FTZ * vf.abs().sum(1)[:, None]
        w = post64[:, f]
        y[:, f] = torch.einsum('g,bgd->bd', w, z)
        pp = torch.einsum('g,bgj->bj', w, p).abs() + torch.einsum('g,bgj->bj', w.abs(), pmax - p + H * U * pmax)
        e32[:, f] = (torch.einsum('g,bgd->bd', w.abs(), eg)
                     + H * U * torch.einsum('g,bgj,bjd->bd', w.abs(), pmax, vf.abs())
                     + (kw + 8) * U * torch.einsum('bj,bjd->bd', pp, vf.abs()))
    return y.reshape(B, H * dh), _out_bound(y, e32).reshape(B, H * dh)


def xca_tile(dh: int) -> int:
    """Tokens per tile of xca.cu."""
    return 32 if dh >= 128 else 64


def xca_reference(qkv: Tensor, tau: Tensor, B: int, N: int, H: int, dh: int) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [B N, H dh] of b200vit_attention_xca on qkv[B N, 3 H dh] (bf16), tau fp32 [H]."""
    q, k, v = qkv.double().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)          # [B, H, N, dh] each
    t = tau.double().view(1, H, 1, 1)
    G = q.transpose(-1, -2) @ k
    PG = torch.zeros_like(G)                                                    # sum over n of |partial sums of G|
    run = torch.zeros_like(G)
    for n0 in range(0, N, 64):
        cs = run[:, :, None] + torch.einsum('bhni,bhnj->bhnij', q[:, :, n0:n0 + 64], k[:, :, n0:n0 + 64]).cumsum(2)
        PG += cs.abs().sum(2)
        run = cs[:, :, -1]

    def recip_norm(a):
        ss = (a * a).sum(2)
        rel = torch.where(ss > 0, U * (a * a).cumsum(2).sum(2) / (2 * ss), torch.zeros_like(ss)) + 2 * U
        return 1.0 / ss.sqrt().clamp_min(NORM_EPS_F), rel

    rq, relq = recip_norm(q)                                                    # [B, H, dh]
    rk, relk = recip_norm(k)
    x = t * rq[..., :, None] * G * rk[..., None, :]
    dx = (t * rq[..., :, None] * PG * rk[..., None, :] * U
          + x.abs() * (relq[..., :, None] + relk[..., None, :] + 3 * U))
    m = x.amax(-1, keepdim=True)
    a = torch.softmax(x, -1)
    ab = torch.expm1(dx + U * ((x - m).abs() + 2 * dx.amax(-1, keepdim=True)) + EXPF_REL)
    sa = (a * ab).sum(-1, keepdim=True)
    dl = (dh // 16 + 4) * U
    th = (ab + sa + dl) / (1 - sa - dl) + 3 * U
    y = v @ a.transpose(-1, -2)                                                 # [B, H, N, dh]
    e32 = v.abs() @ (a * th).transpose(-1, -2) + dh * U * (v.abs() @ (a * (1 + th)).transpose(-1, -2))
    bound = _out_bound(y, e32)
    return (y.permute(0, 2, 1, 3).reshape(B * N, H * dh), bound.permute(0, 2, 1, 3).reshape(B * N, H * dh))
