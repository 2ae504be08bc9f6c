"""fp64 reference with a per-element error bound for the head-mixing attention kernel of headmix.cu
(b200vit_attention_headmix / _ex)  --  TEST INFRASTRUCTURE.

`headmix_reference` returns `(ref, bound)`: fp64 tensors [B N, H dh] on the device of the inputs, to be checked with
oracle.bounds.check.  It takes the kernel's own bf16 qkv and fp32 pre, post, gamma and beta, so the bound counts only
the rounding the kernel does.  Notation as in oracle/attention_bounds.py: u = 2^-24, C_ACC the wgmma accumulation
constant, c = scale_log2e(scale) (the host's fp32 scale log2 e), scores in log2 units.  Per (row i, key j), each step
of the kernel in order, the exact value and the bound of the kernel's difference from it:

  1. Score.  s_h = fl(fl(q_h . k_h) c), the dot product a wgmma m64n16k16 chain over dh:
         ds_h = c (C_ACC dh + 2) u sum|q_h||k_h| + 2 u |s_h|.
  2. Pre-mix (PRE).  s'_g = sum_h pre[h][g] s_h, an fma chain over h = 0 .. HC - 1 in order (the padded heads add
     exact zeros).  ds'_g = sum_h |pre_hg| ds_h (propagated) + u sum_h |partial_h| (the chain's own roundings, the
     partial sums replayed in fp64 in the kernel's order).  Without PRE s' = s, ds' = ds.
  3. lse.  Pass 1 splits the keys into 16-key blocks.  Per block the quad of a row holds 4 keys per lane: the block max
     bm, exp2(s' - bm) per key, 3 adds per lane and 2 shuffle levels (5 roundings, each at most u times the block's
     sum); the running pair merges as sum = sum ex2(m0 - mx) + bs ex2(bm - mx), mx = max(m0, bm); finally
     lse = fl(mx + __log2f(sum)).  Against L = sum_j 2^(s'_j - M) (M the row max), with P_b the partial sum of L over
     blocks 0 .. b, the kernel's sum is off by a relative rho:
       - every key passes its own ex2 and its block's merge factor (EX2_REL each), its score error ds'_j, and
         fp32 arguments (s - bm, bm - mx, and the m0 - mx of every later rise) whose magnitudes telescope to at most
         M - s'_j + 2 max ds': sum_j w_j (2^(ds'_j + u (M - s'_j + 2 max ds')) (1 + EX2_REL)^2 - 1), w = softmax;
       - the running sum is rescaled only at a block where the running max rises: ex2(0) is exact, so blocks whose
         maxima stay below the running max, even with the score errors (bm_b + 2 max ds' < max of bm over 0 .. b-1),
         cost nothing; a block that can raise it charges (EX2_REL + u) P_(b-1) (the ex2 and the product);
       - the sums: u (5 L + L + sum_b P_b) (the block sums, fl(bs f2), and the add of each merge);
       - ftz: terms and rescaled sums below 2^-126 against a kernel sum >= 1: 2 N 2^-126.
     __log2f is within 2^-22 absolute on [0.5, 2] and 2 ulp (4 u relative) elsewhere (CUDA C++ Programming Guide), and
     sum >= 1 (it holds the max key's exp2(0) = 1).  So
         dlse = -log2(1 - rho) + 2^-22 + 4 u (lse - M + 2 max ds') + u |lse|,
     common to a whole (row, head), and nothing divides it out: pass 2's p is not normalised again.
  4. Probabilities.  p_g = ex2(fl(s'_g - lse_g)): x = s' - lse is off by dx = ds' + dlse + u (|x| + ds' + dlse), so
     p~ lies in [p 2^-dx (1 - EX2_REL), p 2^dx (1 + EX2_REL)] (the low end 0 below 2^-126, ftz): dp its half width.
  5. Post-mix and LayerNorm over heads, in the kernel's order:
       acc_f = sum_g post[g][f] p_g, an fma chain over g:  dacc = sum_g |post_gf| dp_g (1 + H u) + u sum_g |partial|;
       coef~_g = fl(fl(sum_f post[g][f]) / H), a sequential fp32 sum and an IEEE division, computed here exactly as the
       kernel does: it differs from coef_g = sum_f post[g][f] / H by the known dcoef_g = |coef~_g - coef_g|;
       mean = sum_g coef~_g p_g, an fma chain (not the mean of the kernel's acc_f, so its error is its own);
       d_f = fl(acc_f - mean) = sum_g (post_gf - coef_g) p_g exactly.  acc and mean take the same p~, so its error
       enters through post - coef, which is 0 for equal heads and small for near-equal ones:
         dd = sum_g |post_gf - coef_g| dp_g + sum_g dcoef_g (p_g + dp_g) + u (sum |partials of acc| + sum |partials of
         mean| + H sum_g (|post_gf| + |coef_g|) dp_g) + u (|d| + dd);
       V = sum_f d_f^2, an fma chain over f:  dV = S + u (sum_f partial_f + H S), S = sum_f (2 |d_f| dd_f + dd_f^2);
       rstd = rsqrtf(fl(fl(V / H) + eps)): a = V / H + eps is off by da = (dV / H)(1 + 2 u) + u V / H + u a (1 + u),
       rstd's relative error rel = (1 / sqrt(1 - da / a) - 1)(1 + 4 u) + 4 u (rsqrtf: 2 ulp).  Exact for the perturbed
       argument, not first order: near-equal heads make V tiny and rstd as large as 1 / sqrt(eps), and rstd then
       multiplies the errors of acc - mean, which the bound keeps;
       P''_f = fma(fl(d_f rstd), gamma_f, beta_f):  dxh = rstd (1 + rel) dd + |xhat| rel + u (|xhat| + ...),
       dP'' = |gamma| dxh + u (|P''| + |gamma| dxh).  Without the LayerNorm P'' = acc, dP'' = dacc.
  6. bf16 replay of P''.  The kernel rounds P'' to bf16 before P V, a rounding (up to 2^-9 relative) far above all its
     fp32 noise, so the reference replays it, as attention_bounds does for P: it uses bf16(P''_j) of the fp64 value and
     charges each key A_j = max(bf16(hi) - bf16(P''), bf16(P'') - bf16(lo)) over its interval [lo, hi] = P'' -+ dP''
     (bf16 rounding is monotone), times |v_j|.  A key whose interval stays within one rounding interval costs
     nothing.  Keys at or past N contribute 0: the kernel zeroes their P'' and the TMA zero-fills V past each sequence.
  7. P V.  One fp32 accumulator per output over all N keys in 16-key wgmma steps, with no rescale.  With the LayerNorm
     P'' is O(1) and signed, so sum_j |P''||v| grows like N while the output grows like sqrt(N): the GEMM form
     (C_ACC N + 2) u sum|P''||v| would be about 16 output ulps at N = 16384.  The partial-sum form instead: step b adds
     T_b = sum over its 16 keys to the running O_b = O_(b-1) + T_b, each step's own term (16 C_ACC + 2) u
     sum_step |P''||v| (P'' within A of the replay) and each accumulation u |O_b|, O_b replayed in fp64 (plus u nb
     sum A |v| for the kernel's partials off the replayed ones).  Confirmed on an H100 80GB HBM3 at its 700 W power
     limit with chains whose exact sum is 0 (one head under the LayerNorm, so P'' = beta = 1; v's second half its
     first half negated in reverse order), N = 1024 to 16384, dh 64 and 128 (tests/test_gpu_headmix_bounds.py,
     test_pv_chain_calibration): the worst |got| / bound was 0.022 on zero-mean values (partial sums of order sqrt(N))
     and 0.098 on values of mean 1 (partial sums of order N), against at most 0.0063 of the GEMM form.
  8. Output.  E32 = sum_j A_j |v_j| + the P V terms; the bf16 rounding of a value within E32 of ref is within half an
     ulp of |ref| + E32:  bound = E32 + ulp_bf16(|ref| + E32) / 2.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from oracle.attention_bounds import EX2_REL, FTZ, _bf16, scale_log2e
from oracle.bounds import C_ACC, U, bf16_ulp

Tensor = torch.Tensor

KB = 16                     # keys per block of both passes (HM_KB)
LOG2F_ABS = 2.0 ** -22      # __log2f on [0.5, 2]: absolute error (CUDA C++ Programming Guide)


def _coef(post: Tensor, H: int) -> Tuple[Tensor, Tensor]:
    """coef_g = mean over f of post[g][f] in fp64, and |coef~_g - coef_g|: coef~ is the kernel's own fp32 value, a
    sequential sum over f divided by H, both IEEE operations, so it is computed here exactly as the kernel does."""
    c32 = torch.zeros(H, dtype=torch.float32, device=post.device)
    for f in range(H):
        c32 = c32 + post[:, f].float()
    c32 = c32 / H
    coef = post.double().sum(1) / H
    return coef, (c32.double() - coef).abs()


def _eps32(eps: float) -> float:
    return torch.tensor(eps, dtype=torch.float32).item()


def headmix_reference(qkv: Tensor, B: int, N: int, H: int, dh: int, scale: float, pre: Optional[Tensor],
                      post: Tensor, ln: Optional[tuple] = None, *, elems: int = 1 << 23) -> Tuple[Tensor, Tensor]:
    """(ref, bound) [B N, H dh] of b200vit_attention_headmix_ex on qkv[B N, 3 H dh] (bf16): pre (fp32 [H, H] or None)
    mixes the scores, post (fp32 [H, H], [input head, output head]) the probabilities, ln = (gamma, beta, eps) or None
    the LayerNorm over heads.  Query rows go in chunks of about `elems` elements per [B, H, rows, N] tensor, so that
    N = 16384 with H = 16 fits on the device."""
    dev = qkv.device
    x = qkv.view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)               # [3, B, H, N, dh]
    q, k, v = x[0].double(), x[1].double(), x[2].double()
    kT, kaT, vabs = k.transpose(-1, -2), k.abs().transpose(-1, -2), v.abs()
    c = scale_log2e(scale)
    post64 = post.double().to(dev)
    pre64 = None if pre is None else pre.double().to(dev)
    if ln is not None:
        gam, bet = ln[0].double().to(dev).view(1, H, 1, 1), ln[1].double().to(dev).view(1, H, 1, 1)
        eps = _eps32(ln[2])
        coef, dcoef = _coef(post.to(dev), H)
    nb = -(-N // KB)
    pad = nb * KB - N
    vb = torch.nn.functional.pad(v, (0, 0, 0, pad)).view(B, H, nb, KB, dh)
    ref = torch.empty(B, H, N, dh, dtype=torch.float64, device=dev)
    bound = torch.empty_like(ref)
    rows = max(1, min(N, elems // max(1, B * H * max(N, nb * dh))))
    for r0 in range(0, N, rows):
        r1 = min(N, r0 + rows)
        qc = q[:, :, r0:r1]
        # 1. scores
        s = (qc @ kT) * c                                               # [B, H, R, N]
        ds = c * (C_ACC * dh + 2) * U * (qc.abs() @ kaT) + 2 * U * s.abs()
        # 2. pre-mix: the chain over h, its partial sums replayed
        if pre64 is not None:
            sm, dsm, ps = torch.zeros_like(s), torch.zeros_like(s), torch.zeros_like(s)
            for h in range(H):
                sm = sm + pre64[h].view(1, H, 1, 1) * s[:, h:h + 1]
                ps += sm.abs()
                dsm = dsm + pre64[h].abs().view(1, H, 1, 1) * ds[:, h:h + 1]
            dsm = dsm + U * ps
            del ps
        else:
            sm, dsm = s, ds
        del s, ds
        # 3. lse
        M = sm.amax(-1, keepdim=True)
        dsmax = dsm.amax(-1, keepdim=True)
        lse = torch.logsumexp(sm * math.log(2), -1, keepdim=True) / math.log(2)
        w = torch.exp2(sm - lse)                                        # the exact probabilities
        L = torch.exp2(lse - M)
        xp = torch.nn.functional.pad(sm, (0, pad), value=-math.inf).view(*sm.shape[:-1], nb, KB)
        bsum = torch.exp2(xp - M[..., None]).sum(-1)                    # [B, H, R, nb]
        P = bsum.cumsum(-1)
        bmax = xp.amax(-1)
        run = bmax.cummax(-1).values
        Pprev = torch.nn.functional.pad(P[..., :-1], (1, 0))
        rise = torch.zeros_like(bmax, dtype=torch.bool)
        rise[..., 1:] = bmax[..., 1:] + 2 * dsmax >= run[..., :-1]
        Prise = torch.where(rise, Pprev, torch.zeros_like(Pprev)).sum(-1, keepdim=True)
        rho = ((w * (torch.exp2(dsm + U * (M - sm + 2 * dsmax)) * (1 + EX2_REL) ** 2 - 1)).sum(-1, keepdim=True)
               + ((EX2_REL + U) * Prise + U * (6 * L + P.sum(-1, keepdim=True))) / L + 2 * N * FTZ)
        del xp, bsum, P, bmax, run, Pprev, rise
        dlse = -torch.log2((1 - rho).clamp_min(1e-300)) + LOG2F_ABS + 4 * U * (lse - M + 2 * dsmax) + U * lse.abs()
        # 4. probabilities
        xx = sm - lse
        dx = dsm + dlse + U * (xx.abs() + dsm + dlse)
        del sm, dsm
        hi = w * torch.exp2(dx) * (1 + EX2_REL)
        lo = w * torch.exp2(-dx) * (1 - EX2_REL)
        lo = torch.where(lo < FTZ, torch.zeros_like(lo), lo)
        dp = torch.maximum(hi - w, w - lo)
        del hi, lo, dx, xx
        # 5. post-mix (every output head at once) and the LayerNorm over heads
        acc, pacc, dacc = torch.zeros_like(w), torch.zeros_like(w), torch.zeros_like(w)
        for g in range(H):
            acc = acc + post64[g].view(1, H, 1, 1) * w[:, g:g + 1]
            pacc += acc.abs()
            dacc = dacc + post64[g].abs().view(1, H, 1, 1) * dp[:, g:g + 1]
        if ln is not None:
            # d_f = sum_g (post_gf - coef_g) p_g: acc and mean see the same p~, so its error enters through
            # post - coef (0 for equal heads), the kernel's own coef~ through |coef~ - coef| p~
            mean, pm, dmix = torch.zeros_like(w[:, :1]), torch.zeros_like(w[:, :1]), torch.zeros_like(w)
            dcm, dabs = torch.zeros_like(w[:, :1]), dacc.clone()
            for g in range(H):
                mean = mean + coef[g].item() * w[:, g:g + 1]
                pm += mean.abs()
                dmix = dmix + (post64[g] - coef[g]).abs().view(1, H, 1, 1) * dp[:, g:g + 1]
                dcm = dcm + dcoef[g].item() * (w[:, g:g + 1] + dp[:, g:g + 1])
                dabs = dabs + abs(coef[g].item()) * dp[:, g:g + 1]
            d = acc - mean
            dd = dmix + dcm + U * (pacc + pm + H * dabs)
            dd = dd + U * (d.abs() + dd)
            del acc, dacc, pacc, mean, pm, dmix, dcm, dabs
            sq = d * d
            V = sq.sum(1, keepdim=True)
            S = (2 * d.abs() * dd + dd * dd).sum(1, keepdim=True)
            dV = S + U * (sq.cumsum(1).sum(1, keepdim=True) + H * S)
            del sq, S
            a = V / H + eps
            da = dV / H * (1 + 2 * U) + U * V / H + U * a * (1 + U)
            rel = (1.0 / torch.sqrt((1.0 - da / a).clamp_min(1e-300)) - 1.0) * (1 + 4 * U) + 4 * U
            rstd = 1.0 / torch.sqrt(a)
            xh = d * rstd
            dxh = rstd * (1 + rel) * dd + xh.abs() * rel
            dxh = dxh + U * (xh.abs() + dxh)
            pp = xh * gam + bet
            dpp = gam.abs() * dxh
            dpp = dpp + U * (pp.abs() + dpp)
            del d, dd, V, dV, a, da, rel, rstd, xh, dxh
        else:
            pp, dpp = acc, dacc * (1 + H * U) + U * pacc
        del w, dp
        # 6. bf16 replay of P''
        pb = _bf16(pp)
        A = torch.maximum(_bf16(pp + dpp) - pb, pb - _bf16(pp - dpp))
        del pp, dpp
        # 7. P V in 16-key steps
        out = pb @ v
        e = A @ vabs
        step = (C_ACC * KB + 2) * U * ((pb.abs() + A) @ vabs)
        pbb = torch.nn.functional.pad(pb, (0, pad)).view(*pb.shape[:-1], nb, KB)
        part = torch.einsum('bhrnk,bhnkd->bhrnd', pbb, vb).cumsum(3).abs().sum(3)
        e32 = e + step + U * part + U * nb * e
        del pb, A, pbb
        ref[:, :, r0:r1] = out
        bound[:, :, r0:r1] = e32 + 0.5 * bf16_ulp(out.abs() + e32)
    back = lambda t: t.permute(0, 2, 1, 3).reshape(B * N, H * dh)     # noqa: E731
    return back(ref), back(bound)


def headmix_inputs(kind: str, B: int, N: int, H: int, dh: int, *, seed: int = 0, device="cpu"):
    """Seeded (qkv, pre, post, (gamma, beta, eps)): qkv from attention_bounds.qkv_inputs for the kinds of
    attention_bounds.KINDS, pre and post N(0, 1), gamma near 1, beta small; kind "near_equal" is qkv "normal" with
    post = 1 / H + 1e-3 noise, so that the heads after the post-mix are nearly equal and the LayerNorm's variance is
    tiny (rstd near 1 / sqrt(eps))."""
    from oracle.attention_bounds import qkv_inputs
    qkv = qkv_inputs("normal" if kind == "near_equal" else kind, [N] * B, H, dh, seed=seed, device=device)
    g = torch.Generator(device=device).manual_seed(seed + 1)
    pre = torch.randn(H, H, generator=g, device=device)
    post = torch.randn(H, H, generator=g, device=device)
    if kind == "near_equal":
        post = 1.0 / H + 1e-3 * post
    ln = (1 + 0.2 * torch.randn(H, generator=g, device=device), 0.1 * torch.randn(H, generator=g, device=device), 1e-5)
    return qkv, pre, post, ln
