"""The error bound of oracle/headmix_bounds.py is neither loose nor broken, and attention_reference's key mask models
the axial kernel's empty rows (CPU only).

Not broken: an fp32 emulation of headmix.cu in the kernel's order passes its bound -- the scores fl(fl(q k) c), the
pre-mix as an fma chain over the heads, pass 1 over 16-key blocks (per lane 4 keys, 2 shuffle levels, the running
max / sum merge), lse = mx + log2(sum), pass 2 p = ex2(s' - lse), the coef / mean / acc / var chains and rsqrt of the
LayerNorm over heads, P'' in bf16, P V in 16-key steps into one fp32 accumulator, the bf16 output -- on
attention_bounds.KINDS and on near-equal heads, for H in {1, 2, 3, 5, 8, 9, 16} in all four modes.
Not loose: the median fp32 part of the bound is a small fraction of the output's half ulp, and each planted defect is
flagged, among them the two the former criterion (close_to) accepts."""
import math

import pytest
import torch

from oracle import attention_bounds as AB
from oracle import bounds as Bd
from oracle import headmix_bounds as HB
from test_attention_family_bounds import fma32, fma_chain, fp32_part

MODES = {"post": (False, False), "post_ln": (False, True), "pre_post": (True, False), "pre_post_ln": (True, True)}
DH = 32


def ex2(x):
    """ex2.approx.ftz.f32, nearly: fp32 exp2 with results below 2^-126 flushed to 0."""
    r = torch.exp2(x.float())
    return torch.where(r < AB.FTZ, torch.zeros_like(r), r)


def headmix_emulate(qkv, B, N, H, dh, scale, pre, post, ln, defect=None):
    """headmix.cu's arithmetic in fp32, in its order (module docstring).  Returns the fp32 output [B N, H dh] before its
    bf16 rounding."""
    x = qkv.float().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    nb = -(-N // 16)
    NK, NR = nb * 16, -(-N // 16) * 16            # keys zero-filled to whole blocks, rows to whole 16-row groups
    q = torch.zeros(B, H, NR, dh)
    q[:, :, :N] = x[0]
    k, v = torch.zeros(B, H, NK, dh), torch.zeros(B, H, NK, dh)
    k[:, :, :N], v[:, :, :N] = x[1], x[2]
    c = torch.tensor(AB.scale_log2e(scale), dtype=torch.float32)
    if defect == "scale":
        c = c * 1.001
    s = (q @ k.transpose(-1, -2)) * c                                   # [B, H, NR, NK]
    sm = fma_chain(pre.view(1, H, H, 1, 1), s[:, :, None], 1) if pre is not None else s
    valid = torch.arange(NK) < N
    # pass 1
    x1 = s if defect == "no_pre_pass1" else sm
    x1 = torch.where(valid, x1, torch.full_like(x1, -math.inf))
    m = ssum = None
    for kb in range(nb - 1 if defect == "drop_tail_block" else nb):
        blk = x1[..., 16 * kb:16 * kb + 16]
        bm = blk.amax(-1)
        e = ex2(blk - bm[..., None])
        lane = [((e[..., 2 * t] + e[..., 2 * t + 1]) + e[..., 8 + 2 * t]) + e[..., 9 + 2 * t] for t in range(4)]
        bs = (lane[0] + lane[1]) + (lane[2] + lane[3])
        if kb == 0:
            m, ssum = bm, bs
        else:
            mx = torch.maximum(m, bm)
            ssum = ssum * ex2(m - mx) + bs * ex2(bm - mx)
            m = mx
    lse = m + torch.log2(ssum)                                          # [B, H, NR]
    if defect == "lse_row8":
        lse = lse[..., torch.arange(NR) ^ 8]
    # pass 2
    p = torch.where(valid, ex2(sm - lse[..., None]), torch.zeros_like(sm))
    acc = fma_chain(post.view(1, H, H, 1, 1), p[:, :, None], 1)         # [B, f, NR, NK]
    if ln is not None:
        gam, bet, eps = ln
        cs = torch.zeros(H)
        for f in range(H):
            cs = cs + post[:, f]
        coef = cs / H
        mean = fma_chain(coef.view(1, H, 1, 1), p, 1)[:, None]
        d = acc - mean
        var = fma_chain(d, d, 1)[:, None]
        var = var / (H - 1 if defect == "var_h1" else H)
        e32 = torch.tensor(eps, dtype=torch.float32)
        rstd = 1.0 / (var.sqrt() + e32) if defect == "eps_outside" else torch.rsqrt(var + e32)
        if defect == "gamma_next":
            gam = gam.roll(-1)
        acc = fma32((d * rstd), gam.view(1, H, 1, 1), bet.view(1, H, 1, 1))
    pb = torch.where(valid, acc, torch.zeros_like(acc)).bfloat16().double()
    o = torch.zeros(B, H, NR, dh)
    for kb in range(nb):
        o = (o.double() + pb[..., 16 * kb:16 * kb + 16] @ v[:, :, 16 * kb:16 * kb + 16].double()).float()
    if defect == "head":
        o[:, H // 3] *= 1.005
    return o[:, :, :N].permute(0, 2, 1, 3).reshape(B * N, H * dh)


def close_to(out, ref):
    """The former criterion of test_gpu_attention_exact.py (and about that of test_gpu_deepvit.py / test_gpu_cait.py):
    True if it accepts `out` against the reference `ref`."""
    tol = 1e-2 * ref.abs().max().item() + 1e-3
    err = (out.double() - ref).abs()
    return bool(err.max().item() <= 2 * tol and (err <= tol + 1e-2 * ref.abs()).double().mean().item() > 0.999)


def case(kind, B, N, H, mode, seed, defect=None):
    qkv, pre, post, ln = HB.headmix_inputs(kind, B, N, H, DH, seed=seed)
    use_pre, use_ln = MODES[mode]
    pre, ln = (pre if use_pre else None), (ln if use_ln else None)
    scale = DH ** -0.5
    ref, bound = HB.headmix_reference(qkv, B, N, H, DH, scale, pre, post, ln)
    got = headmix_emulate(qkv, B, N, H, DH, scale, pre, post, ln, defect)
    return got, ref, bound


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("H", [1, 2, 3, 5, 8, 9, 16])
@pytest.mark.parametrize("kind", AB.KINDS + ("near_equal",))
def test_headmix_fp32_emulation_passes(kind, H, mode):
    if kind == "near_equal" and not MODES[mode][1]:
        pytest.skip("near-equal heads matter to the LayerNorm only")
    worst, parts = 0.0, []
    for N in (1, 15, 16, 17, 64, 65, 197):
        got, ref, bound = case(kind, 1, N, H, mode, seed=N + 31 * H)
        worst = max(worst, Bd.check(got.bfloat16(), ref, bound, f"headmix {kind} H{H} {mode} N{N}"))
        parts.append(fp32_part(ref, bound))
    med = torch.cat(parts).median().item()
    print(f"headmix {kind} H{H} {mode}: worst {worst:.3f}, median fp32 part {med:.4f} half ulps")
    assert med < MEDIAN_FP32_PART[mode]


# The largest median over a case's outputs of (bound - half ulp) / half ulp measured over the sweep above, per mode:
# post 0.084, post_ln 0.41, pre_post 0.56, pre_post_ln 1.91 (all at H = 16; below 0.1 in every mode at H <= 3).  Almost
# all of it is the replay term sum A |v| of step 6: the wgmma score term (C_ACC dh + 2) u sum|q||k|, summed over 16
# heads by the pre-mix and divided by the LayerNorm's spread, moves a few per cent of the P'' intervals across a bf16
# rounding boundary.  The limits keep a margin of about 1.5.
MEDIAN_FP32_PART = {"post": 0.15, "post_ln": 0.6, "pre_post": 0.85, "pre_post_ln": 2.8}

# defect: (kind, N, H, mode, does the former criterion accept it)
DEFECTS = {
    "scale": ("normal", 65, 16, "post", True),                # the score scale off by 0.1 %
    "head": ("normal", 65, 16, "post_ln", True),              # one output head of 16 off by 0.5 %
    "lse_row8": ("normal", 65, 4, "post", False),             # the lse of the row 8 apart
    "no_pre_pass1": ("normal", 65, 4, "pre_post", False),     # pass 1 without the pre-mix
    "drop_tail_block": ("normal", 65, 4, "post", False),      # pass 1 missing the last, partial 16-key block
    "var_h1": ("normal", 65, 4, "post_ln", False),            # the LayerNorm variance over H - 1
    "eps_outside": ("near_equal", 65, 4, "post_ln", False),   # eps added outside the square root
    "gamma_next": ("normal", 65, 4, "post_ln", False),        # the neighbouring head's gamma
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_headmix_planted_defect_is_flagged(defect):
    kind, N, H, mode, old_accepts = DEFECTS[defect]
    clean, ref, bound = case(kind, 2, N, H, mode, seed=5)
    Bd.check(clean.bfloat16(), ref, bound, "clean")
    got, _, _ = case(kind, 2, N, H, mode, seed=5, defect=defect)
    ratio = Bd.excess(got.bfloat16(), ref, bound)
    old = close_to(got.bfloat16(), clean)
    print(f"headmix {defect}: worst |got - ref| / bound {ratio:.2f}, former criterion accepts: {old}")
    assert ratio > 1, defect
    assert old == old_accepts, defect


# ------------------------------------------------------------------------------------------------ axial key mask
def axial_emulate(q, k, v, scale, keep, zero):
    """attention_tile_kernel's arithmetic for one tile per sequence (n <= 64) in fp32: kept keys fl(s c), the others
    -inf; a row with a kept key gets ex2(s - max), one without one 0 (zero) or 1 for every key of its window; l the sum,
    P in bf16, O = P V in fp32, O fl(1 / l) (0 where l = 0)."""
    c = torch.tensor(AB.scale_log2e(scale), dtype=torch.float32)
    s = (q.float() @ k.float().transpose(-1, -2)) * c
    kp = keep[:, None, :].expand_as(s)
    s = torch.where(kp, s, torch.full_like(s, -math.inf))
    has = keep.any(-1)[:, None, None]
    mx = s.amax(-1, keepdim=True)
    e = torch.where(has, ex2(s - torch.where(has, mx, torch.zeros_like(mx))), torch.zeros_like(s) if zero else
                    torch.ones_like(s))
    l = e.sum(-1, keepdim=True)
    o = (e.bfloat16().double() @ v.double()).float()
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    return o * inv


@pytest.mark.parametrize("n", [1, 2, 5, 8, 17, 33, 64])
def test_axial_key_mask_and_empty_rows(n):
    G, dh = 6, 64
    x = AB.qkv_inputs("normal", [n] * G, 1, dh, seed=n).view(G, n, 3, dh)
    q, k, v = x[..., 0, :], x[..., 1, :], x[..., 2, :]
    g = torch.Generator().manual_seed(n)
    keep = torch.rand(G, n, generator=g) > 0.4
    keep[:, 0] = True
    keep[1] = False                                   # sequence 1: every key masked
    keep[4] = False
    scale = dh ** -0.5
    for zero in (True, False):
        ref, bound = AB.attention_reference(q, k, v, scale, key_mask=keep, zero_masked_rows=zero)
        Bd.check(axial_emulate(q, k, v, scale, keep, zero).bfloat16(), ref, bound, f"axial n{n} zero={zero}")
        if zero:
            assert (ref[1] == 0).all() and (bound[1] == 0).all()
        else:
            assert torch.allclose(ref[1], v[1].double().mean(0).expand(n, dh), rtol=0, atol=1e-12)
    # a mask that keeps every key is the unmasked reference, bit for bit
    every = torch.ones(G, n, dtype=torch.bool)
    for a, b in zip(AB.attention_reference(q, k, v, scale, key_mask=every), AB.attention_reference(q, k, v, scale)):
        assert torch.equal(a, b)
