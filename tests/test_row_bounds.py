"""The error bounds of oracle/row_bounds.py are neither loose nor tight (CPU only).

Tight: an fp32 emulation of each row kernel's arithmetic, in its order -- the lane chains and butterflies of
ln_row_stats, emit_row_stats and rmsnorm_heads_kernel, the output formulas -- passes the checker.
Loose: each defect a row kernel could plausibly have, planted into that emulation, is flagged: an unbiased variance,
eps outside the sqrt, gamma / beta one column off, the neighbouring head's gamma, the neighbouring token's or group's
positional row, a position on a class row that has none, statistics of the unrounded values or of the next row, a mean
pool over every row, a one-pass head variance on ill-conditioned heads, sqrt(dh) rounded to an integer."""
import math

import pytest
import torch

from oracle import row_bounds as RB

EPS = 1e-5
f32 = torch.float32


def flagged(got, ref, bound):
    return RB.excess(got, ref, bound) > 1.0


def butterfly(s):
    """xor butterfly over the last dim (the lanes) in fp32; returns lane 0's total."""
    lanes = s.shape[-1]
    idx = torch.arange(lanes)
    o = lanes // 2
    while o:
        s = s + s[..., idx ^ o]
        o //= 2
    return s[..., 0]


def lanes_of(x, vec):
    """x[M, D] -> ([M, K, 32, 4] or [M, K, 32], valid mask): the elements lane l takes at step k (zero padded)."""
    M, D = x.shape
    w = 128 if vec else 32
    K = -(-D // w)
    xp = torch.zeros(M, K * w, dtype=x.dtype)
    xp[:, :D] = x
    valid = torch.zeros(K * w, dtype=torch.bool)
    valid[:D] = True
    shape = (M, K, 32, 4) if vec else (M, K, 32)
    return xp.view(shape), valid.view(shape[1:])


def chain(t):
    """the lane chain s += t[:, k] over k, in fp32; t [M, K, 32]."""
    s = torch.zeros(t.shape[0], t.shape[2], dtype=f32)
    for k in range(t.shape[1]):
        s = s + t[:, k]
    return s


def quad(v):
    return (v[..., 0] + v[..., 1]) + (v[..., 2] + v[..., 3])


def ln_stats32(x, eps=EPS, unbiased=False, eps_outside=False):
    """ln_row_stats in fp32: (mean [M, 1], rstd [M, 1])."""
    D = x.shape[1]
    vec = D % 4 == 0
    xv, valid = lanes_of(x, vec)
    mean = butterfly(chain(quad(xv) if vec else xv)) / D
    mb = mean.view((-1,) + (1,) * (xv.dim() - 1))
    a = torch.where(valid, xv - mb, torch.zeros((), dtype=f32))
    var = butterfly(chain(quad(a * a) if vec else a * a)) / (D - 1 if unbiased else D)
    rstd = torch.rsqrt(var) + eps if eps_outside else torch.rsqrt(var + eps)
    return mean[:, None], rstd[:, None]


def layernorm32(x, g, b, **kw):
    mean, rstd = ln_stats32(x, **kw)
    y = (x - mean) * rstd * g
    return y + b if b is not None else y


def row_stats32(y):
    """emit_row_stats in fp32 on the bf16 copy of the fp32 rows y: [M, 2]."""
    xb = y.bfloat16().float()
    D = y.shape[1]
    vec = D % 4 == 0
    xv, _ = lanes_of(xb, vec)
    if not vec:
        return torch.stack([butterfly(chain(xv)), butterfly(chain(xv * xv))], 1)
    s2 = torch.zeros(xv.shape[0], 32, dtype=f32)
    for k in range(xv.shape[1]):                     # fma(a0, a0, fma(a1, a1, fma(a2, a2, fma(a3, a3, s2))))
        for j in (3, 2, 1, 0):
            s2 = s2 + xv[:, k, :, j] * xv[:, k, :, j]  # exact squares: the fma rounds once, like this add
    return torch.stack([butterfly(chain(quad(xv))), butterfly(s2)], 1)


def head_lanes(x):
    """x[T, H, dh] -> [T, H, LPH, 8] (lane sub holds values 8 sub .. 8 sub + 7; idle lanes zero), active mask."""
    T, H, dh = x.shape
    lph = RB.HEAD_LANES[dh]
    v = torch.zeros(T, H, lph * 8, dtype=x.dtype)
    v[..., :dh] = x
    act = torch.arange(lph) < dh // 8
    return v.view(T, H, lph, 8), act


def fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def rmsnorm_heads32(x, g, sqrt_dh=None):
    """rmsnorm_heads_kernel in fp32; x [T, H, dh] bf16, g [H, dh] -> bf16."""
    dh = x.shape[-1]
    v, _ = head_lanes(x.float())
    ss = torch.zeros(v.shape[:3], dtype=f32)
    for i in range(4):
        ss = fma32(v[..., 2 * i], v[..., 2 * i], fma32(v[..., 2 * i + 1], v[..., 2 * i + 1], ss))
    c = torch.tensor(math.sqrt(dh) if sqrt_dh is None else sqrt_dh, dtype=f32)
    inv = c / torch.sqrt(butterfly(ss)).clamp_min(1e-12)
    return (x.float() * inv[..., None] * g).bfloat16()


def layernorm_heads32(x, g, eps=EPS, one_pass=False, unbiased=False):
    """the LN branch of rmsnorm_heads_kernel in fp32 (two-pass; one_pass: E[v^2] - mean^2) -> bf16."""
    dh = x.shape[-1]
    v, act = head_lanes(x.float())
    k = torch.tensor(1.0 / dh, dtype=f32)
    s1 = torch.zeros(v.shape[:3], dtype=f32)
    for i in range(4):
        s1 = s1 + (v[..., 2 * i] + v[..., 2 * i + 1])
    mean = butterfly(s1) * k
    if one_pass:
        ss = torch.zeros(v.shape[:3], dtype=f32)
        for i in range(4):
            ss = fma32(v[..., 2 * i], v[..., 2 * i], fma32(v[..., 2 * i + 1], v[..., 2 * i + 1], ss))
        var = (butterfly(ss) * k - mean * mean).clamp_min(0)
    else:
        a = v - mean[..., None, None]
        q = torch.zeros(v.shape[:3], dtype=f32)
        for i in range(4):
            q = fma32(a[..., 2 * i], a[..., 2 * i], fma32(a[..., 2 * i + 1], a[..., 2 * i + 1], q))
        q = torch.where(act, q, torch.zeros((), dtype=f32))
        var = butterfly(q) * (torch.tensor(1.0 / (dh - 1), dtype=f32) if unbiased else k)
    inv = torch.rsqrt(var + eps)
    return ((x.float() - mean[..., None]) * inv[..., None] * g).bfloat16()


def gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------- row LayerNorm
@pytest.mark.parametrize("D", [4, 12, 50, 64, 200, 768, 1280])
def test_layernorm_emulation_passes(D):
    g = gen(D)
    x = torch.randn(37, D, generator=g) * 3 + 1
    gm, b = torch.randn(D, generator=g), torch.randn(D, generator=g)
    y = layernorm32(x, gm, b)
    RB.check(y, *RB.layernorm_reference(x, gm, b), "fp32")
    RB.check(y.bfloat16(), *RB.layernorm_reference(x, gm, b, bf16_out=True), "bf16")
    y0 = layernorm32(x, gm, None)
    RB.check(y0, *RB.layernorm_reference(x, gm, None), "no beta")


@pytest.mark.parametrize("D", [64, 50])
def test_layernorm_unbiased_variance_is_flagged(D):
    g = gen(1)
    x = torch.randn(16, D, generator=g)
    gm, b = torch.randn(D, generator=g), torch.randn(D, generator=g)
    ref, bound = RB.layernorm_reference(x, gm, b)
    assert flagged(layernorm32(x, gm, b, unbiased=True), ref, bound)


def test_layernorm_eps_outside_the_sqrt_is_flagged_where_var_is_near_eps():
    g = gen(2)
    D = 256
    x = torch.randn(16, D, generator=g) * 3e-3                 # var ~ 1e-5 ~ eps
    gm, b = torch.randn(D, generator=g), torch.randn(D, generator=g)
    ref, bound = RB.layernorm_reference(x, gm, b)
    RB.check(layernorm32(x, gm, b), ref, bound)
    assert flagged(layernorm32(x, gm, b, eps_outside=True), ref, bound)


def test_layernorm_gamma_or_beta_one_column_off_is_flagged():
    g = gen(3)
    D = 192
    x = torch.randn(16, D, generator=g)
    gm, b = torch.randn(D, generator=g), torch.randn(D, generator=g)
    for bf in (False, True):
        ref, bound = RB.layernorm_reference(x, gm, b, bf16_out=bf)
        for gg, bb in ((torch.roll(gm, 1), b), (gm, torch.roll(b, 1))):
            y = layernorm32(x, gg, bb)
            assert flagged(y.bfloat16() if bf else y, ref, bound)


def test_layernorm_row_gather_and_wide_rows():
    g = gen(4)
    x = torch.randn(40, 72, generator=g)
    gm = torch.randn(64, generator=g)
    rows = torch.tensor([5, 0, 39, 7], dtype=torch.int32)
    y = layernorm32(x[rows.long(), :64], gm, None)
    RB.check(y, *RB.layernorm_reference(x, gm, None, row_index=rows))
    assert flagged(layernorm32(x[(rows.long() + 1) % 40, :64], gm, None), *RB.layernorm_reference(x, gm, None, row_index=rows))


# ---------------------------------------------------------------------------------------------------- token assembly
def embed32(y, gm, b, cls, pos, groups, n, ncls, tail=None, pos_period=1, pos_stride=0, cls_pos=True,
            cls_pos_defect=False, pos_shift=0, period_defect=False):
    """embed_tokens_kernel in fp32 (+ planted defects)."""
    D = y.shape[1]
    ntail = 0 if tail is None else tail.shape[0]
    N = ncls + n + ntail
    x = torch.zeros(groups, N, D)
    ln = layernorm32(y, gm, b).view(groups, n, D) if gm is not None else y.view(groups, n, D)
    for bi in range(groups):
        blk = ((bi + 1 if period_defect else bi) % pos_period) * pos_stride
        for t in range(N):
            if t < ncls:
                v = cls[t]
                if pos is not None and (cls_pos or cls_pos_defect):
                    v = v + pos[blk + t]
            elif t >= ncls + n:
                v = tail[t - ncls - n]
            else:
                v = ln[bi, t - ncls]
                if pos is not None:
                    v = v + pos[blk + t - (0 if cls_pos else ncls) + pos_shift]
            x[bi, t] = v
    return x.view(-1, D)


CASES = {   # (D, groups, n, ncls, ntail, LN, POS, pos_period, cls_pos)
    "vit": (192, 3, 9, 1, 0, True, True, 1, True),
    "odd_d": (50, 2, 7, 2, 0, True, True, 1, True),
    "registers": (64, 2, 6, 0, 4, True, True, 1, True),
    "no_ln": (96, 3, 5, 1, 0, False, True, 1, True),
    "no_pos": (64, 2, 5, 1, 0, True, False, 1, True),
    "grouped_cls_pos": (64, 6, 4, 1, 0, True, True, 3, True),
    "grouped_no_cls_pos": (64, 6, 4, 1, 0, True, True, 3, False),
}


def embed_inputs(case, seed=0):
    D, groups, n, ncls, ntail, ln, has_pos, period, cls_pos = CASES[case]
    g = gen(seed)
    stride = n + (ncls if cls_pos else 0)
    y = torch.randn(groups * n, D, generator=g)
    pos = torch.randn(period * stride + 1, D, generator=g) if has_pos else None
    return dict(y=y, gm=torch.randn(D, generator=g) if ln else None, b=torch.randn(D, generator=g) if ln else None,
                cls=torch.randn(ncls, D, generator=g) if ncls else None, pos=pos, groups=groups, n=n, ncls=ncls,
                tail=torch.randn(ntail, D, generator=g) if ntail else None, pos_period=period,
                pos_stride=stride if period > 1 else 0, cls_pos=cls_pos)


def embed_ref(a):
    return RB.embed_tokens_reference(a["y"], a["gm"], a["b"], a["cls"], a["pos"], a["groups"], a["n"], a["ncls"],
                                     tail=a["tail"], pos_period=a["pos_period"], pos_stride=a["pos_stride"],
                                     cls_pos=a["cls_pos"])


@pytest.mark.parametrize("case", list(CASES))
def test_embed_tokens_emulation_passes(case):
    a = embed_inputs(case)
    x = embed32(**a)
    ref, bound = embed_ref(a)
    RB.check(x, ref, bound, case)
    RB.check(row_stats32(x), *RB.row_stats_reference(x.bfloat16()), case + " stats")


def test_embed_tokens_defects_are_flagged():
    a = embed_inputs("vit")
    ref, bound = embed_ref(a)
    assert flagged(embed32(**a, pos_shift=1), ref, bound)                         # neighbouring token's position
    assert flagged(embed32(**dict(a, gm=torch.roll(a["gm"], 1))), ref, bound)     # gamma one column off
    assert flagged(embed32(**dict(a, b=torch.roll(a["b"], 1))), ref, bound)       # beta one column off
    a = embed_inputs("grouped_cls_pos")
    assert flagged(embed32(**a, period_defect=True), *embed_ref(a))               # another group's positional block
    a = embed_inputs("grouped_no_cls_pos")
    assert flagged(embed32(**a, cls_pos_defect=True), *embed_ref(a))              # position on a class row


def varlen_inputs(seed=0):
    g = gen(seed)
    p, D = 4, 64
    dims = [(8, 12), (4, 4), (12, 8), (4, 20)]
    lengths = [(h // p) * (w // p) for h, w in dims]
    T = sum(lengths)
    return dict(y=torch.randn(T, D, generator=g), gm=torch.randn(D, generator=g), ph=torch.randn(5, D, generator=g),
                pw=torch.randn(6, D, generator=g), lengths=lengths, dims=dims, p=p)


def varlen32(a, transpose=False):
    ln = layernorm32(a["y"], a["gm"], None)
    r, c = RB.varlen_grid(a["lengths"], a["dims"], a["p"], "cpu")
    if transpose:
        r, c = c, r
    return (ln + a["ph"][r]) + a["pw"][c]


def test_embed_varlen_emulation_passes_and_a_transposed_grid_is_flagged():
    a = varlen_inputs()
    ref, bound = RB.embed_varlen_reference(a["y"], a["gm"], a["ph"], a["pw"], a["lengths"], a["dims"], a["p"])
    x = varlen32(a)
    RB.check(x, ref, bound)
    RB.check(row_stats32(x), *RB.row_stats_reference(x.bfloat16()))
    assert flagged(varlen32(a, transpose=True), ref, bound)


# ---------------------------------------------------------------------------------------------------- row statistics
@pytest.mark.parametrize("D", [768, 192, 50])
def test_row_stats_emulation_passes_and_unrounded_or_next_row_sums_are_flagged(D):
    g = gen(D)
    y = torch.randn(64, D, generator=g) * 2 + 0.5
    ref, bound = RB.row_stats_reference(y.bfloat16())
    st = row_stats32(y)
    RB.check(st, ref, bound)
    y64 = y.double()
    unrounded = torch.stack([y64.sum(1), (y64 * y64).sum(1)], 1)
    # every row's sum of squares, and nearly every row's sum, of the fp32 values falls outside the bound
    d = (unrounded - ref).abs() / bound
    assert (d[:, 1] > 1).all() and (d[:, 0] > 1).float().mean() > 0.9
    nxt = st.clone()
    nxt[10] = st[11]
    assert flagged(nxt, ref, bound)


def test_row_stats_bound_is_depth_based():
    assert RB.stats_depths(768) == (13, 29) and RB.stats_depths(50) == (7, 7)
    assert RB.ln_depth(768) == 13 and RB.ln_depth(4096) == 39 and RB.ln_depth(50) == 7


# ---------------------------------------------------------------------------------------------------- head norms
def heads(T, H, dh, seed, scale=1.0, shift=0.0):
    g = gen(seed)
    return (torch.randn(T, H, dh, generator=g) * scale + shift).bfloat16(), torch.randn(H, dh, generator=g)


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_rmsnorm_heads_emulation_passes_and_defects_are_flagged(dh):
    x, gm = heads(64, 5, dh, dh)
    x[3, 2] = 0                                                  # all-zero head: exactly 0
    ref, bound = RB.rmsnorm_heads_reference(x, gm)
    y = rmsnorm_heads32(x, gm)
    RB.check(y, ref, bound)
    assert (y[3, 2] == 0).all()
    assert flagged(rmsnorm_heads32(x, torch.roll(gm, 1, 0)), ref, bound)          # the neighbouring head's gamma
    assert flagged(rmsnorm_heads32(x, torch.roll(gm, 1, 1)), ref, bound)          # gamma one column off
    if dh == 80:
        assert flagged(rmsnorm_heads32(x, gm, sqrt_dh=9.0), ref, bound)           # sqrt(80) rounded to 9


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_layernorm_heads_emulation_passes_and_defects_are_flagged(dh):
    x, gm = heads(64, 5, dh, dh + 1)
    x[1, 1] = 0.75                                               # constant head
    ref, bound = RB.layernorm_heads_reference(x, gm)
    RB.check(layernorm_heads32(x, gm), ref, bound)
    assert flagged(layernorm_heads32(x, gm, unbiased=True), ref, bound)
    assert flagged(layernorm_heads32(x, torch.roll(gm, 1, 0)), ref, bound)


@pytest.mark.parametrize("dh", [64, 80, 128])
def test_one_pass_head_variance_is_flagged_on_ill_conditioned_heads(dh):
    """|mean| / std of several hundred: E[v^2] - mean^2 loses several bf16 ulps of the output in fp32; the two-pass
    form passes.  (The squares of bf16 values add up almost exactly in fp32, so the one-pass error is mostly the
    rounding of mean^2 and of the products with an inexact 1 / dh: at |mean| / std ~ 270 it is about one bf16 ulp for
    dh = 64 and 128 and three for dh = 80; these heads, ~ 700, make it four and more.)"""
    x, gm = heads(128, 4, dh, 7, scale=0.5, shift=300.0)
    ref, bound = RB.layernorm_heads_reference(x, gm)
    RB.check(layernorm_heads32(x, gm), ref, bound, "two-pass")
    assert flagged(layernorm_heads32(x, gm, one_pass=True), ref, bound)


# ---------------------------------------------------------------------------------------------------- mean pool
def test_mean_pool_emulation_passes_and_pooling_every_row_is_flagged():
    g = gen(9)
    x = torch.randn(3, 21, 200, generator=g) + 0.5
    n_pool = 17
    ref, bound = RB.mean_pool_reference(x, n_pool)
    s = torch.zeros(3, 200)
    for t in range(n_pool):
        s = s + x[:, t]
    RB.check(s / n_pool, ref, bound)
    assert flagged(x.mean(1), ref, bound)
