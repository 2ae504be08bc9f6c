"""The error bounds of oracle/attention_fp32_bounds.py are neither loose nor broken (CPU only).

Not broken: an fp32 emulation of each kernel's arithmetic passes its bound on the input distributions of
attention_bounds.KINDS --
  - attn_pool_kernel (NaViT pooling and class-token attention): 8 warps over 4-token groups with an online softmax in
    __expf, the tail group's duplicated token masked, the partials merged with __expf factors, A (1 / L);
  - cls_headmix.cu: fl(q scale log2e), the scores and the pre-mix as fma chains, pass 1 with lane = key (online
    max / sum per lane, shuffle merge, warp merge) into lse = M + log2(L), pass 2 p = ex2(s' - lse), the post-mix chain,
    each warp's P V chain and the sum of the warps' partials;
  - xca.cu: G = q^T k and the column sums of squares as fma chains over the tokens, the norms, the tau scaling, the
    expf softmax over the channels with per-lane sums and a butterfly, V A^T as fma chains over the channels.
Not loose: on the typical element the fp32 part of each bound is a fraction of the output's half ulp, and each planted
defect is flagged, among them one per kernel that the kernel's former criterion accepts."""
import math

import pytest
import torch

from oracle import attention_bounds as AB
from oracle import attention_fp32_bounds as FB
from oracle import bounds as Bd

LOG2E_F = torch.tensor(FB.LOG2E_F, dtype=torch.float32)


def fma32(a, b, c):
    """fp32 fma, nearly: the product is exact in fp64, the sum rounded to fp64 and then to fp32 (a double rounding
    that in rare cases differs by one fp32 ulp from a hardware fma)."""
    return (a.double() * b.double() + c.double()).float()


def fma_chain(a, b, dim):
    """acc = fma(a_i, b_i, acc) over i = 0, 1, ... along `dim` of the broadcast a * b, from acc = 0, in fp32."""
    a, b = torch.broadcast_tensors(a.float(), b.float())
    acc = torch.zeros_like(a.select(dim, 0))
    for i in range(a.shape[dim]):
        acc = fma32(a.select(dim, i), b.select(dim, i), acc)
    return acc


def butterfly(x, dim, width, op):
    """The xor-shuffle reduction over `width` lanes along `dim` (every lane ends with the result): x = op(x, x[lane ^ o])
    for o = width / 2, ..., 1."""
    o = width // 2
    while o:
        idx = torch.arange(x.shape[dim]) ^ o
        x = op(x, x.index_select(dim, idx))
        o //= 2
    return x


def fexp(x):
    """__expf in fp32: ex2 of the fp32 product x log2e_f."""
    return torch.exp2(x.float() * LOG2E_F)


def fp32_part(ref, bound):
    """(bound - half ulp) / half ulp over the nonzero outputs: the fp32 part of the bound, in output half ulps."""
    half = 0.5 * Bd.bf16_ulp(ref.abs())
    return ((bound - half) / half)[ref != 0]


# ------------------------------------------------------------------------------------------------ attn_pool_kernel
def pool_emulate(q, k, v, cls, defect=None):
    """attn_pool_kernel's arithmetic in fp32: q [G, dh] fp32 (the scaled query), k, v [G, nk, dh] bf16 (key 0 the
    query token's own under cls).  Returns the fp32 output before its bf16 rounding."""
    G, nk, dh = k.shape
    kf, vf = k.float(), v.float()
    s = torch.einsum('gd,gjd->gj', q.float(), kf)
    if defect == "scale":
        s = s * 1.001
    j0 = 1 if cls else 0
    parts = []
    for w in range(8):
        m, l, a = torch.full((G,), -math.inf), torch.zeros(G), torch.zeros(G, dh)
        if cls and w == 0 and defect != "drop_self":
            m, l, a = s[:, 0].clone(), torch.ones(G), vf[:, 0].clone()
        for j in range(j0 + 4 * w, nk, 32):
            cnt = min(4, nk - j)
            idx = [j + (i if i < cnt else 0) for i in range(4)]
            sc = s[:, idx].clone()
            if defect != "tail_dup":
                sc[:, cnt:] = -math.inf
            mn = torch.maximum(m, sc.amax(-1))
            corr = fexp(m - mn)
            l, a = l * corr, a * corr[:, None]
            for i in range(4):
                pj = fexp(sc[:, i] - mn)
                l = l + pj
                a = a + pj[:, None] * vf[:, idx[i]]
            m = mn
        parts.append((m, l, a))
    mm = torch.stack([m for m, _, _ in parts]).amax(0)
    L, A = torch.zeros(G), torch.zeros(G, dh)
    for m, l, a in parts:
        f = torch.where(m == -math.inf, torch.zeros_like(m), fexp(m - mm))
        L, A = L + l * f, A + a * f[:, None]
    return A * (1.0 / L)[:, None]


def pool_inputs(kind, nk, G, dh, seed):
    """q [G, dh] bf16, k, v [G, nk, dh] bf16 from attention_bounds.qkv_inputs (q of each sequence's first token)."""
    x = AB.qkv_inputs(kind, [nk] * G, 1, dh, seed=seed).view(G, nk, 3, dh)
    return x[:, 0, 0], x[:, :, 1], x[:, :, 2]


def pool_case(kind, nk, dh, cls, seed, defect=None, G=4):
    q, k, v = pool_inputs(kind, nk, G, dh, seed)
    scale = 0.9 * dh ** -0.5
    qs = q.float() * scale               # CLS: the kernel's fl(q scale); NaViT: the fp32 query it is given
    ref, bound = FB.pool_reference(q if cls else qs, k, v, cls=cls, scale=scale if cls else 1.0)
    got = pool_emulate(qs, k, v, cls, defect).bfloat16()
    # the former criteria, against an fp32 softmax: NaViT allclose(rtol 2e-2, atol 2e-2); CLS |d| <= 2e-2 + 1e-2 |ref|
    want = torch.einsum('gj,gjd->gd', torch.einsum('gd,gjd->gj', qs, k.float()).softmax(-1), v.float())
    d = (got.float() - want).abs()
    old = bool((d <= 2e-2 + 1e-2 * want.abs()).all()) if cls else torch.allclose(got.float(), want, 2e-2, 2e-2)
    return got, ref, bound, old


@pytest.mark.parametrize("cls", [False, True])
@pytest.mark.parametrize("dh", [32, 48, 64, 80, 128])
@pytest.mark.parametrize("kind", AB.KINDS)
def test_pool_fp32_emulation_passes(kind, dh, cls):
    if dh == 48 and not cls:
        pytest.skip("b200vit_attn_pool does not build dim_head 48")
    worst, parts = 0.0, []
    for nk in (1, 2, 3, 5, 31, 33, 129, 197, 258):
        got, ref, bound, _ = pool_case(kind, nk, dh, cls, seed=nk + dh)
        worst = max(worst, Bd.check(got, ref, bound, f"pool cls={cls} {kind} dh{dh} nk{nk}"))
        parts.append(fp32_part(ref, bound))
    med = torch.cat(parts).median().item()
    print(f"attn_pool cls={cls} {kind} dh{dh}: worst {worst:.3f}, median fp32 part {med:.4f} half ulps")
    assert med < 0.5


# defect: (cls, kind, dh, nk, does the former criterion accept it)
POOL_DEFECTS = {
    "scale": (False, "normal", 64, 197, True),       # the scores' scale off by 0.1 %
    "tail_dup": (False, "normal", 64, 197, False),   # the tail group's copies of its one token (197 = 1 mod 4) kept
    "drop_self": (True, "normal", 64, 197, False),   # CLS: the query token's own key left out (n = 196)
    "cls_scale": (True, "normal", 64, 197, True),    # CLS: the scale off by 0.1 %
}


@pytest.mark.parametrize("defect", sorted(POOL_DEFECTS))
def test_pool_planted_defect_is_flagged(defect):
    cls, kind, dh, nk, old_accepts = POOL_DEFECTS[defect]
    clean, ref, bound, _ = pool_case(kind, nk, dh, cls, seed=3)
    Bd.check(clean, ref, bound, "clean")
    got, _, _, old = pool_case(kind, nk, dh, cls, seed=3, defect="scale" if defect == "cls_scale" else defect)
    ratio = Bd.excess(got, ref, bound)
    print(f"attn_pool {defect}: worst |got - ref| / bound {ratio:.2f}, former criterion accepts: {old}")
    assert ratio > 1, defect
    assert old == old_accepts, defect


# ------------------------------------------------------------------------------------------------ cls_headmix.cu
def headmix_operands(kind, n, B, H, dh, seed):
    """The C ABI operands of the class-token kernels from attention_bounds.qkv_inputs: token 0 of each sequence is the
    class token (qkv_self), tokens 1..n its context rows ([k | v], rows = n, first = 0)."""
    I = H * dh
    x = AB.qkv_inputs(kind, [n + 1] * B, H, dh, seed=seed).view(B, n + 1, 3 * I)
    qkv_self = x[:, 0].contiguous()
    ctx = x[:, 1:, I:].reshape(B * n, 2 * I).contiguous() if n else None
    g = torch.Generator().manual_seed(seed + 1)
    pre, post = torch.randn(H, H, generator=g), torch.randn(H, H, generator=g)
    return qkv_self, ctx, pre, post


def cls_headmix_emulate(qkv_self, ctx, n, H, dh, scale, pre, post, defect=None):
    """cls_headmix.cu's arithmetic in fp32, in its order: the scores as fma chains over dh of fl(q scale log2e) and k,
    the pre-mix as a chain over the heads; pass 1 with lane = key (key 32 w + l + 256 r), an online max / sum per lane,
    the 5-level shuffle merge and the sequential merge of the 8 warps into lse = M + log2(L); pass 2 p = ex2(s' - lse),
    the post-mix chain, each warp's fma chain over its keys and the sum of the 8 warps' partials."""
    q, k, v = FB.cls_operands(qkv_self, ctx, n, 0, n, H, dh)
    B, nk = k.shape[:2]
    c = torch.tensor(AB.scale_log2e(scale), dtype=torch.float32)
    if defect == "scale":
        c = c * 1.001
    s = fma_chain((q.float() * c)[:, None], k.float(), -1).transpose(1, 2)           # [B, H, nk]
    sm = fma_chain(pre[None, :, :, None], s[:, :, None], 1)                          # [B, g, nk]
    if defect == "drop_self":
        sm[..., 0] = -math.inf                        # the query token's own key in neither pass
    R = -(-nk // 256)
    x = torch.full((B, H, R * 256), -math.inf)
    x[..., :nk] = sm
    x = x.view(B, H, R, 8, 32)                        # key 256 r + 32 w + l
    m, l = torch.full((B, H, 8, 32), -math.inf), torch.zeros(B, H, 8, 32)
    for r in range(R):
        mn = torch.maximum(m, x[:, :, r])
        mn_safe = torch.where(mn == -math.inf, torch.zeros_like(mn), mn)             # lanes past the keys stay (-inf, 0)
        l = torch.where(mn == -math.inf, l, l * torch.exp2(m - mn_safe) + torch.exp2(x[:, :, r] - mn_safe))
        m = mn
    o = 16
    while o:
        idx = torch.arange(32) ^ o
        m2, l2 = m.index_select(-1, idx), l.index_select(-1, idx)
        mn = torch.maximum(m, m2)
        mn_safe = torch.where(mn == -math.inf, torch.zeros_like(mn), mn)
        l = torch.where(mn == -math.inf, torch.zeros_like(l),
                        l * torch.exp2(m - mn_safe) + l2 * torch.exp2(m2 - mn_safe))
        m = mn
        o //= 2
    m, l = m[..., 0], l[..., 0]                       # [B, H, 8 warps]
    mm = m.amax(-1, keepdim=True)
    L = torch.zeros(B, H)
    for w in range(8):
        L = torch.where(m[..., w] == -math.inf, L, L + l[..., w] * torch.exp2(m[..., w] - mm[..., 0]))
    lse = mm + torch.log2(L)[..., None]
    p = torch.exp2(sm - lse)                          # [B, g, nk]
    pf = fma_chain(post[None, :, :, None], p[:, :, None], 1)                         # [B, f, nk]
    # warp w's keys in its order: rounds r, then the 32 keys 256 r + 32 w + jj
    P = torch.zeros(B, H, R * 256)
    P[..., :nk] = pf
    V = torch.zeros(B, R * 256, H, dh)
    V[:, :nk] = v.float()
    P, V = P.view(B, H, R, 8, 32), V.view(B, R, 8, 32, H, dh)
    acc = torch.zeros(B, 8, H, dh)
    for r in range(R):
        for jj in range(32):
            acc = fma32(P[:, :, r, :, jj].permute(0, 2, 1)[..., None], V[:, r, :, jj], acc)
    out = torch.zeros(B, H, dh)
    for w in range(8):
        out = out + acc[:, w]
    return out.reshape(B, H * dh)


def close_to(out, ref):
    """The former criterion of test_gpu_cait.py: True if it accepts `out` against the fp32 reference `ref`."""
    tol = 1e-2 * ref.abs().max().item() + 1e-3
    err = (out.float() - ref).abs()
    return bool(err.max().item() <= tol + 1e-2 * ref.abs().max().item()
                and (err <= tol + 1e-2 * ref.abs()).float().mean().item() > 0.999)


@pytest.mark.parametrize("H,dh", [(1, 64), (3, 48), (4, 32), (6, 80), (8, 128), (16, 64)])
@pytest.mark.parametrize("kind", AB.KINDS)
def test_cls_headmix_fp32_emulation_passes(kind, H, dh):
    worst, parts = 0.0, []
    for n in (0, 1, 31, 196, 300):
        qkv_self, ctx, pre, post = headmix_operands(kind, n, 3, H, dh, seed=n + H + dh)
        scale = dh ** -0.5
        got = cls_headmix_emulate(qkv_self, ctx, n, H, dh, scale, pre, post).bfloat16()
        ref, bound = FB.cls_headmix_reference(qkv_self, ctx, n, 0, n, H, dh, scale, pre, post)
        worst = max(worst, Bd.check(got, ref, bound, f"cls_headmix {kind} H{H} dh{dh} n{n}"))
        parts.append(fp32_part(ref, bound))
    med = torch.cat(parts).median().item()
    print(f"cls_headmix {kind} H{H} dh{dh}: worst {worst:.3f}, median fp32 part {med:.4f} half ulps")
    assert med < 0.5


# defect: does the former criterion accept it
CLS_HEADMIX_DEFECTS = {"drop_self": False,   # the query token's own key left out of both passes (n = 196)
                       "scale": True}        # the score scale off by 0.1 %


@pytest.mark.parametrize("defect", sorted(CLS_HEADMIX_DEFECTS))
def test_cls_headmix_planted_defect_is_flagged(defect):
    H, dh, n = 8, 48, 196
    qkv_self, ctx, pre, post = headmix_operands("normal", n, 3, H, dh, seed=5)
    scale = dh ** -0.5
    ref, bound = FB.cls_headmix_reference(qkv_self, ctx, n, 0, n, H, dh, scale, pre, post)
    Bd.check(cls_headmix_emulate(qkv_self, ctx, n, H, dh, scale, pre, post).bfloat16(), ref, bound, "clean")
    got = cls_headmix_emulate(qkv_self, ctx, n, H, dh, scale, pre, post, defect).bfloat16()
    ratio = Bd.excess(got, ref, bound)
    old = close_to(got, cls_headmix_emulate(qkv_self, ctx, n, H, dh, scale, pre, post))
    print(f"cls_headmix {defect}: worst |got - ref| / bound {ratio:.2f}, former criterion accepts: {old}")
    assert ratio > 1, defect
    assert old == CLS_HEADMIX_DEFECTS[defect], defect


# ------------------------------------------------------------------------------------------------ xca.cu
def xca_emulate(qkv, tau, B, N, H, dh, defect=None):
    """xca.cu's arithmetic in fp32, in its order: G and the column sums of squares as fma chains over the tokens, the
    reciprocal norms, fl(fl(tau r_i) G_ij) r_j, the row max, expf, each lane's sum of its dh / 16 channels and the
    4-level butterfly, A = e fl(1 / l), then O = V A^T as fma chains over the channels."""
    q, k, v = qkv.float().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)               # [B, H, N, dh]
    G = fma_chain(q[..., :, None], k[..., None, :], 2)                               # [B, H, dh, dh]
    nn = N
    if defect == "tail_norms":                        # the last partial token tile left out of the column norms
        nn = N // FB.xca_tile(dh) * FB.xca_tile(dh)
    rq = 1.0 / fma_chain(q[:, :, :nn], q[:, :, :nn], 2).sqrt().clamp_min(FB.NORM_EPS_F)
    rk = 1.0 / fma_chain(k[:, :, :nn], k[:, :, :nn], 2).sqrt().clamp_min(FB.NORM_EPS_F)
    t = tau.view(1, H, 1, 1) * (1.001 if defect == "scale" else 1.0)
    x = ((t * rq[..., :, None]) * G) * rk[..., None, :]
    e = torch.exp(x - x.amax(-1, keepdim=True))
    R = dh // 16
    el = e.view(B, H, dh, R, 16)                      # channel tx + 16 c: lane tx holds its R channels
    l = torch.zeros(B, H, dh, 16)
    for cc in range(R):
        l = l + el[..., cc, :]
    l = butterfly(l, -1, 16, torch.add)[..., :1]
    a = e * (1.0 / l)
    out = fma_chain(v[:, :, :, None, :], a[:, :, None, :, :], -1)                    # [B, H, N, dh]
    return out.permute(0, 2, 1, 3).reshape(B * N, H * dh)


def xca_inputs(kind, B, N, H, dh, seed):
    qkv = AB.qkv_inputs(kind, [N] * B, H, dh, seed=seed)
    tau = torch.exp(torch.linspace(-2.0, 3.0, H))
    return qkv, tau


def xca_old_criterion(got, want):
    d = (got.float() - want).abs()
    return bool(d.max().item() < 3e-2 and (d <= 1e-2 + 1e-2 * want.abs()).float().mean().item() > 0.999)


@pytest.mark.parametrize("dh", [32, 48, 64, 80, 128])
@pytest.mark.parametrize("kind", AB.KINDS)
def test_xca_fp32_emulation_passes(kind, dh):
    H, B = 3, 2
    worst, parts = 0.0, []
    T = FB.xca_tile(dh)
    for N in (1, T - 1, T + 1, 197, 784, 3136):
        qkv, tau = xca_inputs(kind, B, N, H, dh, seed=N + dh)
        got = xca_emulate(qkv, tau, B, N, H, dh).bfloat16()
        ref, bound = FB.xca_reference(qkv, tau, B, N, H, dh)
        worst = max(worst, Bd.check(got, ref, bound, f"xca {kind} dh{dh} N{N}"))
        parts.append(fp32_part(ref, bound))
    med = torch.cat(parts).median().item()
    print(f"xca {kind} dh{dh}: worst {worst:.3f}, median fp32 part {med:.4f} half ulps")
    assert med < 0.5


def test_xca_zero_and_unequal_columns_pass():
    """A zero q column (its scores are exact zeros: a uniform row) and columns whose norms differ by 2^10."""
    B, N, H, dh = 2, 197, 2, 48
    qkv, tau = xca_inputs("normal", B, N, H, dh, seed=9)
    x = qkv.float().view(B * N, 3, H, dh)
    x[:, 0, 0, 5] = 0
    x[:, 1, 1, 3] *= 32
    x[:, 0, 1, 7] /= 32
    qkv = x.reshape(B * N, -1).bfloat16()
    ref, bound = FB.xca_reference(qkv, tau, B, N, H, dh)
    Bd.check(xca_emulate(qkv, tau, B, N, H, dh).bfloat16(), ref, bound, "xca zero / unequal columns")
    # row 5 of head 0 has zero scores: its reference is the mean of head 0's v columns
    v0 = qkv.double().view(B, N, 3, H, dh)[:, :, 2, 0]
    assert torch.allclose(ref.view(B, N, H, dh)[:, :, 0, 5], v0.mean(-1))


# defect: does the former criterion accept it
XCA_DEFECTS = {"tail_norms": False,   # the last partial token tile (5 of 197 tokens) left out of the column norms
               "scale": True}         # tau off by 0.1 %


@pytest.mark.parametrize("defect", sorted(XCA_DEFECTS))
def test_xca_planted_defect_is_flagged(defect):
    B, N, H, dh = 2, 197, 3, 64
    qkv, tau = xca_inputs("normal", B, N, H, dh, seed=11)
    ref, bound = FB.xca_reference(qkv, tau, B, N, H, dh)
    Bd.check(xca_emulate(qkv, tau, B, N, H, dh).bfloat16(), ref, bound, "clean")
    got = xca_emulate(qkv, tau, B, N, H, dh, defect).bfloat16()
    ratio = Bd.excess(got, ref, bound)
    old = xca_old_criterion(got, xca_emulate(qkv, tau, B, N, H, dh))
    print(f"xca {defect}: worst |got - ref| / bound {ratio:.2f}, former criterion accepts: {old}")
    assert ratio > 1, defect
    assert old == XCA_DEFECTS[defect], defect
