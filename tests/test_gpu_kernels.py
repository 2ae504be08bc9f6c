"""-m gpu: every kernel of libb200vit.so, called through the C ABI, against the oracle's primitives
(oracle/vit_oracle.py) on the same seeded inputs.  Floating point path: tolerance stated per test."""
import math

import pytest
import torch

from oracle import attention_bounds as AB
from oracle import bounds as Bd
from oracle import row_bounds as RB
from oracle import vit_oracle as O
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"


def test_device_and_library():
    assert _lib.device_ok(0)
    _lib.reset_launch_count()


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 128, 256), (591, 1000, 768), (100, 10, 192), (384, 576, 192),
                                   (1, 768, 768), (130, 264, 72)])
def test_gemm_plain(M, N, K):
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device=DEV).bfloat16()
    w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    out = torch.zeros(M, N, device=DEV)
    _lib.gemm(a, w, out_f32=out)
    ref = O.linear(a.float().cpu(), w.float().cpu())
    # fp32 accumulation of exact bf16 products: only summation order differs from the oracle
    assert torch.allclose(out.cpu(), ref, rtol=1e-4, atol=1e-4)


def test_gemm_k_padding_zero_fill():
    torch.manual_seed(0)
    a = torch.randn(256, 64, device=DEV).bfloat16()
    w = torch.randn(192, 64, device=DEV).bfloat16()
    a[:, 48:] = 7.0                 # garbage beyond K=48 must not be read as data: pass k=48 explicitly
    w[:, 48:] = 7.0
    out = torch.zeros(256, 192, device=DEV)
    _lib.gemm(a, w, out_f32=out, k=48)
    ref = a[:, :48].float() @ w[:, :48].float().t()
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-4)


def test_gemm_epilogues_bias_gelu_residual():
    torch.manual_seed(1)
    M, N, K = 394, 768, 512
    a = torch.randn(M, K, device=DEV).bfloat16()
    w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device=DEV)
    r = torch.randn(M, N, device=DEV)
    lin = O.linear(a.float().cpu(), w.float().cpu(), b.cpu())
    # bias + GELU -> bf16  (FeedForward first half, vit.py:20-21)
    ob = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    _lib.gemm(a, w, out_bf16=ob, bias=b, gelu=True)
    Bd.check(ob, *Bd.gemm_reference(a, w, bias=b, gelu=True, bf16_out=True), "bias + GELU -> bf16")
    # bias + residual, in place on the fp32 stream (vit.py:80-81)
    x = r.clone()
    _lib.gemm(a, w, out_f32=x, bias=b, resid=x)
    assert torch.allclose(x.cpu(), lin + r.cpu(), rtol=1e-4, atol=1e-4)
    Bd.check(x, *Bd.gemm_reference(a, w, bias=b, resid=r), "bias + residual")


def test_gemm_lnfold_and_stats():
    torch.manual_seed(2)
    M, N, K = 260, 512, 768
    a = (torch.randn(M, K, device=DEV) * 2 + 0.3).bfloat16()
    g = torch.randn(K, device=DEV)
    be = torch.randn(K, device=DEV)
    w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    wg = (w.float() * g).bfloat16()                         # gamma folded into W, rounded like the product path
    col_s = wg.float().sum(1)
    t = w.float() @ be
    af = a.float()
    sums = torch.stack([af.sum(1), (af * af).sum(1)], 1).contiguous()
    out = torch.zeros(M, N, device=DEV)
    st = torch.full((M, _lib.stats_parts(N), 2), 9.0, device=DEV)     # every slot must be overwritten
    ob = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    # partial input statistics in two unequal parts: the kernel adds them up in order
    sums2 = torch.stack([sums * 0.25, sums * 0.75], 1).contiguous()
    _lib.gemm(a, wg, out_f32=out, out_bf16=ob, bias=t.contiguous(), ln_sums=sums2, col_s=col_s.contiguous(),
              stats_out=st)
    st_parts, st = st, st.sum(1)
    # (a) the kernel's arithmetic, against the same folded formula evaluated in fp32 on the host
    mu = af.mean(1, keepdim=True)
    rstd = torch.rsqrt((af * af).mean(1, keepdim=True) - mu * mu + 1e-5)
    same = (rstd * (af @ wg.float().t() - mu * col_s[None]) + t[None]).cpu()
    assert torch.allclose(out.cpu(), same, rtol=2e-3, atol=2e-3)
    # (b) every element within its bound of the fp64 LayerNorm-folded GEMM of the same inputs (oracle/bounds.py), and
    # near the oracle's exact LayerNorm -> Linear: only the bf16 rounding of gamma*W separates the two
    ref, e = Bd.gemm_reference(a, wg, bias=t, ln_sums=sums2, col_s=col_s)
    Bd.check(out, ref, e, "LN fold fp32")
    Bd.check(ob, ref, Bd.bf16_bound(ref, e), "LN fold bf16")
    Bd.check(st_parts, *Bd.stats_reference(ob, st_parts.shape[1]), "stats")
    ref = O.linear(O.layer_norm(af.cpu(), g.cpu(), be.cpu()), w.float().cpu())
    assert (out.cpu() - ref).abs().max() < 0.05
    rb = ob.float()
    assert torch.allclose(st[:, 0], rb.sum(1), rtol=1e-4, atol=1e-2)
    assert torch.allclose(st[:, 1], (rb * rb).sum(1), rtol=1e-4, atol=1e-2)


def test_layernorm_row_gather_no_bias():
    torch.manual_seed(4)
    x = torch.randn(197 * 4, 256, device=DEV)
    g = torch.randn(256, device=DEV)
    rows = torch.arange(0, 197 * 4, 197, device=DEV, dtype=torch.int32)
    of = torch.zeros(4, 256, device=DEV)
    _lib.layernorm(x, g, None, out_f32=of, row_index=rows)
    assert torch.allclose(of.cpu(), O.layer_norm(x[rows.long()].cpu(), g.cpu(), None), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("C,H,W,p", [(3, 224, 224, 16), (3, 32, 32, 4), (3, 224, 224, 14), (1, 64, 32, 8),
                                     (3, 384, 256, 16), (3, 48, 16, 16), (4, 32, 32, 16)])
def test_patchify_ln(C, H, W, p):
    torch.manual_seed(5)
    img = torch.randn(3, C, H, W, device=DEV).bfloat16()
    pd = C * p * p
    ldo = (pd + 63) // 64 * 64
    g, b = torch.randn(pd, device=DEV), torch.randn(pd, device=DEV)
    out = torch.full((3 * (H // p) * (W // p), ldo), 7.0, device=DEV, dtype=torch.bfloat16)
    _lib.patchify_ln(img, g, b, out, p, p)
    # within one bf16 ulp (plus the fp32 error of the LayerNorm) of the fp64 LayerNorm of every patch
    Bd.check(out[:, :pd], *Bd.layernorm_reference(O.patchify(img, p, p).reshape(-1, pd), g, b), "patchify_ln")
    assert (out[:, pd:] == 0).all()


@pytest.mark.parametrize("B,C,H,W,D", [(3, 3, 224, 224, 256), (2, 3, 32, 48, 64), (2, 1, 64, 64, 128), (5, 3, 16, 16, 64),
                                        (2, 3, 16, 512, 72), (1, 4, 48, 16, 64)])
def test_patch_embed_tma_matches_patchify_layernorm_linear(B, C, H, W, D):
    """im2col-free patch embedding: the wgmma GEMM reads the NCHW image through a 5-D TMA map, LayerNorm(patch) is
    folded into its epilogue -- against Rearrange -> LayerNorm -> Linear (vit.py:100-102) in fp32 on the CPU."""
    torch.manual_seed(H * W + C)
    pd = C * 256
    img = torch.randn(B, C, H, W, device=DEV).bfloat16()
    g, be = 1 + 0.2 * torch.randn(pd), 0.1 * torch.randn(pd)
    w = (torch.randn(D, pd) / pd ** 0.5).bfloat16().float()
    b = 0.1 * torch.randn(D)
    wg = w * g[None, :]
    w_perm = wg.view(D, 256, C).permute(0, 2, 1).reshape(D, pd).bfloat16().contiguous().to(DEV)
    col_s = w_perm.float().sum(1).contiguous()
    bias = (w @ be + b).to(DEV).contiguous()
    n = (H // 16) * (W // 16)
    y = torch.full((B * n, D), float("nan"), device=DEV)
    stats = torch.zeros(B * n, 2, device=DEV)
    _lib.patch_embed_tma(img, w_perm, bias, col_s, stats, y)
    patches = O.patchify(img.float().cpu(), 16, 16)                                 # [B, n, (p1 p2 c)]
    ref = O.linear(O.layer_norm(patches, g, be), w, b).reshape(B * n, D)
    assert torch.allclose(stats[:, 0].cpu(), patches.reshape(B * n, -1).sum(1), rtol=1e-4, atol=1e-2)
    d = (y.cpu() - ref).abs()
    print(f"patch_embed_tma {B}x{C}x{H}x{W} -> {D}: max {d.max():.4f} mean {d.mean():.5f}")
    assert torch.isfinite(y).all() and d.max() < 3e-2 and d.mean() < 4e-3     # gamma (.) W is rounded to bf16


@pytest.mark.parametrize("M,N,K", [(2048, 768, 768), (1300, 1024, 512),
                                   (1536, 384, 384), (1100, 320, 2304)])   # last N tile only partly valid (ViT-S dims)
def test_gemm_pair_kernel_dual_epilogue(M, N, K):
    """Producer epilogue of the residual GEMMs: fp32 stream in place + bf16 copy + row statistics."""
    torch.manual_seed(M)
    a = torch.randn(M, K, device=DEV).bfloat16()
    w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device=DEV)
    x0 = torch.randn(M, N, device=DEV)
    x = x0.clone()
    xb = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    st = torch.full((M, _lib.stats_parts(N), 2), 123.0, device=DEV)          # every slot must be overwritten
    _lib.gemm(a, w, out_f32=x, out_bf16=xb, bias=b, resid=x, stats_out=st)
    st2 = st.clone()
    x2 = x0.clone()
    _lib.gemm(a, w, out_f32=x2, out_bf16=xb, bias=b, resid=x2, stats_out=st2)
    assert torch.equal(st, st2) and torch.equal(x, x2)                        # deterministic, no atomics
    st = st.sum(1)
    ref = O.linear(a.float().cpu(), w.float().cpu(), b.cpu()) + x0.cpu()
    assert torch.allclose(x.cpu(), ref, rtol=1e-4, atol=1e-4)
    assert torch.equal(xb, x.bfloat16())
    xr = xb.float()
    assert torch.allclose(st[:, 0], xr.sum(1), rtol=1e-4, atol=2e-2)
    assert torch.allclose(st[:, 1], (xr * xr).sum(1), rtol=1e-4, atol=2e-2)


def test_gelu_epilogue_accuracy():
    """The GELU of the GEMM epilogue follows the erf definition to 1.2e-5 absolute (before the bf16 rounding of the
    output): drive it with acc = 0 and the probe values in the bias vector."""
    K, N, M = 64, 4096, 128
    xs = torch.linspace(-8, 8, N, device=DEV)
    a = torch.zeros(M, K, device=DEV, dtype=torch.bfloat16)
    w = torch.zeros(N, K, device=DEV, dtype=torch.bfloat16)
    ob = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    _lib.gemm(a, w, out_bf16=ob, bias=xs.contiguous(), gelu=True)
    ref = O.gelu_erf(xs.double().cpu())
    got = ob[5].double().cpu()
    assert ((got - ref).abs() <= 1.2e-5 + ref.abs() * 2.0 ** -8).all()


@pytest.mark.parametrize("B,N,H", [(4, 197, 12), (3, 64, 3), (2, 257, 16), (5, 50, 4), (2, 16, 2), (2, 129, 2),
                                   (1, 512, 1), (2, 1, 2),
                                   # more CTAs than SMs, key counts on and just past a key-block boundary
                                   (40, 197, 12), (70, 196, 16), (200, 128, 3), (37, 224, 5), (3, 225, 2), (9, 33, 7)])
@pytest.mark.parametrize("tiled", [False, True])  # test hook 15: the tiled kernel at 128 < N <= 256 as well
def test_attention(B, N, H, tiled):
    torch.manual_seed(N)
    dh = 64
    I = H * dh
    qkv = torch.randn(B * N, 3 * I, device=DEV).bfloat16()
    out = torch.full((B * N, I), float("nan"), device=DEV, dtype=torch.bfloat16)   # unwritten elements fail
    _lib.lib().b200vit_debug_set(15, int(tiled))
    try:
        _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
        torch.cuda.synchronize()
    finally:
        _lib.lib().b200vit_debug_set(15, 0)
    # every element within its bound of the fp64 attention that replays the kernel's bf16 P (oracle/attention_bounds.py)
    ref, bound = AB.qkv_attention_reference(qkv, [N] * B, H, dh, dh ** -0.5)
    Bd.check(out, ref, bound, f"attention B{B} N{N} H{H} hook 15 = {tiled}")


@pytest.mark.parametrize("B,N,H", [(2, 257, 16), (3, 197, 4), (5, 64, 2), (2, 400, 3), (1, 512, 2), (40, 129, 5)])
def test_attention_dim_head_80(B, N, H):
    """Canonical ViT-H/14 head width (reference vit.py:86 `dim_head`)."""
    torch.manual_seed(N)
    dh = 80
    I = H * dh
    qkv = torch.randn(B * N, 3 * I, device=DEV).bfloat16()
    out = torch.full((B * N, I), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
    ref, bound = AB.qkv_attention_reference(qkv, [N] * B, H, dh, dh ** -0.5)
    view = lambda t: t.view(B * N, H, dh)
    r64 = Bd.check(view(out)[..., :64], view(ref)[..., :64], view(bound)[..., :64], f"dh80 B{B} N{N} dims 0..63")
    r16 = Bd.check(view(out)[..., 64:], view(ref)[..., 64:], view(bound)[..., 64:], f"dh80 B{B} N{N} dims 64..79")
    print(f"dh80 B{B} N{N}: worst |got - ref| / bound dims 0..63 {r64:.3f}, dims 64..79 {r16:.3f}")


@pytest.mark.parametrize("dh", [64, 80])
@pytest.mark.parametrize("B,N,H", [(3, 257, 4), (2, 258, 2), (2, 260, 3), (40, 257, 16), (1, 261, 2), (300, 257, 2)])
def test_attention_key_tail(B, N, H, dh):
    """N = 256 + (1..5): the last keys sit alone in the final key block.  Checked against the fp64 oracle with the tail
    keys made the dominant ones."""
    torch.manual_seed(N + dh)
    I = H * dh
    qkv = torch.randn(B * N, 3 * I, device=DEV)
    qkv.view(B, N, 3, I)[:, N - 2:, 1] *= 2.5            # the last keys attract most of the attention
    qkv = qkv.bfloat16()
    out = torch.full((B * N, I), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
    ref, bound = AB.qkv_attention_reference(qkv, [N] * B, H, dh, dh ** -0.5)
    Bd.check(out, ref, bound, f"key tail N{N} dh{dh}")


def test_attention_is_deterministic_and_batch_invariant():
    """The same (image, head) must give the same bits wherever it lands in the batch and on repeated launches."""
    torch.manual_seed(11)
    B, N, H, dh = 64, 197, 12, 64
    _lib.lib().b200vit_debug_set(15, 1)         # the tiled kernel at N 197 (test hook), restored below
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV).bfloat16()
    out = torch.zeros(B * N, H * dh, device=DEV, dtype=torch.bfloat16)
    out2 = torch.zeros_like(out)
    _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
    _lib.attention(qkv, out2, B, N, H, dh, dh ** -0.5)
    assert torch.equal(out, out2)
    sub = qkv[5 * N: 9 * N].contiguous()
    out3 = torch.zeros(4 * N, H * dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention(sub, out3, 4, N, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    _lib.lib().b200vit_debug_set(15, 0)
    assert torch.equal(out3, out[5 * N: 9 * N])


def test_gemm_long_k_block_n_variants_agree():
    """Long-K fp32 epilogues with 128- and 256-column tiles (test hook 12 forces either): the same bits."""
    torch.manual_seed(12)
    M, N, K = 2048 + 64, 768, 3072
    a = torch.randn(M, K, device=DEV).bfloat16()
    w = (torch.randn(N, K, device=DEV) * 0.02).bfloat16()
    bias = torch.randn(N, device=DEV)
    x0 = torch.randn(M, N, device=DEV)
    res = {}
    L = _lib.lib()
    for ew in (1, 2):
        L.b200vit_debug_set(12, ew)
        try:
            x = x0.clone()
            xb = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
            st = torch.full((M, _lib.stats_parts(N), 2), float("nan"), device=DEV)
            _lib.gemm(a, w, out_f32=x, out_bf16=xb, bias=bias, resid=x, stats_out=st)
            y = torch.zeros(M, N, device=DEV)
            _lib.gemm(a, w, out_f32=y, bias=bias)
            torch.cuda.synchronize()
        finally:
            L.b200vit_debug_set(12, 0)
        res[ew] = (x, xb, st.sum(dim=1), y)
    ref, e = Bd.gemm_reference(a, w, bias=bias, resid=x0)
    ref_y, e_y = Bd.gemm_reference(a, w, bias=bias)
    for ew in (1, 2):
        x, xb, st, y = res[ew]
        assert torch.isfinite(st).all()
        Bd.check(x, ref, e, f"long K, residual, hook 12 = {ew}")
        Bd.check(y, ref_y, e_y, f"long K, fp32, hook 12 = {ew}")
        assert torch.equal(xb, x.bfloat16())
        assert torch.allclose(st[:, 0].cpu(), xb.float().sum(1).cpu(), rtol=1e-3, atol=1e-2)
        assert torch.allclose(st[:, 1].cpu(), (xb.float() ** 2).sum(1).cpu(), rtol=1e-3, atol=1e-2)
    assert torch.equal(res[1][0], res[2][0]) and torch.equal(res[1][3], res[2][3])


def test_attention_large_logits_are_stable():
    torch.manual_seed(9)
    B, N, H, dh = 2, 197, 2, 64
    qkv = (torch.randn(B * N, 3 * H * dh, device=DEV) * 6).bfloat16()      # |s| up to ~300: softmax nearly one-hot
    out = torch.full((B * N, H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
    assert torch.isfinite(out.float()).all()
    Bd.check(out, *AB.qkv_attention_reference(qkv, [N] * B, H, dh, dh ** -0.5), "large logits")


def _same_bits(a, b):
    """bit equality, NaN payloads included."""
    return torch.equal(a.view(torch.int16 if a.dtype == torch.bfloat16 else torch.int32),
                       b.view(torch.int16 if b.dtype == torch.bfloat16 else torch.int32))


def test_rowstats_cast():
    """The bf16 copy bit for bit, the (sum, sum of squares) within the depth-based bound of
    oracle/row_bounds.py at D on the float4 path (768, 192) and the scalar path (50); rows past M untouched."""
    for D in (768, 192, 50):
        torch.manual_seed(D)
        M = 333
        x = torch.randn(M, D, device=DEV) * 2 + 0.5
        xb = torch.full((M + 2, D), float("nan"), device=DEV, dtype=torch.bfloat16)
        st = torch.full((M + 2, 2), float("nan"), device=DEV)
        _lib.rowstats_cast(x, xb[:M], st[:M])
        assert _same_bits(xb[:M], x.bfloat16())
        r = RB.check(st[:M], *RB.row_stats_reference(xb[:M]), f"rowstats_cast D={D}")
        print(f"excess rowstats_cast D={D}: {r:.3f}")
        assert torch.isnan(xb[M:].float()).all() and torch.isnan(st[M:]).all()
        xb2, st2 = torch.empty_like(xb[:M]), torch.empty_like(st[:M])
        _lib.rowstats_cast(x, xb2, st2)
        assert _same_bits(xb2, xb[:M]) and _same_bits(st2, st[:M])


def test_mean_pool_and_cast():
    """mean_pool within the bound of oracle/row_bounds.py (n_pool < N as with register tokens, n_pool = 1, D not a
    multiple of 256): repeat calls give the same bits, a NaN stays in its image, rows past n_pool are not read.
    cast_f32_bf16 equals torch's round-to-nearest-even bit for bit at n % 8 = 0 .. 7, n < 8, +-0, subnormals,
    +-Inf and NaN, and writes nothing past n."""
    nan = float("nan")
    for B, N, D, n_pool in [(8, 197, 768, 197), (5, 21, 200, 17), (3, 9, 100, 1), (4, 65, 300, 64)]:
        torch.manual_seed(N + D)
        x = torch.randn(B, N, D, device=DEV) + 0.3
        o = torch.full((B + 1, D), nan, device=DEV)
        _lib.mean_pool(x, o[:B], B, N, D, n_pool)
        r = RB.check(o[:B], *RB.mean_pool_reference(x, n_pool), f"mean_pool {B}x{N}x{D} n_pool={n_pool}")
        print(f"excess mean_pool {B}x{N}x{D} n_pool={n_pool}: {r:.3f}")
        assert torch.isnan(o[B:]).all()
        o2 = torch.full((B + 1, D), nan, device=DEV)
        _lib.mean_pool(x, o2[:B], B, N, D, n_pool)
        assert _same_bits(o2, o)
        xn = x.clone()
        xn[1, n_pool - 1, 3] = nan
        if n_pool < N:
            xn[2, n_pool:] = nan                                     # rows past n_pool (register tokens)
        on = torch.full((B + 1, D), nan, device=DEV)
        _lib.mean_pool(xn, on[:B], B, N, D, n_pool)
        others = [0] + list(range(2, B))
        assert torch.isnan(on[1, 3]) and _same_bits(on[others], o[others])
    special = torch.tensor([0.0, -0.0, 1e-40, -1e-40, 1.17e-38, float("inf"), float("-inf"), nan,
                            1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 3.4e38], device=DEV)
    for n in [1, 3, 7, 8, 9, 15, 16, 17, 1000, 1001, 1002, 1003, 1004, 1005, 1006, 1007, 4096 + 5, 8 * 197 * 768]:
        g = torch.Generator(device=DEV).manual_seed(n)
        x = torch.randn(n, generator=g, device=DEV) * 100
        x[:min(n, special.numel())] = special[:min(n, special.numel())]
        out = torch.full((n + 8,), nan, device=DEV, dtype=torch.bfloat16)
        _lib.cast_f32_bf16(x, out[:n])
        want = x.bfloat16()
        ok = ~torch.isnan(want)
        assert torch.equal(out[:n].view(torch.int16)[ok], want.view(torch.int16)[ok]), n
        assert torch.equal(torch.isnan(out[:n]), torch.isnan(want)) and torch.isnan(out[n:].float()).all(), n


def test_kernels_were_launched_by_the_library():
    assert _lib.launch_count() > 0
