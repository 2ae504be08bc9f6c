"""-m gpu: every kernel of libb200vit.so, called through the C ABI, against the oracle's primitives
(oracle/vit_oracle.py) on the same seeded inputs.  Floating point path: tolerance stated per test."""
import math

import pytest
import torch

from oracle import vit_oracle as O
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"


def within(got, ref, rtol=1e-2, atol=1e-3):
    got, ref = got.float().cpu(), ref.float().cpu()
    return ((got - ref).abs() <= atol + rtol * ref.abs()).float().mean().item()


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
    w[:, 48:] = 0.0
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
    assert within(ob, O.gelu_erf(lin)) > 0.999          # bf16 output rounding only (rtol 1e-2 / atol 1e-3)
    # bias + residual, in place on the fp32 stream (vit.py:80-81)
    x = r.clone()
    _lib.gemm(a, w, out_f32=x, bias=b, resid=x)
    assert torch.allclose(x.cpu(), lin + r.cpu(), rtol=1e-4, atol=1e-4)


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
    st = st.sum(1)
    # (a) the kernel's arithmetic, against the same folded formula evaluated in fp32 on the host
    mu = af.mean(1, keepdim=True)
    rstd = torch.rsqrt((af * af).mean(1, keepdim=True) - mu * mu + 1e-5)
    same = (rstd * (af @ wg.float().t() - mu * col_s[None]) + t[None]).cpu()
    assert torch.allclose(out.cpu(), same, rtol=2e-3, atol=2e-3)
    # (b) against the oracle's exact LayerNorm -> Linear: only the bf16 rounding of gamma*W separates them
    ref = O.linear(O.layer_norm(af.cpu(), g.cpu(), be.cpu()), w.float().cpu())
    assert within(out, ref) > 0.95 and (out.cpu() - ref).abs().max() < 0.05
    rb = ob.float()
    assert torch.allclose(st[:, 0], rb.sum(1), rtol=1e-4, atol=1e-2)
    assert torch.allclose(st[:, 1], (rb * rb).sum(1), rtol=1e-4, atol=1e-2)


@pytest.mark.parametrize("M,D", [(1000, 768), (77, 50), (513, 1280)])
def test_layernorm(M, D):
    torch.manual_seed(3)
    x = torch.randn(M, D, device=DEV) * 3 + 1
    g, b = torch.randn(D, device=DEV), torch.randn(D, device=DEV)
    of = torch.zeros(M, D, device=DEV)
    ob = torch.zeros(M, D, device=DEV, dtype=torch.bfloat16)
    _lib.layernorm(x, g, b, out_bf16=ob, out_f32=of)
    ref = O.layer_norm(x.cpu(), g.cpu(), b.cpu())
    assert torch.allclose(of.cpu(), ref, rtol=1e-5, atol=1e-5)
    assert torch.equal(ob.cpu(), of.cpu().bfloat16())


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
    ref = O.layer_norm(O.patchify(img.float().cpu(), p, p), g.cpu(), b.cpu()).reshape(-1, pd)
    assert torch.equal(out[:, :pd].cpu(), ref.bfloat16()) or within(out[:, :pd], ref) > 0.9999
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


@pytest.mark.parametrize("ncls", [0, 1])
def test_embed_tokens(ncls):
    torch.manual_seed(6)
    B, n, D = 3, 49, 192
    y = torch.randn(B * n, D, device=DEV)
    g, be = torch.randn(D, device=DEV), torch.randn(D, device=DEV)
    cls = torch.randn(ncls, D, device=DEV) if ncls else None
    pos = torch.randn(n + ncls, D, device=DEV)
    x = torch.zeros(B * (n + ncls), D, device=DEV)
    xb = torch.zeros(B * (n + ncls), D, device=DEV, dtype=torch.bfloat16)
    st = torch.zeros(B * (n + ncls), 1, 2, device=DEV)
    _lib.embed_tokens(y, g, be, cls, pos, x, B, n, ncls, xb=xb, stats=st)
    st = st[:, 0]
    t = O.layer_norm(y.cpu(), g.cpu(), be.cpu()).view(B, n, D)
    if ncls:
        t = torch.cat([cls.cpu()[None].expand(B, -1, -1), t], 1)
    assert torch.allclose(x.cpu(), (t + pos.cpu()[None]).reshape(-1, D), rtol=1e-5, atol=1e-5)
    # bf16 copy and its row statistics (inputs of the first LN-folded GEMM)
    assert torch.equal(xb, x.bfloat16())
    xr = xb.float()
    assert torch.allclose(st[:, 0], xr.sum(1), rtol=1e-5, atol=1e-3)
    assert torch.allclose(st[:, 1], (xr * xr).sum(1), rtol=1e-5, atol=1e-3)


def test_rowstats_cast():
    torch.manual_seed(8)
    x = torch.randn(333, 768, device=DEV) * 2 + 0.5
    xb = torch.zeros(333, 768, device=DEV, dtype=torch.bfloat16)
    st = torch.zeros(333, 1, 2, device=DEV)
    _lib.rowstats_cast(x, xb, st)
    st = st[:, 0]
    assert torch.equal(xb, x.bfloat16())
    xr = xb.float()
    assert torch.allclose(st[:, 0], xr.sum(1), rtol=1e-5, atol=1e-3)
    assert torch.allclose(st[:, 1], (xr * xr).sum(1), rtol=1e-5, atol=1e-3)


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
@pytest.mark.parametrize("kernel", [0, 2])      # test hook 1: 0 = 64-key blocks (default), 2 = 128-key blocks
def test_attention(B, N, H, kernel):
    torch.manual_seed(N)
    dh = 64
    I = H * dh
    qkv = torch.randn(B * N, 3 * I, device=DEV).bfloat16()
    out = torch.zeros(B * N, I, device=DEV, dtype=torch.bfloat16)
    _lib.lib().b200vit_debug_set(1, kernel)
    try:
        _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
        torch.cuda.synchronize()
    finally:
        _lib.lib().b200vit_debug_set(1, 0)
    q, k, v = qkv.float().cpu().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    ref = (O.softmax_last((q @ k.transpose(-1, -2)) * dh ** -0.5) @ v).permute(0, 2, 1, 3).reshape(B * N, I)
    # bf16 P and bf16 output: rtol 1e-2 / atol 1e-3 per element, allow 0.5 % stragglers
    assert within(out, ref) > 0.995
    assert (out.float().cpu() - ref).abs().max() < 2e-2


@pytest.mark.parametrize("knob,value,B,N", [(1, 2, 3, 197), (1, 2, 40, 128), (1, 2, 2, 50), (13, 1, 3, 197)])
def test_attention_kernel_variants_agree(knob, value, B, N):
    """b200vit_debug_set(1, 2) streams the keys in 128-key blocks, (13, 1) puts half of the softmax exponentials on
    the FMA pipe: every implementation must produce the same attention."""
    L = _lib.lib()
    torch.manual_seed(7)
    H, dh = 4, 64
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV).bfloat16()
    ref_out = torch.zeros(B * N, H * dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention(qkv, ref_out, B, N, H, dh, dh ** -0.5)
    out = torch.zeros_like(ref_out)
    L.b200vit_debug_set(knob, value)
    if knob == 13:
        L.b200vit_debug_set(1, 2)
    try:
        _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
        torch.cuda.synchronize()
    finally:
        L.b200vit_debug_set(knob, 0)
        L.b200vit_debug_set(1, 0)
    assert within(out, ref_out.float().cpu(), rtol=2e-2, atol=2e-3) > 0.999


@pytest.mark.parametrize("B,N,H", [(2, 257, 16), (3, 197, 4), (5, 64, 2), (2, 400, 3), (1, 512, 2), (40, 129, 5)])
def test_attention_dim_head_80(B, N, H):
    """Canonical ViT-H/14 head width (reference vit.py:86 `dim_head`)."""
    torch.manual_seed(N)
    dh = 80
    I = H * dh
    qkv = torch.randn(B * N, 3 * I, device=DEV).bfloat16()
    out = torch.zeros(B * N, I, device=DEV, dtype=torch.bfloat16)
    _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
    q, k, v = qkv.float().cpu().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    ref = (O.softmax_last((q @ k.transpose(-1, -2)) * dh ** -0.5) @ v).permute(0, 2, 1, 3).reshape(B * N, I)
    d = (out.float().cpu() - ref).abs().view(B * N, H, dh)
    print(f"dh80 B{B} N{N}: max err dims 0..63 {d[..., :64].max():.4f}, dims 64..79 {d[..., 64:].max():.4f}")
    assert within(out, ref) > 0.995
    assert (out.float().cpu() - ref).abs().max() < 2e-2


@pytest.mark.parametrize("dh", [64, 80])
@pytest.mark.parametrize("B,N,H", [(3, 257, 4), (2, 258, 2), (2, 260, 3), (40, 257, 16), (1, 261, 2), (300, 257, 2)])
def test_attention_key_tail(B, N, H, dh):
    """N = 256 + (1..5): the last keys sit alone in the final key block.  Checked against the fp32 oracle with the tail
    keys made the dominant ones, with 64-key and 128-key blocks (test hook 1 = 1 / 2), and the two against each other."""
    torch.manual_seed(N + dh)
    I = H * dh
    qkv = torch.randn(B * N, 3 * I, device=DEV)
    qkv.view(B, N, 3, I)[:, N - 2:, 1] *= 2.5            # the last keys attract most of the attention
    qkv = qkv.bfloat16()
    L = _lib.lib()
    outs = {}
    for tails in (1, 2):
        out = torch.zeros(B * N, I, device=DEV, dtype=torch.bfloat16)
        L.b200vit_debug_set(1, tails)
        try:
            _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
            torch.cuda.synchronize()
        finally:
            L.b200vit_debug_set(1, 0)
        outs[tails] = out.float().cpu()
    q, k, v = qkv.float().cpu().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    ref = (O.softmax_last((q @ k.transpose(-1, -2)) * dh ** -0.5) @ v).permute(0, 2, 1, 3).reshape(B * N, I)
    for tails in (1, 2):
        assert within(outs[tails], ref) > 0.995, tails
        assert (outs[tails] - ref).abs().max() < 2e-2, tails
    assert (outs[1] - outs[2]).abs().max() < 2e-2


def test_attention_is_deterministic_and_batch_invariant():
    """The same (image, head) must give the same bits wherever it lands in the batch and on repeated launches."""
    torch.manual_seed(11)
    B, N, H, dh = 64, 197, 12, 64
    _lib.lib().b200vit_debug_set(1, 2)          # 128-key blocks (test hook), restored below
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
    _lib.lib().b200vit_debug_set(1, 0)
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
    ref = x0.cpu() + a.float().cpu() @ w.float().cpu().t() + bias.cpu()
    for ew in (1, 2):
        x, xb, st, y = res[ew]
        assert torch.isfinite(st).all()
        assert within(x, ref, rtol=1e-3, atol=2e-3) > 0.999
        assert torch.equal(xb, x.bfloat16())
        assert torch.allclose(st[:, 0].cpu(), xb.float().sum(1).cpu(), rtol=1e-3, atol=1e-2)
        assert torch.allclose(st[:, 1].cpu(), (xb.float() ** 2).sum(1).cpu(), rtol=1e-3, atol=1e-2)
    assert torch.equal(res[1][0], res[2][0]) and torch.equal(res[1][3], res[2][3])


def test_attention_large_logits_are_stable():
    torch.manual_seed(9)
    B, N, H, dh = 2, 197, 2, 64
    qkv = (torch.randn(B * N, 3 * H * dh, device=DEV) * 6).bfloat16()      # |s| up to ~300: softmax nearly one-hot
    out = torch.zeros(B * N, H * dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5)
    assert torch.isfinite(out.float()).all()
    q, k, v = qkv.float().cpu().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    ref = (O.softmax_last((q @ k.transpose(-1, -2)) * dh ** -0.5) @ v).permute(0, 2, 1, 3).reshape(B * N, H * dh)
    assert within(out, ref, rtol=2e-2, atol=2e-2) > 0.99


def test_mean_pool_and_cast():
    torch.manual_seed(10)
    x = torch.randn(8, 197, 768, device=DEV)
    o = torch.zeros(8, 768, device=DEV)
    _lib.mean_pool(x, o, 8, 197, 768)
    assert torch.allclose(o.cpu(), x.cpu().mean(1), rtol=1e-5, atol=1e-6)
    xb = torch.zeros(x.numel(), device=DEV, dtype=torch.bfloat16)
    _lib.cast_f32_bf16(x.view(-1), xb)
    assert torch.equal(xb.cpu(), x.view(-1).cpu().bfloat16())


def test_kernels_were_launched_by_the_library():
    assert _lib.launch_count() > 0
