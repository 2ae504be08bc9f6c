"""Residual epilogue of b200vit_gemm_bf16 (the fp32 residual tile staged in shared memory by TMA): in place and from a
separate buffer, row strides wider than N, M and N tails at both tile widths, and its argument check."""
import ctypes
import math

import pytest
import torch

from oracle import bounds as Bd
from vit_pytorch_b200 import _lib, build

DEV = "cuda"


def test_residual_needs_ldo_multiple_of_4():
    if not _lib.LIB_PATH.exists():
        build.build()
    lib = _lib.lib()
    p = ctypes.c_void_p(256)
    # M=4, N=6, K=8, ldo=6: 24-byte rows cannot be a TMA tensor, so the call is refused before any device work
    rc = lib.b200vit_gemm_bf16(p, 8, p, 8, None, p, 6, None, p, None, 0, 1e-5, None, None, 4, 6, 8, _lib.EPI_RESIDUAL,
                               None)
    assert rc == -1 and b"multiple of 4" in lib.b200vit_last_error()


def _run(block_n, M, N, K, ldo, in_place, seed):
    """x = a w^T + bias + r through the library with tile width block_n (hook 12: 1 = 128, 2 = 256) into an fp32
    buffer of row stride ldo; returns (x, bf16 copy, stats, reference)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device=DEV, generator=g)
    r_full = torch.randn(M, ldo, device=DEV, generator=g)
    x_full = r_full.clone() if in_place else torch.full((M, ldo), 5.0, device=DEV)
    xb_full = torch.zeros(M, ldo, device=DEV, dtype=torch.bfloat16)
    st = torch.full((M, _lib.stats_parts(N), 2), float("nan"), device=DEV)
    x, xb = x_full[:, :N], xb_full[:, :N]
    L = _lib.lib()
    L.b200vit_debug_set(12, block_n)
    try:
        _lib.gemm(a, w, out_f32=x, out_bf16=xb, bias=b, resid=x if in_place else r_full[:, :N], stats_out=st)
        torch.cuda.synchronize()
    finally:
        L.b200vit_debug_set(12, 0)
    ref = a.float() @ w.float().t() + b + r_full[:, :N]
    # columns past N are left alone
    pad_ref = r_full[:, N:] if in_place else torch.full_like(r_full[:, N:], 5.0)
    assert torch.equal(x_full[:, N:], pad_ref) and not xb_full[:, N:].any()
    return x, xb, st, ref


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [1, 2])
@pytest.mark.parametrize("M,N,K,ldo", [(300, 320, 192, 320),     # M tail, N tail at both widths (320 = 256 + 64)
                                       (257, 768, 256, 772),     # one-row M tail, ldo > N
                                       (130, 200, 64, 256),      # N tail inside a 64-column slab, ldo > N
                                       (64, 36, 128, 40)])       # a single tile narrower than one 32-column box + 4
def test_residual_separate_and_in_place(block_n, M, N, K, ldo):
    seed = M + N + K
    x1, xb1, st1, ref = _run(block_n, M, N, K, ldo, in_place=True, seed=seed)
    x2, xb2, st2, _ = _run(block_n, M, N, K, ldo, in_place=False, seed=seed)
    assert torch.allclose(x1, ref, rtol=1e-4, atol=1e-4)
    # the same arithmetic whether the residual is read in place or from its own buffer
    assert torch.equal(x1, x2) and torch.equal(xb1, xb2) and torch.equal(st1, st2)
    assert torch.equal(xb1, x1.bfloat16())
    s = st1.sum(1)
    xr = xb1.float()
    assert torch.allclose(s[:, 0], xr.sum(1), rtol=1e-4, atol=1e-2)
    assert torch.allclose(s[:, 1], (xr * xr).sum(1), rtol=1e-4, atol=1e-2)


@pytest.mark.gpu
def test_residual_tile_widths_agree():
    """Both tile widths give the same bits on a multi-tile problem with a partial last N tile."""
    outs = [_run(bn, 700, 640, 320, 640, in_place=True, seed=7)[:3] for bn in (1, 2)]
    for u, v in zip(*outs):
        assert torch.equal(u, v)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [1, 2])
def test_bias_lnfold_gelu_n_tail(block_n):
    """Bias, col_s and the LN-fold row sums staged in shared memory, N not a multiple of either tile width."""
    torch.manual_seed(3)
    M, N, K = 333, 392, 256
    a = (torch.randn(M, K, device=DEV) + 0.2).bfloat16()
    w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device=DEV)
    col_s = w.float().sum(1).contiguous()
    af = a.float()
    sums = torch.stack([af.sum(1), (af * af).sum(1)], 1)
    parts = torch.stack([sums * 0.5, sums * 0.25, sums * 0.25], 1).contiguous()   # three partial sums per row
    out = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    plain = torch.zeros(M, N, device=DEV)
    L = _lib.lib()
    L.b200vit_debug_set(12, block_n)
    try:
        _lib.gemm(a, w, out_bf16=out, bias=b, gelu=True, ln_sums=parts, col_s=col_s)
        _lib.gemm(a, w, out_f32=plain, bias=b)
        torch.cuda.synchronize()
    finally:
        L.b200vit_debug_set(12, 0)
    assert torch.allclose(plain, af @ w.float().t() + b, rtol=1e-4, atol=1e-4)
    Bd.check(out, *Bd.gemm_reference(a, w, bias=b, ln_sums=parts, col_s=col_s, gelu=True, bf16_out=True),
             f"LN fold + GELU, hook 12 = {block_n}")
