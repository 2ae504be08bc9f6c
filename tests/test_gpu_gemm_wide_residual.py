"""The 256-wide residual GEMM with TMA stores (gemm_bf16_kernel<256, 4, false, true, true>) against the 128-wide
TMA-store instance (test hook 12 = 1) and the 256-wide direct-store instance (hook 14), bit for bit: the fp32 sum, its
bf16 copy and the row statistics.  Residuals in place and from their own buffer, with and without bias; N tails
inside and across the four 64-column slabs of a tile; row strides wider than N; M tails; k-block counts around the
4-stage ring; and grids in which every CTA runs several tiles, so that it reuses its residual slabs and staging
chunk.  Rows past M and columns between N and the row stride are never written.  One fp64 check at an encoder
shape."""
import math

import pytest
import torch

from oracle import bounds as Bd
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
STAGES = 4                          # ring stages of the 256-wide residual instance
F32_SENT, BF16_SENT = 5.0, 7.0

# (block_n hook, direct-store hook) of the instance under test and of its two references
WIDE_TMA, NARROW_TMA, WIDE_DIRECT = (2, 0), (1, 0), (2, 1)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(M, N, K, ldo, in_place, bias, hooks, seed):
    """One launch into buffers of two extra rows and row stride ldo around the output; returns the full buffers and
    the residual buffer it was given (the margins hold sentinels, or -- in place -- the residual that was there)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = (torch.randn(M, K, device=DEV, generator=g) + 0.1).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device=DEV, generator=g)
    r_full = torch.randn(M + 2, ldo, device=DEV, generator=g)
    of_full = r_full.clone() if in_place else torch.full((M + 2, ldo), F32_SENT, device=DEV)
    ob_full = torch.full((M + 2, ldo), BF16_SENT, device=DEV, dtype=torch.bfloat16)
    st = torch.full((M, _lib.stats_parts(N), 2), float("nan"), device=DEV)
    resid = of_full[:M, :N] if in_place else r_full[:M, :N]
    L = _lib.lib()
    L.b200vit_debug_set(12, hooks[0])
    L.b200vit_debug_set(14, hooks[1])
    try:
        _lib.gemm(a, w, out_f32=of_full[:M, :N], out_bf16=ob_full[:M, :N], bias=b if bias else None, resid=resid,
                  stats_out=st)
        torch.cuda.synchronize()
    finally:
        L.b200vit_debug_set(12, 0)
        L.b200vit_debug_set(14, 0)
    return ob_full, of_full, st, r_full


def _agree(M, N, K, ldo, in_place=True, bias=True, seed=0):
    new = _run(M, N, K, ldo, in_place, bias, WIDE_TMA, seed)
    for ref in (NARROW_TMA, WIDE_DIRECT):
        old = _run(M, N, K, ldo, in_place, bias, ref, seed)
        for what, u, v in zip(("bf16", "fp32", "stats"), new[:3], old[:3]):
            assert torch.equal(u, v), (what, ref, M, N, K, ldo, in_place, bias)
    ob_full, of_full, _, r_full = new
    assert (ob_full[M:] == BF16_SENT).all() and (ob_full[:, N:] == BF16_SENT).all()
    pad = r_full if in_place else torch.full_like(r_full, F32_SENT)
    assert torch.equal(of_full[M:], pad[M:]) and torch.equal(of_full[:, N:], pad[:, N:])
    assert torch.equal(ob_full[:M, :N], of_full[:M, :N].bfloat16())


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("in_place", [True, False])
@pytest.mark.parametrize("N", [200, 320, 392, 768, 1024, 1280])
def test_wide_residual_matches_narrow_and_direct(N, in_place, bias):
    for M in (1, 300):
        for ldo in (N, N + 24):
            _agree(M, N, 192, ldo, in_place, bias, seed=M * 7 + N + ldo)


@pytest.mark.parametrize("K", [64, 64 * (STAGES - 1), 64 * (STAGES + 1), 64 * (2 * STAGES + 1), 3072, 3000])
def test_wide_residual_k_blocks(K):
    """1, S - 1, S + 1 and 2S + 1 k blocks of the S-stage ring, FC2's K, and a K whose last block is partial."""
    _agree(257, 768, K, 776, seed=K)


@pytest.mark.parametrize("extra", [(0, 1), (1, -1), (1, 0), (1, 1), (2, 1), (4, 3)])
def test_wide_residual_tiles_per_cta(extra):
    """1, SMs - 1, SMs, SMs + 1, 2 SMs + 1 and 4 SMs + 3 tiles of 128 x 256 (N = 256, an M tail in the last row of
    tiles): from one tile per CTA to five, each reusing the CTA's slabs and staging chunk."""
    tiles = extra[0] * _sms() + extra[1]
    _agree(128 * tiles - 37, 256, 128, 264, in_place=extra[1] != 0, seed=tiles)


def test_wide_residual_fp64_bound():
    """The encoder's FC2 shape (N 768, K 3072) against an fp64 reference, element by element, in row chunks."""
    M, N, K, chunk = 2 * 128 * _sms() + 77, 768, 3072, 8192
    x = Bd.gemm_inputs(M, N, K, seed=21, device=DEV)
    ob_full, of_full, st = _run_fp64_case(x, M, N)
    for r0 in range(0, M, chunk):
        rs = slice(r0, min(r0 + chunk, M))
        ref, e = Bd.gemm_reference(x["a"][rs], x["w"], bias=x["bias"], resid=x["resid"][rs])
        Bd.check(of_full[rs], ref, e, f"wide residual fp32 rows {r0}+")
        Bd.check(ob_full[rs], ref, Bd.bf16_bound(ref, e), f"wide residual bf16 rows {r0}+")
        sref, sb = Bd.stats_reference(ob_full[rs], st.shape[1])
        Bd.check(st[rs], sref, sb, f"wide residual stats rows {r0}+")


def _run_fp64_case(x, M, N):
    of = x["resid"].clone()
    ob = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    st = torch.empty(M, _lib.stats_parts(N), 2, device=DEV)
    L = _lib.lib()
    L.b200vit_debug_set(12, WIDE_TMA[0])
    try:
        _lib.gemm(x["a"], x["w"], out_f32=of, out_bf16=ob, bias=x["bias"], resid=of, stats_out=st)
        torch.cuda.synchronize()
    finally:
        L.b200vit_debug_set(12, 0)
    return ob, of, st
