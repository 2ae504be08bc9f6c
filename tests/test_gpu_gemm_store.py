"""The TMA-store epilogue of b200vit_gemm_bf16 against the direct-store epilogue (test hook 14), bit for bit: every
flag combination the library issues, both tile widths (hook 12; 256-wide residual tiles store directly either way),
M and N tails, row strides wider than N, residuals in place and from their own buffer, and launches with several tiles
per CTA, which reuse the staging buffers and residual slabs.  Rows past M and columns between N and the row stride
are never written."""
import math
import os
import shutil
import subprocess

import pytest
import torch

from oracle import bounds as Bd
from vit_pytorch_b200 import _lib

DEV = "cuda"
K = 192
MS = (1, 257, 300)
NS = (36, 200, 320, 392)   # inside one box, across 64-column boxes, 256 + 64, 256 + 136
MODES = ("bias", "bias_lnfold", "bias_lnfold_gelu", "resid_stats", "resid_stats_bias", "resid_stats_bias_separate")


def test_library_contains_tma_stores():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump) or not _lib.LIB_PATH.exists():
        pytest.skip("cuobjdump or library not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True).stdout
    assert "UTMASTG" in sass


def _hooked(direct, block_n, fn):
    L = _lib.lib()
    L.b200vit_debug_set(14, int(direct))
    L.b200vit_debug_set(12, block_n)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        L.b200vit_debug_set(14, 0)
        L.b200vit_debug_set(12, 0)


def _inputs(M, N, seed, ldo=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = (torch.randn(M, K, device=DEV, generator=g) + 0.1).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device=DEV, generator=g)
    col_s = w.float().sum(1).contiguous()
    af = a.float()
    sums = torch.stack([af.sum(1), (af * af).sum(1)], 1)
    parts = torch.stack([sums * 0.5, sums * 0.25, sums * 0.25], 1).contiguous()
    r_full = torch.randn(M + 2, ldo or N, device=DEV, generator=g)
    return a, w, b, col_s, parts, r_full


def _run(mode, M, N, ldo, direct, block_n, seed):
    """One launch into buffers of two extra rows and row stride ldo, pre-filled with sentinels; returns the full
    buffers so that the caller sees the untouched margins too."""
    a, w, b, col_s, parts, r_full = _inputs(M, N, seed, ldo)
    ob_full = torch.full((M + 2, ldo), 7.0, device=DEV, dtype=torch.bfloat16)
    ob = ob_full[:M, :N]
    if mode.startswith("resid"):
        in_place = not mode.endswith("separate")
        of_full = r_full.clone() if in_place else torch.full((M + 2, ldo), 5.0, device=DEV)
        of = of_full[:M, :N]
        st = torch.full((M, _lib.stats_parts(N), 2), float("nan"), device=DEV)
        resid = of if in_place else r_full[:M, :N]
        bias = b if "bias" in mode.split("_")[2:] else None
        _hooked(direct, block_n, lambda: _lib.gemm(a, w, out_f32=of, out_bf16=ob, bias=bias, resid=resid, stats_out=st))
        return ob_full, of_full, st, r_full
    lnfold = "lnfold" in mode
    _hooked(direct, block_n, lambda: _lib.gemm(a, w, out_bf16=ob, bias=b, gelu=mode.endswith("gelu"),
                                               ln_sums=parts if lnfold else None, col_s=col_s if lnfold else None))
    return ob_full, None, None, r_full


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [1, 2])
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("mode", MODES)
def test_tma_store_matches_direct_store(mode, N, block_n):
    for M in MS:
        for ldo in sorted({(N // 8 + 1) * 8, N if N % 8 == 0 else (N // 8 + 1) * 8}):
            seed = M * 1000 + N + ldo
            new = _run(mode, M, N, ldo, False, block_n, seed)
            old = _run(mode, M, N, ldo, True, block_n, seed)
            for u, v in zip(new[:3], old[:3]):
                if u is not None:
                    assert torch.equal(u, v), (mode, M, N, ldo)
            ob_full, of_full, _, r_full = new
            # margins: sentinels, or the residual that was there (in place)
            assert (ob_full[M:] == 7.0).all() and (ob_full[:, N:] == 7.0).all()
            if of_full is not None:
                pad = r_full if not mode.endswith("separate") else torch.full_like(r_full, 5.0)
                assert torch.equal(of_full[M:], pad[M:]) and torch.equal(of_full[:, N:], pad[:, N:])
                assert torch.equal(ob_full[:M, :N], of_full[:M, :N].bfloat16())


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [0, 1, 2])
@pytest.mark.parametrize("mode", ["bias_lnfold_gelu", "resid_stats_bias", "resid_stats_bias_separate"])
def test_tma_store_many_tiles_per_cta(mode, block_n):
    """More than two tiles per CTA, so every CTA writes its staging buffers and residual slabs again after their
    previous stores, plus an M tail."""
    M, N = 2 * 128 * torch.cuda.get_device_properties(0).multi_processor_count + 1, 320
    new = _run(mode, M, N, N, False, block_n, seed=17)
    old = _run(mode, M, N, N, True, block_n, seed=17)
    for u, v in zip(new[:3], old[:3]):
        if u is not None:
            assert torch.equal(u, v)
    assert (new[0][M:] == 7.0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [1, 2])
def test_tma_store_matches_reference(block_n):
    M, N, ldo = 300, 392, 400
    ob_full, _, _, _ = _run("bias_lnfold_gelu", M, N, ldo, False, block_n, seed=11)
    a, w, b, col_s, parts, _ = _inputs(M, N, 11, ldo)
    Bd.check(ob_full[:M, :N], *Bd.gemm_reference(a, w, bias=b, ln_sums=parts, col_s=col_s, gelu=True, bf16_out=True),
             f"TMA store, hook 12 = {block_n}")


@pytest.mark.gpu
def test_headnorm_gemm_matches_direct_store():
    M, heads, dh = 257, 2, 64
    N = 3 * heads * dh
    a, w, b, col_s, parts, _ = _inputs(M, N, 5)
    gamma = torch.rand(2 * heads * dh, device=DEV) + 0.5
    outs = []
    for direct in (False, True):
        full = torch.full((M + 2, N), 7.0, device=DEV, dtype=torch.bfloat16)
        _hooked(direct, 0, lambda: _lib.gemm_headnorm(a, w, out_bf16=full[:M], head_gamma=gamma, norm_heads=2 * heads,
                                                      dh=dh, bias=b, ln_sums=parts, col_s=col_s))
        assert (full[M:] == 7.0).all()
        outs.append(full)
    assert torch.equal(*outs)


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [1, 2])
def test_unaligned_bf16_rows_store_directly(block_n):
    """ldo = 36 bf16 (72-byte rows) cannot be a TMA tensor: the launch stores from the registers and is still right."""
    M, N = 300, 36
    a, w, b, _, _, _ = _inputs(M, N, 3)
    full = torch.full((M + 2, N), 7.0, device=DEV, dtype=torch.bfloat16)
    _hooked(False, block_n, lambda: _lib.gemm(a, w, out_bf16=full[:M], bias=b))
    assert (full[M:] == 7.0).all()
    assert torch.allclose(full[:M].float(), a.float() @ w.float().t() + b, rtol=1e-2, atol=2e-2)
