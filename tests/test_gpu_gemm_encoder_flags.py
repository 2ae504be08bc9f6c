"""The GEMM instances compiled for the encoder layer's flag sets against the direct-store epilogue (test hook 14), bit
for bit, row statistics included: the ViT-B/16 layer's four GEMMs, with the encoder's flags, buffers and in-place fp32
residual, at M = 512 * 197 (whole 128-row tiles, several tiles per CTA) and at an M tail with fewer tiles than SMs."""
import math

import pytest
import torch

from vit_pytorch_b200 import _lib

DEV = "cuda"
D, HIDDEN = 768, 3072


def _direct(v):
    _lib.lib().b200vit_debug_set(14, int(v))


def _run(name, M, seed, direct):
    g = torch.Generator(device=DEV).manual_seed(seed)
    n, k = {"qkv": (3 * D, D), "fc1": (HIDDEN, D), "out_proj": (D, D), "fc2": (D, HIDDEN),
            "fc2_no_bias": (D, HIDDEN)}[name]
    a = (torch.randn(M, k, device=DEV, generator=g) + 0.1).bfloat16()
    w = (torch.randn(n, k, device=DEV, generator=g) / math.sqrt(k)).bfloat16()
    b = torch.randn(n, device=DEV, generator=g)
    _direct(direct)
    try:
        if name in ("qkv", "fc1"):
            # LN-fold row sums over the parts the residual GEMMs write (stats_parts(768) = 6), as the encoder passes
            af = a.float()
            sums = torch.stack([af.sum(1), (af * af).sum(1)], 1)
            w6 = torch.tensor([0.25, 0.25, 0.125, 0.125, 0.125, 0.125], device=DEV)
            parts = (sums[:, None, :] * w6[None, :, None]).contiguous()
            col_s = w.float().sum(1).contiguous()
            out = torch.full((M, n), 7.0, device=DEV, dtype=torch.bfloat16)
            _lib.gemm(a, w, out_bf16=out, bias=b, gelu=name == "fc1", ln_sums=parts, col_s=col_s)
            torch.cuda.synchronize()
            return (out,)
        x = torch.randn(M, n, device=DEV, generator=g)
        xb = torch.full((M, n), 7.0, device=DEV, dtype=torch.bfloat16)
        st = torch.full((M, _lib.stats_parts(n), 2), float("nan"), device=DEV)
        _lib.gemm(a, w, out_bf16=xb, out_f32=x, bias=None if name == "fc2_no_bias" else b, resid=x, stats_out=st)
        torch.cuda.synchronize()
        return xb, x, st
    finally:
        _direct(0)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [512 * 197, 7 * 197])
@pytest.mark.parametrize("name", ["qkv", "fc1", "out_proj", "fc2", "fc2_no_bias"])
def test_encoder_flag_sets_match_direct_store(name, M):
    new = _run(name, M, 3, False)
    old = _run(name, M, 3, True)
    for u, v in zip(new, old):
        assert torch.equal(u, v), name
    if len(new) == 3:
        assert not torch.isnan(new[2]).any()
