"""Head widths of the fused path (dim_head 32, 64, 80, 128): the one Python rule, and the C ABI's argument checks for
every entry point that takes a head width (no compute, no GPU needed: every call below fails its argument checks
before it touches a device)."""
import ctypes

import pytest

from vit_pytorch_b200 import ViT, _lib, build
from vit_pytorch_b200.engine import HEAD_WIDTHS, head_width_reason
from vit_pytorch_b200.simple_vit_with_qk_norm import SimpleViT as QKNormViT

SUPPORTED = (32, 64, 80, 128)
REFUSED = (16, 48, 96, 160)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_supported_widths():
    assert tuple(HEAD_WIDTHS) == SUPPORTED
    for dh in SUPPORTED:
        assert head_width_reason(dh) is None
    for dh in REFUSED:
        r = head_width_reason(dh)
        assert r is not None and f"dim_head={dh}" in r and "32, 64, 80 and 128" in r


@pytest.mark.parametrize("dh", SUPPORTED + REFUSED)
def test_unsupported_reason_follows_the_head_width_rule(dh):
    """At 197 and 1025 tokens (single-pass and key-block attention) and with a per-head q/k norm."""
    heads = 2
    vit = ViT(image_size=32, patch_size=8, num_classes=5, dim=64, depth=1, heads=heads, mlp_dim=96, dim_head=dh)
    qk = QKNormViT(image_size=32, patch_size=8, num_classes=5, dim=64, depth=1, heads=heads, mlp_dim=96, dim_head=dh)
    for m in (vit, qk):
        eng = m.transformer.engine()
        for n in (197, 1025):
            r = eng.unsupported_reason(n)
            if dh in SUPPORTED:
                assert r is None, (type(m).__name__, n, r)
            else:
                assert r is not None and "32, 64, 80 and 128" in r, (type(m).__name__, n, r)


P = ctypes.c_void_p
GOOD = P(256)        # 16-byte aligned, never dereferenced: the calls fail their argument checks first
ODD = P(258)         # not 16-byte aligned


def _err(lib) -> str:
    return lib.b200vit_last_error().decode()


@pytest.mark.parametrize("dh", [32, 128])
def test_new_widths_pass_the_dim_head_check(lib, dh):
    """dh 32 / 128 get past the head-width check of every entry point and fail on the later, invalid argument."""
    # single-pass attention: N > 512, then a misaligned pointer
    assert lib.b200vit_attention(GOOD, GOOD, 1, 4096, 1, dh, 0.1, None) == -1
    assert "512" in _err(lib) and "dim_head" not in _err(lib)
    assert lib.b200vit_attention(ODD, GOOD, 1, 16, 1, dh, 0.1, None) == -1
    assert "16-byte aligned" in _err(lib) and "dim_head" not in _err(lib)
    # key-block attention: misaligned pointer, then a head count beyond the grid
    assert lib.b200vit_attention_varlen(ODD, GOOD, GOOD, GOOD, 1, 16, 1, 1, dh, 0.1, None) == -1
    assert "16-byte aligned" in _err(lib) and "dim_head" not in _err(lib)
    assert lib.b200vit_attention_varlen(GOOD, GOOD, GOOD, GOOD, 1, 16, 1, 70000, dh, 0.1, None) == -1
    assert "exceeds the grid" in _err(lib)
    # head norms: rows that do not hold nheads * dh columns, and a misaligned buffer
    for fn, extra in ((lib.b200vit_rmsnorm_heads, ()), (lib.b200vit_layernorm_heads, (1e-5,))):
        assert fn(GOOD, 3 * dh - 8, GOOD, 4, 3, dh, *extra, None) == -1
        assert f"ld={3 * dh - 8}" in _err(lib) and "dim_head" not in _err(lib)
        assert fn(ODD, 3 * dh, GOOD, 4, 3, dh, *extra, None) == -1
        assert "16-byte aligned" in _err(lib) and "dim_head" not in _err(lib)
    # q/k norm of a packed qkv buffer: the row stride is 3 * H * dh
    assert lib.b200vit_qk_rmsnorm(ODD, GOOD, 4, 5, dh, None) == -1
    assert f"ld={3 * 5 * dh}" in _err(lib) and "rmsnorm_heads" in _err(lib)
    # GEMM + head norm: norm_heads * dh must fit N, then the flags are checked
    assert lib.b200vit_gemm_headnorm_bf16(GOOD, 64, GOOD, 64, GOOD, 64, None, None, 0, 1e-5, None, GOOD, 2, dh, 0.0,
                                          16, 2 * dh - 8, 64, 0, None) == -1
    assert "do not fit" in _err(lib)
    assert lib.b200vit_gemm_headnorm_bf16(GOOD, 64, GOOD, 64, GOOD, 64, None, None, 0, 1e-5, None, GOOD, 2, dh, 0.0,
                                          16, 2 * dh, 64, _lib.EPI_GELU, None) == -1
    assert "unsupported flags" in _err(lib)


def test_norm_heads_times_dh_must_fit_n(lib):
    """The fit check uses the real head width: 2 heads of 80 do not fit 144 columns (2 x 64 would)."""
    assert lib.b200vit_gemm_headnorm_bf16(GOOD, 64, GOOD, 64, GOOD, 64, None, None, 0, 1e-5, None, GOOD, 2, 80, 0.0,
                                          16, 144, 64, 0, None) == -1
    assert "2 heads do not fit N=144" in _err(lib)


def test_refused_width_is_named(lib):
    """dim_head 48 is refused by every entry point that takes a head width, with the width in the message."""
    dh = 48
    calls = {
        "attention": lambda: lib.b200vit_attention(GOOD, GOOD, 1, 16, 1, dh, 0.1, None),
        "attention_varlen": lambda: lib.b200vit_attention_varlen(GOOD, GOOD, GOOD, GOOD, 1, 16, 1, 1, dh, 0.1, None),
        "rmsnorm_heads": lambda: lib.b200vit_rmsnorm_heads(GOOD, 3 * dh, GOOD, 4, 3, dh, None),
        "layernorm_heads": lambda: lib.b200vit_layernorm_heads(GOOD, 3 * dh, GOOD, 4, 3, dh, 1e-5, None),
        "qk_rmsnorm": lambda: lib.b200vit_qk_rmsnorm(GOOD, GOOD, 4, 5, dh, None),
        "attn_pool": lambda: lib.b200vit_attn_pool(GOOD, GOOD, GOOD, GOOD, 2, 3, dh, None),
        "gemm_headnorm": lambda: lib.b200vit_gemm_headnorm_bf16(GOOD, 64, GOOD, 64, GOOD, 64, None, None, 0, 1e-5, None,
                                                                GOOD, 2, dh, 0.0, 16, 2 * dh, 64, 0, None),
    }
    for name, call in calls.items():
        assert call() == -1, name
        msg = _err(lib)
        assert "dim_head=48" in msg and "(32, 64, 80 or 128)" in msg, (name, msg)
