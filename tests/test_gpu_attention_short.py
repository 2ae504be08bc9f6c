"""-m gpu: the persistent attention kernel for 129 to 256 tokens against the tiled kernel it stands in for.

b200vit_attention_ex sends fixed-length launches with 128 < N <= 256 and dim_head 32 or 64 to the persistent kernel of
csrc/attention_short.cu; test hook 15 keeps them on the tiled kernel of csrc/attention.cu.  The two run the same
arithmetic per 64-key block (the persistent one narrows the last block to the keys that exist), so every output must be
the same bits: on Gaussian inputs, next to a NaN / Inf image, with several (image, head) items per CTA and a ragged last
round, and from one run to the next.  Rows of `out` past B N stay untouched.
"""
import contextlib

import pytest
import torch

from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
WIDTHS = [32, 64]                                  # the head widths the persistent kernel is built for
LENGTHS = [129, 130, 144, 191, 192, 193, 197, 208, 255, 256]
BATCHES = [1, 3, 300]                              # 300 x H items: several per CTA and a ragged last round


@contextlib.contextmanager
def tiled_kernel():
    """Test hook 15 of include/b200vit.h: every fixed-length launch takes the tiled kernel."""
    L = _lib.lib()
    assert L.b200vit_debug_set(15, 1) == 0
    try:
        yield
    finally:
        L.b200vit_debug_set(15, 0)


def run(qkv, B, N, H, dh, tail_rows=7):
    """Output rows [0, B N) and the `tail_rows` rows of the allocation behind them (filled with 5)."""
    buf = torch.full((B * N + tail_rows, H * dh), 5.0, device=DEV, dtype=torch.bfloat16)
    _lib.attention(qkv, buf[:B * N], B, N, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    return buf[:B * N], buf[B * N:]


def same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("N", LENGTHS)
@pytest.mark.parametrize("dh", WIDTHS)
def test_short_kernel_matches_tiled_kernel_bit_for_bit(dh, N, B):
    H = 2
    g = torch.Generator(device=DEV).manual_seed(dh * 100000 + N * 1000 + B)
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV, generator=g).bfloat16()
    with tiled_kernel():
        want, _ = run(qkv, B, N, H, dh)
    got, tail = run(qkv, B, N, H, dh)
    assert torch.isfinite(want.float()).all()
    assert torch.equal(got, want)
    assert (tail == 5.0).all(), "rows past B N were written"
    again, _ = run(qkv, B, N, H, dh)
    assert torch.equal(again, got), "two runs differ"


@pytest.mark.parametrize("B", [3, 300])
@pytest.mark.parametrize("N", LENGTHS)
@pytest.mark.parametrize("dh", WIDTHS)
def test_short_kernel_next_to_a_nan_image(dh, N, B):
    """Image 1 all NaN, image 2 with +Inf values: every other image as in the clean run, and the whole output the
    bits of the tiled kernel."""
    H = 2
    I = H * dh
    g = torch.Generator(device=DEV).manual_seed(dh * 100000 + N * 1000 + B + 1)
    qkv = torch.randn(B * N, 3 * I, device=DEV, generator=g).bfloat16()
    clean, _ = run(qkv, B, N, H, dh)
    bad = qkv.clone()
    bad[N:2 * N] = float("nan")
    bad[2 * N:3 * N, 2 * I:] = float("inf")
    with tiled_kernel():
        want, _ = run(bad, B, N, H, dh)
    got, tail = run(bad, B, N, H, dh)
    assert same_bits(got, want)
    assert torch.equal(got[:N], clean[:N]) and torch.equal(got[3 * N:], clean[3 * N:])
    assert torch.isnan(got[N:2 * N].float()).all()
    assert (tail == 5.0).all()


def kernels_launched(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages()]


def test_dispatch_by_length_width_and_hooks():
    """The persistent kernel runs for 128 < N <= 256 at dim_head 32 and 64, and nowhere else."""
    H = 2

    def names(N, dh, mask_self=False):
        qkv = torch.randn(2 * N, 3 * H * dh, device=DEV).bfloat16()
        out = torch.empty(2 * N, H * dh, device=DEV, dtype=torch.bfloat16)
        return kernels_launched(lambda: _lib.attention(qkv, out, 2, N, H, dh, dh ** -0.5, mask_self=mask_self))

    def is_short(ks):
        short = [k for k in ks if "attention_short_kernel" in k]
        tiled = [k for k in ks if "attention_kernel" in k]
        assert len(short) + len(tiled) == 1, ks
        return bool(short)

    for dh in WIDTHS:
        assert not is_short(names(128, dh)) and is_short(names(129, dh))
        assert is_short(names(256, dh)) and not is_short(names(257, dh))
        assert not is_short(names(197, dh, mask_self=True))
        with tiled_kernel():
            assert not is_short(names(197, dh))
    for dh in (80, 128):                           # two resident items do not fit in shared memory
        assert not is_short(names(197, dh))
