"""-m gpu: every output element of the softmax attention kernels of attention.cu (b200vit_attention / _ex,
b200vit_attention_varlen / _ex) within its bound of the fp64 reference of oracle/attention_bounds.py, which replays the
kernel's deliberate bf16 rounding of the probabilities and bounds only its fp32 noise and the output rounding.

Every instance (the default kernel of each length, the tiled kernel at every length, MASK_SELF) on four input
distributions (attention_bounds.KINDS), at the key counts around the block edges, the production launches with more
CTAs than two waves, a NaViT pack and single sequences of 4097 and 16384 keys.  Outputs start as NaN, so an element the
kernel does not write fails too.  The worst |got - ref| / bound of each kernel and instance is printed at the end of the
module."""
import contextlib
import random

import pytest
import torch

from oracle import attention_bounds as AB
from oracle import bounds as Bd
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
# instance: (test hook 15, MASK_SELF) of b200vit_attention; hook 15 = 1 runs the tiled kernel at 128 < N <= 256 too
PLAIN_CONFIGS = {"default": (0, False), "tiled": (1, False), "mask_self": (0, True)}
# instance: MASK_SELF of b200vit_attention_varlen
VARLEN_CONFIGS = {"kb64": False, "mask_self": True}
LENGTHS = (1, 2, 16, 63, 64, 65, 127, 128, 129, 197, 256, 257, 511, 512)
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst |got - ref| / bound per kernel and instance:")
    for key in sorted(WORST):
        print(f"  {key}: {WORST[key]:.3f}")


def record(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), ratio)


@contextlib.contextmanager
def hooks(**kv):
    """Test hooks of include/b200vit.h (key -> value), reset to 0 afterwards."""
    L = _lib.lib()
    try:
        for k, v in kv.items():
            assert L.b200vit_debug_set(int(k[1:]), v) == 0
        yield
    finally:
        for k in kv:
            L.b200vit_debug_set(int(k[1:]), 0)


def plain_bound(qkv, B, N, H, dh, cfg):
    """b200vit_attention under instance `cfg` against its bound: returns the worst ratio."""
    k15, ms = PLAIN_CONFIGS[cfg]
    out = torch.full((B * N, H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    with hooks(k15=k15):
        _lib.attention(qkv, out, B, N, H, dh, dh ** -0.5, mask_self=ms)
        torch.cuda.synchronize()
    ref, bound = AB.qkv_attention_reference(qkv, [N] * B, H, dh, dh ** -0.5, mask_self=ms)
    ratio = Bd.check(out, ref, bound, f"attention {cfg} B{B} N{N} H{H} dh{dh}")
    record(("attention", cfg), ratio)
    return ratio


def varlen_bound(qkv, lengths, H, dh, cfg):
    ms = VARLEN_CONFIGS[cfg]
    cu, tp, tiles = _lib.varlen_index(lengths, DEV)
    out = torch.full((sum(lengths), H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attention_varlen(qkv, out, cu, tp, tiles, H, dh, dh ** -0.5, mask_self=ms)
    torch.cuda.synchronize()
    ref, bound = AB.qkv_attention_reference(qkv, lengths, H, dh, dh ** -0.5, mask_self=ms)
    ratio = Bd.check(out, ref, bound, f"attention_varlen {cfg} {len(lengths)} sequences H{H} dh{dh}")
    record(("attention_varlen", cfg), ratio)
    return ratio


@pytest.mark.parametrize("kind", AB.KINDS)
@pytest.mark.parametrize("cfg", sorted(PLAIN_CONFIGS))
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_attention_within_bound(dh, cfg, kind):
    B, H = 2, 2
    for N in LENGTHS:
        qkv = AB.qkv_inputs(kind, [N] * B, H, dh, seed=N * 7 + dh, device=DEV)
        plain_bound(qkv, B, N, H, dh, cfg)


# (name, H, dh, N, MASK_SELF): ViT-B/16, ViT-L/16, ViT-H/14 at 224 px and the small-dataset ViT's LSA at 32 px / p 4
PRODUCTION = [("vit_b16", 12, 64, 197, False), ("vit_l16", 16, 64, 197, False), ("vit_h14", 16, 80, 257, False),
              ("lsa", 16, 64, 65, True)]


@pytest.mark.parametrize("kind", AB.KINDS)
@pytest.mark.parametrize("name,H,dh,N,ms", PRODUCTION)
def test_attention_production_launch_within_bound(name, H, dh, N, ms, kind):
    """A batch whose grid exceeds two waves of the device's SMs, so CTAs run back to back on each SM."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = (N + 127) // 128
    B = 2 * sms // (tiles * H) + 1
    assert B * tiles * H > 2 * sms
    qkv = AB.qkv_inputs(kind, [N] * B, H, dh, seed=B + N, device=DEV)
    plain_bound(qkv, B, N, H, dh, "mask_self" if ms else "default")


def navit_lengths(count, seed):
    """Images of side 16 * randrange(4, 33) pixels in 16-pixel patches: 16 to 1024 tokens each (bench.py's navit)."""
    rng = random.Random(seed)
    return [rng.randrange(4, 33) * rng.randrange(4, 33) for _ in range(count)]


@pytest.mark.parametrize("kind", AB.KINDS)
@pytest.mark.parametrize("cfg", sorted(VARLEN_CONFIGS))
@pytest.mark.parametrize("dh", [64, 80])
def test_attention_varlen_navit_pack_within_bound(dh, cfg, kind):
    lengths = navit_lengths(12, seed=dh) + [1, 2, 129]
    H = 3
    qkv = AB.qkv_inputs(kind, lengths, H, dh, seed=len(kind) + dh, device=DEV)
    varlen_bound(qkv, lengths, H, dh, cfg)


@pytest.mark.parametrize("N", [4097, 16384])
def test_attention_varlen_long_sequence_within_bound(N):
    H, dh = 2, 64
    qkv = AB.qkv_inputs("normal", [N], H, dh, seed=N, device=DEV)
    varlen_bound(qkv, [N], H, dh, "kb64")


@pytest.mark.parametrize("N,varlen", [(512, False), (4096, True), (16384, True)])
def test_pv_accumulation_error_against_c_acc(N, varlen):
    """C_ACC was measured on GEMM chains of K <= 832; P V chains run to 16384 keys.  With q = 0 every e is exactly 1,
    l = N and 1 / l = 2^-log2(N) exactly, so got * N is the bf16 rounding of the kernel's fp32 sum of the values; the
    values spread over 17 binades, and the last key cancels the others' sum, so the sum is small against sum |v| and
    the bf16 rounding does not hide the accumulation error.  Measured |O - sum v| / (N u sum|v|) must stay below
    C_ACC."""
    H, dh = 1, 64
    g = torch.Generator(device=DEV).manual_seed(N)
    v = torch.randn(N, dh, generator=g, device=DEV) * torch.exp2(torch.randint(-8, 9, (N, dh), generator=g, device=DEV))
    v = v.bfloat16()
    v[-1] = (-v[:-1].double().sum(0)).bfloat16()
    qkv = torch.zeros(N, 3 * dh, device=DEV, dtype=torch.bfloat16)
    qkv[:, dh:2 * dh] = torch.randn(N, dh, generator=g, device=DEV).bfloat16()
    qkv[:, 2 * dh:] = v
    out = torch.full((N, dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    if varlen:
        cu, tp, tiles = _lib.varlen_index([N], DEV)
        _lib.attention_varlen(qkv, out, cu, tp, tiles, H, dh, dh ** -0.5)
    else:
        _lib.attention(qkv, out, 1, N, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    s = v.double().sum(0)
    got = out.double() * N                                                 # = bf16(O), O the fp32 sum
    err = ((got - s[None]).abs() - 0.5 * Bd.bf16_ulp(got)).clamp_min(0)    # |O - sum v| is at least this
    ratio = (err / (N * Bd.U * v.double().abs().sum(0)[None])).max().item()
    res = (0.5 * Bd.bf16_ulp(got) / (N * Bd.U * v.double().abs().sum(0)[None])).max().item()
    print(f"P V chain of {N} keys: worst |O - sum v| / (K u sum|v|) >= {ratio:.4f} (resolution {res:.4f})")
    record(("pv_chain_over_K_u_abs", f"K={N}"), ratio)
    assert res < 0.05 and ratio <= Bd.C_ACC
    ref, bound = AB.qkv_attention_reference(qkv, [N], H, dh, dh ** -0.5)
    Bd.check(out, ref, bound, f"uniform N{N}")
