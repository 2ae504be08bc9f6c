"""-m gpu: every output element of the fp32-softmax attention kernels -- b200vit_attn_pool (NaViT pooling),
b200vit_attention_cls (class-token attention), b200vit_attention_cls_headmix (CaiT's class attention with talking heads)
and b200vit_attention_xca (XCiT) -- within its bound of the fp64 reference of oracle/attention_fp32_bounds.py.

Outputs are views into NaN-filled buffers with extra rows and columns: an element the kernel does not write fails the
check, and the elements outside the view must keep their NaN.  Two numbers per kernel and instance are printed at the
end of the module: the worst |got - ref| / bound, which the half-ulp output term alone brings near 1 wherever ref sits
near a bf16 rounding midpoint, and the worst share of the fp32 part of the bound the kernel used,
(|got - ref| - ulp(ref) / 2) / (bound - ulp(ref) / 2): a lower bound on the kernel's fp32 error before its output
rounding, against what the bound allows for it."""
import math
import random

import pytest
import torch

from oracle import attention_bounds as AB
from oracle import attention_fp32_bounds as FB
from oracle import bounds as Bd
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst |got - ref| / bound and worst share of the bound's fp32 part used, per kernel and instance:")
    for key in sorted(WORST):
        print(f"  {key}: {WORST[key][0]:.3f}  fp32 part {WORST[key][1]:.3f}")


def fp32_use(got, ref, bound):
    """max over the elements of (|got - ref| - ulp(ref) / 2) / (bound - ulp(ref) / 2), at least 0."""
    half = 0.5 * Bd.bf16_ulp(ref.abs())
    r = ((got.double() - ref).abs() - half).clamp_min(0) / (bound - half)
    return r.max().item() if r.numel() else 0.0


def check(got, ref, bound, key, what):
    """Bd.check, and the two worst ratios of `key` recorded for the report."""
    ratio = Bd.check(got, ref, bound, what)
    old = WORST.get(key, (0.0, 0.0))
    WORST[key] = (max(old[0], ratio), max(old[1], fp32_use(got, ref, bound)))


def nan_view(rows, cols):
    """A NaN-filled bf16 buffer of one extra row and 8 extra columns, and its [rows, cols] view."""
    buf = torch.full((rows + 1, cols + 8), float("nan"), device=DEV, dtype=torch.bfloat16)
    return buf, buf[:rows, :cols]


def outside_untouched(buf, rows, cols):
    return bool(torch.isnan(buf[rows:].float()).all() and torch.isnan(buf[:, cols:].float()).all())


# ------------------------------------------------------------------------------------------------ attn_pool (NaViT)
def rms_rows(x, H, dh, g):
    """Per-head RMS normalisation with a gain near 1, as NaViT's k before pooling."""
    T = x.shape[0]
    y = x.float().view(T, H, dh)
    y = y * torch.rsqrt(y.pow(2).mean(-1, keepdim=True) + 1e-6)
    return (y * (1 + 0.2 * torch.randn(H, dh, generator=g, device=DEV))).reshape(T, H * dh)


def pool_lengths(seed):
    """A NaViT pack: lengths 1 to 1024, below 32 and of every residue mod 4."""
    rng = random.Random(seed)
    return [1, 2, 3, 4, 5, 6, 7, 31, 33, 34, 35, 255, 257, 1024, 1023] + [rng.randrange(1, 1025) for _ in range(6)]


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("H", [1, 3, 16])
def test_attn_pool_within_bound(H, dh):
    g = torch.Generator(device=DEV).manual_seed(H * 1000 + dh)
    lengths = pool_lengths(H + dh)
    T, I = sum(lengths), H * dh
    k = rms_rows(torch.randn(T, I, device=DEV, generator=g), H, dh, g)
    kv = torch.cat([k, torch.randn(T, I, device=DEV, generator=g)], 1).bfloat16().contiguous()
    # an RMS-normalised query at the model's scale dh^-0.5 times a gain: scores of std about 3, peaked rows
    qn = (rms_rows(torch.randn(1, I, device=DEV, generator=g), H, dh, g) * 3 * dh ** -0.5).reshape(-1).contiguous()
    cu, _, _ = _lib.varlen_index(lengths, DEV)
    S = len(lengths)
    # the C ABI writes out as a dense [S, H dh] block: the NaN fill beyond it is the buffer's trailing rows
    buf = torch.full((S + 2, I), float("nan"), device=DEV, dtype=torch.bfloat16)
    out = buf[:S]
    _lib.attn_pool(kv, qn, cu, out, H, dh)
    torch.cuda.synchronize()
    ref, bound = FB.navit_pool_reference(kv, qn, lengths, H, dh)
    check(out, ref, bound, ("attn_pool", f"dh{dh}"), f"attn_pool H{H} dh{dh}")
    assert torch.isnan(buf[S:].float()).all()


# ------------------------------------------------------------------------------------------------ class-token kernels
CLS_N = [0, 1, 3, 4, 5, 31, 32, 33, 255, 256, 257, 576, 4096]


def cls_inputs(B, n, H, dh, first, seed, kind="normal"):
    """qkv_self [B, 3 H dh] and strided context rows (rows per image n + first + 1, 16 unused columns per row)."""
    I = H * dh
    rows, ld = n + first + 1, 2 * I + 16
    x = AB.qkv_inputs(kind, [rows + 1] * B, H, dh, seed=seed, device=DEV).view(B, rows + 1, 3 * I)
    qkv_self = x[:, 0].contiguous()
    ctx = torch.randn(B * rows, ld, device=DEV).bfloat16()
    ctx[:, :2 * I] = x[:, 1:, I:].reshape(B * rows, 2 * I)
    return qkv_self, ctx, rows


@pytest.mark.parametrize("kind", ["normal", "peaked"])
@pytest.mark.parametrize("first", [0, 1])
@pytest.mark.parametrize("dh", [32, 48, 64, 80, 128])
def test_attention_cls_within_bound(dh, first, kind):
    B, H = 3, 3
    I = H * dh
    for n in CLS_N:
        qkv_self, ctx, rows = cls_inputs(B, n, H, dh, first, seed=n * 31 + dh + first, kind=kind)
        scale = 0.9 * dh ** -0.5
        buf, out = nan_view(B, I)
        _lib.attention_cls(qkv_self, ctx[:, :2 * I] if n else None, out, rows, first, n, H, dh, scale)
        torch.cuda.synchronize()
        ref, bound = FB.cls_reference(qkv_self, ctx, rows, first, n, H, dh, scale)
        check(out, ref, bound, ("attention_cls", f"dh{dh}"), f"attention_cls {kind} dh{dh} n{n} first{first}")
        assert outside_untouched(buf, B, I)
        if n == 0:
            assert torch.equal(out, qkv_self[:, 2 * I:])       # one key: the output is its value


@pytest.mark.parametrize("kind", ["normal", "peaked"])
@pytest.mark.parametrize("first", [0, 1])
@pytest.mark.parametrize("H,dh", [(1, 64), (3, 48), (4, 32), (5, 80), (8, 128), (12, 80), (16, 64)])
def test_attention_cls_headmix_within_bound(H, dh, first, kind):
    B, I = 3, H * dh
    g = torch.Generator(device=DEV).manual_seed(H * 100 + dh)
    pre, post = torch.randn(H, H, device=DEV, generator=g), torch.randn(H, H, device=DEV, generator=g)
    for n in CLS_N:
        qkv_self, ctx, rows = cls_inputs(B, n, H, dh, first, seed=n * 17 + H + dh + first, kind=kind)
        scale = dh ** -0.5 if n % 2 else 0.7 * dh ** -0.5
        buf, out = nan_view(B, I)
        _lib.attention_cls_headmix(qkv_self, ctx[:, :2 * I], out, rows, first, n, H, dh, scale, pre, post)
        torch.cuda.synchronize()
        ref, bound = FB.cls_headmix_reference(qkv_self, ctx, rows, first, n, H, dh, scale, pre, post)
        check(out, ref, bound, ("attention_cls_headmix", f"H{H} dh{dh}"),
              f"attention_cls_headmix {kind} H{H} dh{dh} n{n} first{first}")
        assert outside_untouched(buf, B, I)


# ------------------------------------------------------------------------------------------------ xca
def run_xca(qkv, tau, B, N, H, dh, what):
    I = H * dh
    # the C ABI takes out as a dense [B N, H dh] block: the NaN fill beyond it is the buffer's trailing rows
    buf = torch.full((B * N + 2, I), float("nan"), device=DEV, dtype=torch.bfloat16)
    out = buf[:B * N]
    _lib.attention_xca(qkv, tau, out, B, N, H, dh)
    torch.cuda.synchronize()
    ref, bound = FB.xca_reference(qkv, tau, B, N, H, dh)
    check(out, ref, bound, ("attention_xca", f"dh{dh}"), what)
    assert torch.isnan(buf[B * N:].float()).all()


@pytest.mark.parametrize("kind", AB.KINDS)
@pytest.mark.parametrize("dh", [32, 48, 64, 80, 128])
def test_attention_xca_within_bound(dh, kind):
    B, H = 2, 6
    T = FB.xca_tile(dh)
    tau = torch.exp(torch.linspace(-2.0, 3.0, H, device=DEV))
    for N in (1, T - 1, T, T + 1, 196, 197, 784, 3136):
        qkv = AB.qkv_inputs(kind, [N] * B, H, dh, seed=N + dh, device=DEV)
        run_xca(qkv, tau, B, N, H, dh, f"xca {kind} dh{dh} N{N}")


@pytest.mark.parametrize("dh", [48, 128])
def test_attention_xca_zero_and_unequal_columns_within_bound(dh):
    """Zero q and k columns (exact zero scores, a uniform row) and columns whose norms differ by 2^10."""
    B, N, H = 2, 197, 4
    qkv = AB.qkv_inputs("normal", [N] * B, H, dh, seed=dh, device=DEV).float().view(B * N, 3, H, dh)
    qkv[:, 0, 0, 5] = 0
    qkv[:, 1, 2, 7] = 0
    qkv[:, 1, 1, 3] *= 32
    qkv[:, 0, 1, 9] /= 32
    qkv = qkv.reshape(B * N, -1).bfloat16()
    tau = torch.tensor([1.0, math.exp(3.0), 2.0, math.exp(-2.0)], device=DEV)
    run_xca(qkv, tau, B, N, H, dh, f"xca zero / unequal columns dh{dh}")
