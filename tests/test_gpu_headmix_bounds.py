"""-m gpu: every output element of the head-mixing attention kernel (b200vit_attention_headmix / _ex) within its bound
of the fp64 reference of oracle/headmix_bounds.py, on every built instance: dh 32 / 48 / 64 / 80 / 128 x head capacity
4 / 8 / 16 x with and without the pre-mix, each with and without the LayerNorm over heads.

Outputs go into NaN-filled buffers longer than the output (the C ABI writes a dense [B N, H dh] block, so the NaN past
it is the buffer's trailing elements): an element the kernel does not write fails the check, and the trailing ones must
keep their NaN.  Two numbers per instance are printed at the end of the module: the worst |got - ref| / bound, which
the half-ulp output term alone brings near 1 wherever ref sits near a bf16 rounding midpoint, and the worst share of
the fp32 part of the bound the kernel used, (|got - ref| - ulp(ref) / 2) / (bound - ulp(ref) / 2)."""
import pytest
import torch

from oracle import bounds as Bd
from oracle import headmix_bounds as HB
from oracle.bounds import C_ACC, U
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORST = {}
HEAD_COUNTS = [(H, dh) for dh in (32, 48, 64, 80, 128) for H in range(1, 17) if H * dh <= 1024]
MODES = {"post": (False, False), "post_ln": (False, True), "pre_post": (True, False), "pre_post_ln": (True, True)}
NS = (1, 15, 16, 17, 63, 64, 65, 129, 197)


def capacity(H, dh):
    """The head capacity of the instance that runs H heads (launch_headmix_hc)."""
    return 4 if H <= 4 else 8 if H <= 8 or dh == 128 else 16


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst |got - ref| / bound and worst share of the bound's fp32 part used, per instance (dh, capacity, pre):")
    for key in sorted(WORST):
        print(f"  {key}: {WORST[key][0]:.3f}  fp32 part {WORST[key][1]:.3f}")


def fp32_use(got, ref, bound):
    """max over the elements of (|got - ref| - ulp(ref) / 2) / (bound - ulp(ref) / 2), at least 0."""
    half = 0.5 * Bd.bf16_ulp(ref.abs())
    r = ((got.double() - ref).abs() - half).clamp_min(0) / (bound - half)
    return r.max().item() if r.numel() else 0.0


def run(qkv, B, N, H, dh, scale, pre, post, ln):
    """The kernel's output in a NaN-filled buffer with 777 trailing elements; checks those keep their NaN and that a
    second call gives identical bits."""
    T, I = B * N, H * dh
    buf = torch.full((T * I + 777,), float("nan"), device=DEV, dtype=torch.bfloat16)
    out = buf[:T * I].view(T, I)
    _lib.attention_headmix(qkv, out, B, N, H, dh, scale, post, ln, pre=pre)
    first = out.clone()
    _lib.attention_headmix(qkv, out, B, N, H, dh, scale, post, ln, pre=pre)
    torch.cuda.synchronize()
    assert torch.isnan(buf[T * I:].float()).all(), "elements past the output were written"
    assert torch.equal(out, first), "repeated calls differ"
    return out


def check(qkv, B, N, H, dh, scale, pre, post, ln, what):
    out = run(qkv, B, N, H, dh, scale, pre, post, ln)
    ref, bound = HB.headmix_reference(qkv, B, N, H, dh, scale, pre, post, ln)
    ratio = Bd.check(out, ref, bound, what)
    key = (dh, capacity(H, dh), pre is not None)
    old = WORST.get(key, (0.0, 0.0))
    WORST[key] = (max(old[0], ratio), max(old[1], fp32_use(out, ref, bound)))


def inputs(kind, B, N, H, dh, mode, seed):
    qkv, pre, post, ln = HB.headmix_inputs(kind, B, N, H, dh, seed=seed, device=DEV)
    use_pre, use_ln = MODES[mode]
    return qkv, (pre if use_pre else None), post, (ln if use_ln else None)


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("H,dh", HEAD_COUNTS)
def test_headmix_within_bound(H, dh, mode):
    B = 3
    for N in NS:
        qkv, pre, post, ln = inputs("normal", B, N, H, dh, mode, seed=H * 1000 + dh * 10 + N)
        check(qkv, B, N, H, dh, dh ** -0.5, pre, post, ln, f"headmix H{H} dh{dh} {mode} N{N}")


@pytest.mark.parametrize("kind", ["peaked", "late_max", "vmean", "near_equal"])
@pytest.mark.parametrize("H,dh", [(3, 48), (8, 64), (16, 64), (5, 128)])
def test_headmix_within_bound_on_input_kinds(H, dh, kind):
    """attention_bounds' distributions, and near-equal heads (post = 1 / H + 1e-3 noise) under the LayerNorm, where the
    variance over heads is tiny and rstd near 1 / sqrt(eps)."""
    B = 2
    for mode in (("post_ln", "pre_post_ln") if kind == "near_equal" else sorted(MODES)):
        for N in (65, 197):
            qkv, pre, post, ln = inputs(kind, B, N, H, dh, mode, seed=N + H + dh)
            check(qkv, B, N, H, dh, dh ** -0.5, pre, post, ln, f"headmix {kind} H{H} dh{dh} {mode} N{N}")


@pytest.mark.parametrize("model,N,mode", [("deepvit", 65, "post_ln"), ("cait", 64, "pre_post")])
def test_headmix_readme_shapes(model, N, mode):
    """DeepViT's re-attention and CaiT's talking heads at the READMEs' 16 heads x 64, randn mixing matrices."""
    B, H, dh = 4, 16, 64
    qkv, pre, post, ln = inputs("normal", B, N, H, dh, mode, seed=N)
    check(qkv, B, N, H, dh, dh ** -0.5, pre, post, ln, f"{model} N{N}")


@pytest.mark.parametrize("H,dh,mode", [(3, 48, "post_ln"), (8, 128, "pre_post"), (16, 64, "pre_post_ln")])
def test_headmix_within_bound_16384(H, dh, mode):
    """The longest sequence the kernel takes, one instance per head capacity."""
    N = 16384
    qkv, pre, post, ln = inputs("normal", 1, N, H, dh, mode, seed=H + dh)
    check(qkv, 1, N, H, dh, dh ** -0.5, pre, post, ln, f"headmix H{H} dh{dh} {mode} N{N}")


@pytest.mark.parametrize("pattern", ["walk", "ramp"])
@pytest.mark.parametrize("dh", [64, 128])
def test_pv_chain_calibration(dh, pattern):
    """The P V term of the bound (16-key steps into one fp32 accumulator) on a chain with an exact answer: one head
    with the LayerNorm over it makes P'' = beta = 1 for every key, so out = sum_j v_j, and v's second half is its first
    half negated in reverse order, so the exact sum is 0 and the output is the accumulation error alone.  walk: v of
    mean 0 (partial sums of order sqrt(N)); ramp: v of mean 1 (partial sums of order N).  The worst |got| / bound is
    printed beside the same error over the GEMM form (C_ACC N + 2) u sum|v|."""
    H = 1
    post = torch.ones(1, 1, device=DEV)
    ln = (torch.ones(1, device=DEV), torch.ones(1, device=DEV), 1e-5)
    for N in (1024, 4096, 16384):
        g = torch.Generator(device=DEV).manual_seed(N + dh)
        half = torch.randn(N // 2, dh, generator=g, device=DEV) * (0.5 if pattern == "ramp" else 1.0)
        if pattern == "ramp":
            half += 1.0
        half = half.bfloat16()
        qkv = torch.randn(N, 3 * dh, generator=g, device=DEV).bfloat16()
        qkv[:, 2 * dh:] = torch.cat([half, -half.flip(0)])
        out = run(qkv, 1, N, H, dh, dh ** -0.5, None, post, ln)
        ref, bound = HB.headmix_reference(qkv, 1, N, H, dh, dh ** -0.5, None, post, ln)
        assert (ref == 0).all()
        Bd.check(out, ref, bound, f"P V chain {pattern} dh{dh} N{N}")
        gemm = (C_ACC * N + 2) * U * qkv[:, 2 * dh:].double().abs().sum(0)
        got = out.double().abs()
        print(f"P V chain {pattern} dh{dh} N{N}: worst |got| / bound {(got / bound).max().item():.3f}, "
              f"/ GEMM form {(got / gemm).max().item():.4f}")
