"""-m gpu: the overlapping-patch unfold kernel (b200vit_unfold_patches), the pooling kernel (b200vit_pit_pool) and the fused
PiT on the H100.  The unfold is checked bit for bit against F.unfold; the pool against an fp64 conv2d with a
per-element bound; the model's CUDA-graph replay, weight updates and fallback rules (its reference parity is in
test_gpu_family_parity.py)."""
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.pit import PiT, Transformer

sys.path.insert(0, GOLDEN_DIR)
from pit_spec import FAMILY, PIT_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
U32 = 2.0 ** -24


def stats(got, ref, rtol=1e-2, atol=1e-3):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), (d <= atol + rtol * ref.float().cpu().abs()).float().mean().item()


# ------------------------------------------------------------------------------------------------ unfold_patches
def _unfold(img, p, s, ldo, extra=4096):
    """unfold_patches into the head of a NaN-poisoned flat buffer `extra` elements longer than the output."""
    B, C, H, W = img.shape
    rows = B * ((H - p) // s + 1) * ((W - p) // s + 1)
    big = torch.full((rows * ldo + extra,), float("nan"), device=DEV, dtype=torch.bfloat16)
    out = big[:rows * ldo].view(rows, ldo)
    _lib.unfold_patches(img, out, p, s)
    return big, out


@pytest.mark.parametrize("p", [2, 3, 7, 8, 14, 16])
@pytest.mark.parametrize("C", [1, 3, 4])
@pytest.mark.parametrize("hw", [(32, 32), (30, 45), (17, 64)])
def test_unfold_patches_is_bit_exact(hw, C, p):
    H, W = hw
    s = p // 2
    B = 4 if p >= 7 else 2
    torch.manual_seed(p * 100 + C * 10 + H)
    img = torch.randn(B, C, H, W, device=DEV).bfloat16()
    K = C * p * p
    ldo = (K + 63) // 64 * 64
    big, out = _unfold(img, p, s, ldo)
    want = F.unfold(img.float(), p, stride=s).transpose(1, 2).reshape(-1, K).bfloat16()
    assert torch.equal(out[:, :K], want)
    assert (out[:, K:] == 0).all()                                        # the K padding is zeros, not NaN
    assert not torch.isnan(out.float()).any()
    assert torch.isnan(big[out.numel():].float()).all()                  # nothing past the output is written


@pytest.mark.parametrize("p,s", [(14, 7), (16, 8), (4, 3), (5, 1)])
def test_unfold_patches_any_stride_and_repeat_calls(p, s):
    torch.manual_seed(p + s)
    img = torch.randn(3, 3, 224 if p >= 14 else 37, 224 if p >= 14 else 29, device=DEV).bfloat16()
    K = 3 * p * p
    ldo = (K + 7) // 8 * 8
    _, out = _unfold(img, p, s, ldo)
    want = F.unfold(img.float(), p, stride=s).transpose(1, 2).reshape(-1, K).bfloat16()
    assert torch.equal(out[:, :K], want)
    first = out.clone()
    _lib.unfold_patches(img, out, p, s)
    assert torch.equal(out, first)


# ------------------------------------------------------------------------------------------------ pit_pool
def pool_reference(x, B, h, w, w9, b9):
    """fp64 (ref, bound): the depthwise stride-2 convolution with channel multiplier 2 by conv2d, and per element the
    fp32 error of 9 accumulated taps and the bias plus the bf16 rounding of the result (2^-8 |v|)."""
    D = x.shape[1]
    grid = x.double().view(B, 1 + h * w, D)[:, 1:].reshape(B, h, w, D).permute(0, 3, 1, 2)
    wt = w9.double().t().reshape(2 * D, 1, 3, 3)
    ref = F.conv2d(grid, wt, b9.double(), stride=2, padding=1, groups=D)
    mag = F.conv2d(grid.abs(), wt.abs(), b9.double().abs(), stride=2, padding=1, groups=D)
    ref, mag = (t.flatten(2).transpose(1, 2) for t in (ref, mag))           # b, t, 2D
    bound = 2.0 ** -8 * ref.abs() + 12 * U32 * mag + 1e-30
    return ref, bound


def _pool(x, B, h, w, w9, b9, pad_cols=8, pad_rows=2):
    """pit_pool into views of NaN-poisoned buffers wider and longer than the outputs."""
    D = x.shape[1]
    n2 = ((h + 1) // 2) * ((w + 1) // 2)
    abig = torch.full((B * (1 + n2) + pad_rows, 2 * D + pad_cols), float("nan"), device=DEV, dtype=torch.bfloat16)
    cbig = torch.full((B + pad_rows, D + pad_cols), float("nan"), device=DEV, dtype=torch.bfloat16)
    a, cls = abig[:B * (1 + n2), :2 * D], cbig[:B, :D]
    _lib.pit_pool(x, B, h, w, w9, b9, a, cls)
    return abig, cbig, a, cls


def _pool_inputs(B, h, w, D, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B * (1 + h * w), D, device=DEV, generator=g)
    w9 = 0.4 * torch.randn(9, 2 * D, device=DEV, generator=g)
    b9 = 0.2 * torch.randn(2 * D, device=DEV, generator=g)
    return x, w9, b9


@pytest.mark.parametrize("D", [8, 64, 256, 1024])
@pytest.mark.parametrize("grid", [(1, 1), (2, 2), (3, 5), (7, 7), (16, 16), (31, 31)])
def test_pit_pool_against_fp64(grid, D):
    h, w = grid
    B = 4 if D <= 256 else 2
    x, w9, b9 = _pool_inputs(B, h, w, D, h * 1000 + w * 10 + D)
    abig, cbig, a, cls = _pool(x, B, h, w, w9, b9)
    n2 = ((h + 1) // 2) * ((w + 1) // 2)
    av = a.view(B, 1 + n2, 2 * D)
    ref, bound = pool_reference(x, B, h, w, w9, b9)
    err = (av[:, 1:].double() - ref).abs()
    assert (err <= bound).all(), (err / bound).max().item()
    assert (av[:, 0] == 0).all()                                          # the cls slots are zero filled
    assert torch.equal(cls, x.view(B, 1 + h * w, D)[:, 0].bfloat16())      # bit copies of the cls rows
    assert torch.isnan(abig[:, 2 * D:].float()).all() and torch.isnan(abig[B * (1 + n2):].float()).all()
    assert torch.isnan(cbig[:, D:].float()).all() and torch.isnan(cbig[B:].float()).all()


def test_pit_pool_keeps_each_image_to_itself_and_repeats_bits():
    B, h, w, D = 3, 7, 7, 64
    x, w9, b9 = _pool_inputs(B, h, w, D, 5)
    _, _, a, cls = _pool(x, B, h, w, w9, b9)
    a0, c0 = a.clone(), cls.clone()
    for _ in range(2):
        _lib.pit_pool(x, B, h, w, w9, b9, a, cls)
        assert torch.equal(a, a0) and torch.equal(cls, c0)
    rows = 1 + h * w
    x[rows:2 * rows] = float("nan")                                       # image 1, its cls row included
    _lib.pit_pool(x, B, h, w, w9, b9, a, cls)
    n2 = 1 + 16
    assert torch.equal(a[:n2], a0[:n2]) and torch.equal(a[2 * n2:], a0[2 * n2:])
    assert torch.equal(cls[0], c0[0]) and torch.equal(cls[2], c0[2])


# ------------------------------------------------------------------------------------------------ model
def test_readme_config_takes_the_fused_path():
    m = PiT(image_size=224, patch_size=14, dim=256, num_classes=1000, depth=(3, 3, 3), heads=16, mlp_dim=2048,
            dropout=0.1, emb_dropout=0.1).eval().to(DEV, torch.bfloat16)
    x = torch.randn(2, 3, 224, 224, device=DEV).bfloat16()
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        assert m(x).shape == (2, 1000)


def test_direct_transformer_call_runs_fused():
    torch.manual_seed(3)
    t = Transformer(64, 2, 2, 32, 128).eval()
    with torch.no_grad():
        for p in t.parameters():
            p.copy_(p.bfloat16().float())
    ref = Transformer(64, 2, 2, 32, 128).eval()
    ref.load_state_dict(t.state_dict())
    t = t.to(DEV, torch.bfloat16)
    x = torch.randn(3, 50, 64, device=DEV).bfloat16()
    with torch.inference_mode():
        assert t.fused_reason(x) is None
        _lib.reset_launch_count()
        out = t(x)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = ref(x.float().cpu())
    scale = want.abs().max().item()
    mx, frac = stats(out, want, rtol=1e-2, atol=1e-2 * scale)
    assert mx < 2e-2 * scale and frac > 0.99, (mx, frac, scale)


def test_cuda_graph_replay_is_bit_identical():
    from vit_pytorch_b200.graph import GraphedForward
    spec = PIT_CASES["heads_tuple"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    a = FAMILY.input(spec).to(DEV)
    b = torch.randn_like(a.float()).bfloat16()
    with torch.inference_mode():
        ya, yb = m(a).clone(), m(b).clone()
        g = GraphedForward(m, a)
        assert torch.equal(g(b), yb)
        assert torch.equal(g(a), ya)


def test_weight_updates_reach_the_fused_output():
    """load_state_dict and an in-place update of a pool weight both rebuild the prepared weights: afterwards the fused
    output equals, bit for bit, that of a fresh model loaded with the same state."""
    spec = PIT_CASES["heads_tuple"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        before = m(x).clone()
    with torch.no_grad():
        m.layers[1].downsample.net[0].weight.mul_(-1.0)
        m.layers[3].cls_ff.bias.add_(0.5)
    fresh = FAMILY.build(spec).to(DEV, torch.bfloat16)
    with torch.inference_mode():
        fresh(x)                                          # prepares fresh's weights from the old state first
    fresh.load_state_dict(m.state_dict())
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        after = m(x)
        assert not torch.equal(after, before)
        assert torch.equal(after, fresh(x))


FALLBACK_KW = dict(image_size=32, patch_size=8, num_classes=3, dim=32, depth=(1, 1), heads=2, mlp_dim=64, dim_head=32)


def test_fallback_rules_on_the_gpu():
    m = PiT(**FALLBACK_KW).eval().to(DEV, torch.bfloat16)
    x = torch.randn(2, 3, 32, 32, device=DEV).bfloat16()
    assert "autograd" in m.fused_reason(x)
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        assert m.fused_reason(x.float()) is not None
        assert "positional table" in m.fused_reason(torch.randn(2, 3, 40, 40, device=DEV).bfloat16())
        h = m.layers[1].register_forward_hook(lambda *a: None)
        assert "hooks" in m.fused_reason(x)
        h.remove()
        s = PiT(**{**FALLBACK_KW, "dim_head": 48}).eval().to(DEV, torch.bfloat16)
        assert "dim_head=48" in s.fused_reason(x)
        assert s(x).shape == (2, 3)                        # eager, like the reference
        bad = torch.randn(2, 3, 12, 24, device=DEV).bfloat16()             # a 2 x 5 grid: 10 tokens
        assert "int(sqrt(n))" in m.fused_reason(bad)
        with pytest.raises(RuntimeError):
            m(bad)
