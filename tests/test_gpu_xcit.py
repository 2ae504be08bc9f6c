"""-m gpu: the cross-covariance attention kernel (b200vit_attention_xca), the local patch interaction kernel
(b200vit_local_patch_interaction), class attention at dim_head 48 and the fused XCiT on the H100.  The attention kernels
are checked against the fp64 references and per-element bounds of oracle/attention_fp32_bounds.py, the patch
interaction against those of oracle/lpi_bounds.py; the model's CUDA-graph replay and fallback rules
(its reference parity is in test_gpu_family_parity.py)."""
import sys

import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import attention_fp32_bounds as FB
from oracle import bounds as Bd
from oracle.lpi_bounds import lpi_reference
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.xcit import XCATransformer, XCiT

sys.path.insert(0, GOLDEN_DIR)
from xcit_spec import FAMILY, XCIT_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def stats(got, ref, rtol=1e-2, atol=1e-3):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), (d <= atol + rtol * ref.float().cpu().abs()).float().mean().item()


# ------------------------------------------------------------------------------------------------ attention_xca
@pytest.mark.parametrize("N", [1, 63, 64, 65, 196, 197, 784, 3136])
@pytest.mark.parametrize("dh", [32, 48, 64, 80, 128])
@pytest.mark.parametrize("H", [1, 3, 8, 16])
def test_attention_xca_against_fp32(H, dh, N):
    torch.manual_seed(H * 1000 + dh + N)
    B = 2
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV).bfloat16()
    tau = torch.exp(torch.randn(H, device=DEV))
    out = torch.full((B * N, H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attention_xca(qkv, tau, out, B, N, H, dh)
    ref, bound = FB.xca_reference(qkv, tau, B, N, H, dh)
    Bd.check(out, ref, bound, f"xca H{H} dh{dh} N{N}")


def test_attention_xca_zero_columns_and_peaky_tau():
    """An all-zero q or k column gives zero scores (F.normalize's eps), never NaN; a large tau gives a near one-hot
    softmax over the channels."""
    B, N, H, dh = 2, 197, 4, 48
    torch.manual_seed(0)
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV).bfloat16()
    qkv[:, 5] = 0                                          # q column 5 of head 0
    qkv[:, H * dh + 2 * dh + 7] = 0                        # k column 7 of head 2
    tau = torch.tensor([1.0, 30.0, 2.0, 0.5], device=DEV)
    out = torch.full((B * N, H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
    _lib.attention_xca(qkv, tau, out, B, N, H, dh)
    ref, bound = FB.xca_reference(qkv, tau, B, N, H, dh)
    Bd.check(out, ref, bound, "xca zero columns")


def test_attention_xca_repeat_calls_are_bit_identical_and_stay_in_place():
    B, N, H, dh = 3, 784, 8, 48
    torch.manual_seed(1)
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV).bfloat16()
    tau = torch.exp(torch.randn(H, device=DEV))
    # `out` is a view of the leading columns of a wider, poisoned buffer: nothing beyond it may be written
    big = torch.full((B * N + 4, H * dh + 64), float("nan"), device=DEV, dtype=torch.bfloat16)
    out = big[:B * N].view(-1)[:B * N * H * dh].view(B * N, H * dh)
    _lib.attention_xca(qkv, tau, out, B, N, H, dh)
    first = out.clone()
    for _ in range(3):
        _lib.attention_xca(qkv, tau, out, B, N, H, dh)
        assert torch.equal(out, first)
    assert torch.isnan(big.view(-1)[B * N * H * dh:].float()).all()


def test_attention_xca_keeps_each_image_to_itself():
    B, N, H, dh = 3, 65, 4, 64
    torch.manual_seed(2)
    qkv = torch.randn(B * N, 3 * H * dh, device=DEV).bfloat16()
    tau = torch.ones(H, device=DEV)
    out = torch.empty(B * N, H * dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention_xca(qkv, tau, out, B, N, H, dh)
    clean = out.clone()
    qkv[N:2 * N] = float("nan")
    _lib.attention_xca(qkv, tau, out, B, N, H, dh)
    assert torch.equal(out[:N], clean[:N]) and torch.equal(out[2 * N:], clean[2 * N:])


# ------------------------------------------------------------------------------------------------ local patch interaction
@pytest.mark.parametrize("D", [64, 384, 1024])
@pytest.mark.parametrize("k", [1, 3, 5, 7])
@pytest.mark.parametrize("grid", [(1, 1), (1, 7), (2, 2), (6, 8), (14, 14), (56, 56)])
def test_local_patch_interaction_against_fp32(grid, k, D):
    gh, gw = grid
    B = 2
    M = B * gh * gw
    torch.manual_seed(gh * 100 + gw + k + D)
    x = torch.randn(M, D, device=DEV)
    ln = (1 + 0.2 * torch.randn(D, device=DEV), 0.3 * torch.randn(D, device=DEV), 1e-5)
    w1, w2 = 0.3 * torch.randn(k * k, D, device=DEV), 0.3 * torch.randn(k * k, D, device=DEV)
    b1, b2 = 0.2 * torch.randn(D, device=DEV), 0.2 * torch.randn(D, device=DEV)
    x0 = x.clone()
    y = torch.full_like(x, float("nan"))
    yb = torch.empty(M, D, device=DEV, dtype=torch.bfloat16)
    ys = torch.empty(M, 2, device=DEV)
    scratch = torch.empty(M, 2, device=DEV)
    _lib.local_patch_interaction(x, y, scratch, ln, w1, b1, w2, b2, B, gh, gw, k, y_bf16=yb, y_stats=ys)
    assert torch.equal(x, x0)                              # the input stream is left as it was
    Bd.check(y, *lpi_reference(x, ln, w1, b1, w2, b2, B, gh, gw, k), f"lpi {gh}x{gw} k{k} D{D}")
    # the bf16 copy and the statistics are exactly what rowstats_cast writes for y
    rb, rs = torch.empty_like(yb), torch.empty_like(ys)
    _lib.rowstats_cast(y, rb, rs)
    assert torch.equal(yb, rb) and torch.equal(ys, rs)
    # without the copy: the same y
    y2 = torch.empty_like(x)
    _lib.local_patch_interaction(x, y2, scratch, ln, w1, b1, w2, b2, B, gh, gw, k)
    assert torch.equal(y2, y)


# ------------------------------------------------------------------------------------------------ attention_cls, dh 48
def test_attention_cls_dim_head_48():
    torch.manual_seed(4)
    B, H, dh, rows, n = 3, 6, 48, 197, 196
    I = H * dh
    qkv = torch.randn(B, 3 * I, device=DEV).bfloat16()
    ctx = (2 * torch.randn(B * rows, 2 * I, device=DEV)).bfloat16()
    out = torch.full((B, I), 5.0, device=DEV).bfloat16()
    scale = dh ** -0.5
    _lib.attention_cls(qkv, ctx, out, rows, 1, n, H, dh, scale)
    ref, bound = FB.cls_reference(qkv, ctx, rows, 1, n, H, dh, scale)
    Bd.check(out, ref, bound, "attention_cls dh48")


# ------------------------------------------------------------------------------------------------ model
def test_cuda_graph_replay_is_bit_identical():
    from vit_pytorch_b200.graph import GraphedForward
    spec = XCIT_CASES["dh48_n196"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    a = FAMILY.input(spec).to(DEV)
    b = torch.randn_like(a.float()).bfloat16()
    with torch.inference_mode():
        ya, yb = m(a).clone(), m(b).clone()
        g = GraphedForward(m, a)
        assert torch.equal(g(b), yb)
        assert torch.equal(g(a), ya)


def test_cuda_graph_refused_with_layer_dropout():
    from vit_pytorch_b200.graph import GraphedForward
    spec = XCIT_CASES["dh32"]
    m = FAMILY.build({**spec, "layer_dropout": 0.1}).to(DEV, torch.bfloat16)
    with pytest.raises(RuntimeError, match="layer_dropout"):
        GraphedForward(m, FAMILY.input(spec).to(DEV))


def test_direct_xcit_transformer_call():
    torch.manual_seed(3)
    t = XCATransformer(96, 2, 2, 48, 192, local_patch_kernel_size=5).eval()
    with torch.no_grad():
        for p in list(t.parameters()) + [b for b in t.buffers() if b.is_floating_point()]:
            p.copy_(p.bfloat16().float())
    ref = XCATransformer(96, 2, 2, 48, 192, local_patch_kernel_size=5).eval()
    ref.load_state_dict(t.state_dict())
    t = t.to(DEV, torch.bfloat16)
    x = torch.randn(3, 6, 9, 96, device=DEV).bfloat16()
    with torch.inference_mode():
        assert t.fused_reason(x) is None
        _lib.reset_launch_count()
        out = t(x)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = ref(x.float().cpu())
    assert out.shape == (3, 6, 9, 96)
    scale = want.abs().max().item()
    mx, frac = stats(out, want, rtol=1e-2, atol=1e-2 * scale)
    assert mx < 2e-2 * scale and frac > 0.99, (mx, frac, scale)


def test_running_var_change_reaches_the_fused_output():
    """BatchNorm's running statistics are buffers, not parameters: an in-place update must still rebuild the folded
    conv1 weights.  After it the fused output equals, bit for bit, that of a fresh model loaded with the same state."""
    spec = XCIT_CASES["dh32"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        before = m(x).clone()
    with torch.no_grad():
        for _, lpi, _ in m.xcit_transformer.layers:
            lpi.fn.net[3].running_var.mul_(0.01)          # BatchNorm now scales conv1 by 10
    fresh = FAMILY.build(spec).to(DEV, torch.bfloat16)
    fresh.load_state_dict(m.state_dict())
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        after = m(x)
        assert torch.equal(after, fresh(x))
    assert not torch.equal(after, before)


def test_train_mode_forward_reaches_the_fused_output():
    """A train-mode forward (BatchNorm recalibration, or training with the backbone frozen) updates the running
    statistics in place without bumping their version counters.  The next eval forward runs fused and equals, bit for
    bit, a fresh model loaded with the same state."""
    spec = XCIT_CASES["dh32"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        before = m(x).clone()
    m.train()
    with torch.no_grad():
        m(3 * torch.randn(8, *x.shape[1:], device=DEV).bfloat16())
    m.eval()
    fresh = FAMILY.build(spec).to(DEV, torch.bfloat16)
    fresh.load_state_dict(m.state_dict())
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        after = m(x)
        assert torch.equal(after, fresh(x))
    assert not torch.equal(after, before)


FALLBACK_KW = dict(image_size=32, patch_size=4, num_classes=3, dim=64, depth=1, cls_depth=1, mlp_dim=64)


def _model(**kw):
    return XCiT(**{**FALLBACK_KW, "heads": 4, "dim_head": 32, **kw}).eval().to(DEV, torch.bfloat16)


def test_fallback_unsupported_head_width():
    m, x = _model(heads=2, dim_head=96), torch.randn(2, 3, 32, 32, device=DEV).bfloat16()
    with torch.inference_mode():
        assert "dim_head=96" in m.fused_reason(x)
        assert m(x).shape == (2, 3)                        # eager, like the reference


def test_fallback_kernel_size():
    m, x = _model(local_patch_kernel_size=9), torch.randn(2, 3, 32, 32, device=DEV).bfloat16()
    with torch.inference_mode():
        assert "local_patch_kernel_size=9" in m.fused_reason(x)
        assert m(x).shape == (2, 3)


def test_fallback_batchnorm_in_training_mode():
    """With the default dropout = 0 a .train() model has no dropout to refuse it: BatchNorm's batch statistics do."""
    m, x = _model(), torch.randn(2, 3, 32, 32, device=DEV).bfloat16()
    m.train()
    with torch.no_grad():
        assert "BatchNorm2d" in m.fused_reason(x)
        m(x)
    m.eval()
    m.xcit_transformer.layers[0][1].fn.net[3].train()
    with torch.inference_mode():
        assert "BatchNorm2d" in m.fused_reason(x)


def test_fallback_positional_table_and_divisibility():
    m = _model()
    with torch.inference_mode():
        assert "positional table" in m.fused_reason(torch.randn(2, 3, 36, 36, device=DEV).bfloat16())
        assert "divisible" in m.fused_reason(torch.randn(2, 3, 30, 30, device=DEV).bfloat16())
        assert "channel count" in m.fused_reason(torch.randn(2, 1, 32, 32, device=DEV).bfloat16())
        assert m.fused_reason(torch.randn(2, 3, 32, 32, device=DEV)) is not None        # fp32 input


def test_fallback_hooks_and_autograd():
    m, x = _model(), torch.randn(2, 3, 32, 32, device=DEV).bfloat16()
    assert "autograd" in m.fused_reason(x)
    h = m.xcit_transformer.layers[0][0].fn.to_qkv.register_forward_hook(lambda *a: None)
    with torch.inference_mode():
        assert "hooks" in m.fused_reason(x)
    h.remove()
    with torch.inference_mode():
        assert m.fused_reason(x) is None
