"""-m gpu: the variants and attention without output projection through the fused sm_90a path, against
the UNMODIFIED reference's fp32 logits (goldens) with the reference's own bf16 error as the pass criterion."""
import importlib

import pytest
import torch

from conftest import load_golden
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
ALL = ["vit_tiny_noproj", "simplevit_registers", "simplevit_qknorm", "simplevit_patchdrop", "simplevit_flash",
       "simplevit_1d", "simplevit_3d", "simplevit_3d_pf1"]


def dropin_class(kind: str):
    if kind == "vit":
        from vit_pytorch_b200 import ViT
        return ViT
    return importlib.import_module("vit_pytorch_b200." + kind).SimpleViT


@pytest.mark.parametrize("name", ALL)
@pytest.mark.parametrize("mode", ["fold", "exact"])
def test_variant_fused_against_reference_golden(name, mode, monkeypatch):
    monkeypatch.setenv("B200VIT_LN_MODE", mode)
    g = load_golden(name)
    m = dropin_class(g["kind"])(**g["kwargs"]).eval()
    m.load_state_dict(g["state_dict"])
    m = m.to(DEV, torch.bfloat16)
    img = g["input"].to(DEV)
    _lib.reset_launch_count()
    with torch.inference_mode():
        assert m.fused_reason(img) is None, m.fused_reason(img)
        out = m(img)
    assert _lib.launch_count() > 0
    ref = g["logits_fp32"]
    d = (out.float().cpu() - ref).abs()
    floor = (g["logits_ref_bf16"] - ref).abs()
    print(f"{name} [{mode}]: fused max {d.max():.5f} mean {d.mean():.5f}; reference-bf16 max {floor.max():.5f} "
          f"mean {floor.mean():.5f}")
    assert out.shape == ref.shape and torch.isfinite(out.float()).all()
    # no worse than the reference's own bf16 forward on the same inputs (small slack on the max of a tiny sample)
    assert d.mean() <= floor.mean() * 1.05 + 1e-4 and d.max() <= floor.max() * 1.5 + 1e-3


def test_register_tokens_do_not_enter_the_pool():
    """The mean runs over the patch tokens only: changing how many registers exist changes the logits only through
    attention, and the fused result equals the model's own PyTorch graph."""
    from vit_pytorch_b200.simple_vit_with_register_tokens import SimpleViT
    torch.manual_seed(0)
    m = SimpleViT(image_size=64, patch_size=8, num_classes=12, dim=128, depth=2, heads=2, mlp_dim=256,
                  num_register_tokens=3).eval().to(DEV, torch.bfloat16)
    img = torch.randn(5, 3, 64, 64, device=DEV).bfloat16()
    with torch.inference_mode():
        fused = m(img)
        eager = m.float().forward_eager(img.float())
    assert (fused.float() - eager).abs().max() < 2e-2


def test_flash_variant_accepts_other_resolutions():
    from vit_pytorch_b200.simple_flash_attn_vit import SimpleViT
    torch.manual_seed(1)
    m = SimpleViT(image_size=64, patch_size=8, num_classes=6, dim=128, depth=1, heads=2, mlp_dim=256).eval()
    m = m.to(DEV, torch.bfloat16)
    for hw in ((64, 64), (32, 48), (8, 8)):
        img = torch.randn(2, 3, *hw, device=DEV).bfloat16()
        with torch.inference_mode():
            assert m.fused_reason(img) is None
            fused = m(img)
            eager = m.forward_eager(img)
        assert (fused.float() - eager.float()).abs().max() < 3e-2


@pytest.mark.parametrize("name", ["navit_nested_tiny", "navit_nested_noqknorm"])
@pytest.mark.parametrize("mode", ["fold", "exact"])
def test_navit_nested_fused_against_reference_golden(name, mode, monkeypatch):
    """Nested-tensor NaViT front-end (reference na_vit_nested_tensor.py) on the padding-free fused path: per-head
    LayerNorm of q / k as the QKV GEMM's epilogue (EPI_HEADLN), varlen attention with scale dim_head ** -0.5."""
    monkeypatch.setenv("B200VIT_LN_MODE", mode)
    from vit_pytorch_b200.na_vit_nested_tensor import NaViT
    g = load_golden(name)
    m = NaViT(**g["kwargs"]).eval()
    m.load_state_dict(g["state_dict"])
    m = m.to(DEV, torch.bfloat16)
    imgs = [im.to(DEV) for im in g["images"]]
    _lib.reset_launch_count()
    with torch.inference_mode():
        assert m.fused_reason(imgs) is None, m.fused_reason(imgs)
        out = m(imgs)
    assert _lib.launch_count() > 0
    ref = g["logits_fp32"]
    d = (out.float().cpu() - ref).abs()
    floor = (g["logits_ref_bf16"] - ref).abs()
    print(f"{name} [{mode}]: fused max {d.max():.5f} mean {d.mean():.5f}; reference-bf16 max {floor.max():.5f} "
          f"mean {floor.mean():.5f}")
    assert out.shape == ref.shape and torch.isfinite(out.float()).all()
    assert d.mean() <= floor.mean() * 1.05 + 1e-4 and d.max() <= floor.max() * 1.5 + 1e-3


@pytest.mark.parametrize("M", [300, 2048])
def test_gemm_head_layernorm_epilogue(M):
    """EPI_HEADLN: (v - mean) * rsqrt(var + eps) * gamma per 64-wide head, in the GEMM epilogue (M >= 1024) and in the
    stand-alone kernel (small M) -- against torch on the bf16-rounded projection."""
    torch.manual_seed(M)
    K, H = 128, 3
    N = 3 * H * 64
    a = torch.randn(M, K, device=DEV).bfloat16()
    w = (torch.randn(N, K, device=DEV) / K ** 0.5).bfloat16()
    gamma = (1 + 0.2 * torch.randn(2 * H * 64, device=DEV)).contiguous()
    out = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    _lib.gemm_headnorm(a, w, out_bf16=out, head_gamma=gamma, norm_heads=2 * H, head_layernorm_eps=1e-5)
    y = (a.float() @ w.float().t()).bfloat16().float()
    ref = y.clone()
    yn = torch.nn.functional.layer_norm(y[:, : 2 * H * 64].reshape(M, 2 * H, 64), (64,), None, None, 1e-5)
    ref[:, : 2 * H * 64] = (yn * gamma.view(2 * H, 64)).reshape(M, -1)
    assert torch.allclose(out.float(), ref, rtol=2e-2, atol=2e-2)
    # the v third is the plain projection (accumulation order differs from torch's: compare within a bf16 ulp)
    assert torch.allclose(out[:, 2 * H * 64:].float(), y[:, 2 * H * 64:], rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize("pf", [1, 2, 4])
def test_video_front_end_matches_its_own_pytorch_graph(pf):
    """simple_vit_3d on a larger clip: the (pf p1 p2 c) boxes reach the 2-D patch kernels as a (B, C, F*H, W) image
    (frame_patch_size 1 with 16 x 16 boxes: the TMA patch embedding); compared with the module's own fp32 graph."""
    from vit_pytorch_b200.simple_vit_3d import SimpleViT
    torch.manual_seed(2)
    m = SimpleViT(image_size=(64, 48), image_patch_size=16, frames=8, frame_patch_size=pf, num_classes=9, dim=192,
                  depth=2, heads=3, mlp_dim=384).eval().to(DEV, torch.bfloat16)
    video = torch.randn(3, 3, 8, 64, 48, device=DEV).bfloat16()
    _lib.reset_launch_count()
    with torch.inference_mode():
        assert m.fused_reason(video) is None, m.fused_reason(video)
        fused = m(video)
        assert _lib.launch_count() > 0
        eager = m.float().forward_eager(video.float())
    assert fused.shape == (3, 9)
    assert (fused.float() - eager).abs().max() < 2e-2


def test_series_front_end_matches_its_own_pytorch_graph():
    from vit_pytorch_b200.simple_vit_1d import SimpleViT
    torch.manual_seed(3)
    m = SimpleViT(seq_len=4096, patch_size=8, num_classes=5, dim=128, depth=2, heads=2, mlp_dim=256, channels=6)
    m = m.eval().to(DEV, torch.bfloat16)
    series = torch.randn(2, 6, 4096, device=DEV).bfloat16()
    with torch.inference_mode():
        assert m.fused_reason(series) is None, m.fused_reason(series)
        fused = m(series)
        eager = m.float().forward_eager(series.float())
    assert (fused.float() - eager).abs().max() < 2e-2
