"""-m gpu: the strided short-sequence attention kernel, the grouped token assembly and the fused ViViT on the H100.
Every element of the attention kernel's output is checked against the fp64 reference and bound of
oracle/attention_bounds.py, the token assembly against a torch expression; the model's fallback rules, direct
transformer calls and LayerNorm modes (its reference parity is in test_gpu_family_parity.py)."""
import sys

import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import bounds as Bd
from oracle.attention_bounds import axial_reference
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.vivit import FactorizedTransformer, Transformer, ViViT

sys.path.insert(0, GOLDEN_DIR)
from vivit_spec import FAMILY, VIVIT_CASES, vivit_mask  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
RTOL, ATOL = 1e-2, 1e-3


def stats(got, ref):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), (d <= ATOL + RTOL * ref.float().cpu().abs()).float().mean().item()


# ------------------------------------------------------------------------------------------------------ attention_axial
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("L", [1, 2, 5, 8, 17, 33, 64])
@pytest.mark.parametrize("G", [1, 3, 50, 197])
def test_attention_axial_against_fp32(dh, L, G):
    torch.manual_seed(dh * 1000 + L * 10 + G)
    B, H = 3, 2
    T = B * L * G
    qkv = torch.randn(T, 3 * H * dh, device=DEV).bfloat16()
    scale = dh ** -0.5
    partial = torch.rand(B, L, device=DEV) > 0.4
    partial[:, 0] = True                                   # every sequence keeps a key
    full = partial.clone()
    full[1] = False                                        # batch element 1: every key masked
    for name, km in (("none", None), ("partial", partial), ("full", full)):
        km8 = None if km is None else km.to(torch.uint8).contiguous()
        for zero in (True, False):
            if km is None and not zero:
                continue
            # out has rows beyond the addressed set: they must keep their NaN fill
            buf = torch.full((T + 5, H * dh), float("nan"), device=DEV, dtype=torch.bfloat16)
            _lib.attention_axial(qkv, buf[:T], km8, B, L, G, H, dh, scale, zero)
            ref, bound = axial_reference(qkv, km, B, L, G, H, dh, scale, zero)
            Bd.check(buf[:T], ref, bound, f"axial {name} zero={zero}")
            assert torch.isnan(buf[T:].float()).all()
            again = torch.empty(T, H * dh, device=DEV, dtype=torch.bfloat16)
            _lib.attention_axial(qkv, again, km8, B, L, G, H, dh, scale, zero)
            assert torch.equal(again, buf[:T])             # deterministic


# ------------------------------------------------------------------------------------------------------ token assembly
@pytest.mark.parametrize("ncls", [0, 1])
@pytest.mark.parametrize("n,n_max", [(6, 6), (4, 9)])
def test_embed_tokens_grouped(ncls, n, n_max):
    torch.manual_seed(ncls * 10 + n)
    B, F, Fmax, D = 3, 4, 5, 96
    y = torch.randn(B * F * n, D, device=DEV)
    g, be = 1 + 0.1 * torch.randn(D, device=DEV), 0.1 * torch.randn(D, device=DEV)
    pos = torch.randn(Fmax * n_max, D, device=DEV)
    cls = torch.randn(1, D, device=DEV) if ncls else None
    N = n + ncls
    x = torch.empty(B * F * N, D, device=DEV)
    xb = torch.empty(B * F * N, D, device=DEV, dtype=torch.bfloat16)
    st = torch.empty(B * F * N, 2, device=DEV)
    _lib.embed_tokens_grouped(y, g, be, cls, pos, x, B * F, n, ncls, pos_period=F, pos_stride=n_max, cls_pos=False,
                              xb=xb, stats=st)
    tok = torch.nn.functional.layer_norm(y.view(B, F, n, D), (D,), g, be, eps=1e-5)
    tok = tok + pos.view(Fmax, n_max, D)[None, :F, :n]                 # pos_embedding[:, :frames, :seq]
    if ncls:
        tok = torch.cat((cls.view(1, 1, 1, D).expand(B, F, 1, D), tok), dim=2)
    want = tok.reshape(-1, D)
    torch.testing.assert_close(x, want, rtol=1e-5, atol=1e-5)
    assert torch.equal(xb, x.bfloat16())
    torch.testing.assert_close(st[:, 0], xb.float().sum(1), rtol=1e-4, atol=1e-3)


# ------------------------------------------------------------------------------------------------------ model
def test_fallback_reasons():
    kw = dict(image_size=16, image_patch_size=8, num_classes=3, dim=64, spatial_depth=1, temporal_depth=1, heads=2,
              dim_head=32, mlp_dim=64)
    long = ViViT(frames=130, frame_patch_size=2, **kw).eval().to(DEV, torch.bfloat16)      # 65 frame patches
    x = torch.randn(1, 3, 130, 16, 16, device=DEV).bfloat16()
    mask = torch.ones(1, 130, dtype=torch.bool, device=DEV)
    with torch.inference_mode():
        assert long.fused_reason(x) is None
        assert "masked temporal sequences of 66 tokens" in long.fused_reason(x, mask)
        out = long(x, mask)                                 # eager, like the reference
    assert out.shape == (1, 3)
    fsa = ViViT(frames=130, frame_patch_size=2, variant="factorized_self_attention", **kw).eval().to(DEV,
                                                                                                    torch.bfloat16)
    with torch.inference_mode():
        assert "65 frame patches" in fsa.fused_reason(x)
    m = ViViT(frames=8, frame_patch_size=2, dropout=0.1, use_flash_attn=False, **kw).to(DEV, torch.bfloat16)
    x = torch.randn(2, 3, 8, 16, 16, device=DEV).bfloat16()
    with torch.inference_mode():
        assert "mask of shape" in m.eval().fused_reason(x, torch.ones(2, 4, dtype=torch.bool, device=DEV))
        assert m.train().fused_reason(x) == "dropout is active"
        m.eval()
        assert m.fused_reason(x) is None
        h = m.spatial_transformer.layers[0][0].attend.register_forward_hook(lambda *a: None)
        assert "hooks" in m.fused_reason(x)
        h.remove()
        assert "different devices" in m.fused_reason(x, torch.ones(2, 8, dtype=torch.bool))
    sdpa_drop = ViViT(frames=8, frame_patch_size=2, dropout=0.1, **kw).eval().to(DEV, torch.bfloat16)
    with torch.inference_mode():
        assert "dropout" in sdpa_drop.fused_reason(x)


def _pair(cls, *args, **kwargs):
    torch.manual_seed(3)
    m = cls(*args, **kwargs).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(p.bfloat16().float())
    ref = cls(*args, **kwargs).eval()
    ref.load_state_dict(m.state_dict())
    return m.to(DEV, torch.bfloat16), ref.to(DEV)


@pytest.mark.parametrize("flash", [True, False])
def test_direct_transformer_call_with_mask(flash):
    m, ref = _pair(Transformer, 128, 2, 2, 64, 256, use_flash_attn=flash)
    torch.manual_seed(4)
    x = torch.randn(5, 9, 128, device=DEV).bfloat16()
    mask = torch.rand(5, 9, device=DEV) > 0.3
    mask[:, 0] = True
    with torch.inference_mode():
        assert m.fused_reason(x, mask) is None
        _lib.reset_launch_count()
        out = m(x, mask)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = ref(x.float(), mask)
    mx, frac = stats(out, want)
    assert mx < 6e-2 and frac > 0.85, (mx, frac)


@pytest.mark.parametrize("masked", [False, True])
def test_direct_factorized_transformer_call(masked):
    m, ref = _pair(FactorizedTransformer, 128, 2, 2, 64, 256)
    torch.manual_seed(5)
    x = torch.randn(2, 6, 17, 128, device=DEV).bfloat16()
    mask = None
    if masked:
        mask = torch.rand(2, 6, device=DEV) > 0.3
        mask[:, 0] = True
    with torch.inference_mode():
        assert m.fused_reason(x, mask) is None
        _lib.reset_launch_count()
        out = m(x, mask)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = ref(x.float(), mask)
    assert out.shape == x.shape
    mx, frac = stats(out, want)
    assert mx < 6e-2 and frac > 0.85, (mx, frac)


def test_exact_layernorm_mode_matches_fold(monkeypatch):
    spec = VIVIT_CASES["fsa_cls_softmax"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    mask = vivit_mask(spec, "partial").to(DEV)
    with torch.inference_mode():
        fold = m(x, mask).float()
        monkeypatch.setenv("B200VIT_LN_MODE", "exact")
        exact = m(x, mask).float()
    assert (fold - exact).abs().max().item() < 2e-2
