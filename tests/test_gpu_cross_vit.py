"""-m gpu: the class-token cross-attention kernel and the fused CrossViT on the H100.  The kernel is checked against the
fp64 reference and per-element bound of oracle/attention_fp32_bounds.py; the model at batch one and its fallback rules
(its reference parity is in test_gpu_family_parity.py)."""
import sys

import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import attention_fp32_bounds as FB
from oracle import bounds as Bd
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.cross_vit import CrossViT, Transformer
from vit_pytorch_b200.extractor import Extractor

sys.path.insert(0, GOLDEN_DIR)
from cross_vit_spec import CROSS_VIT_CASES, FAMILY  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
RTOL, ATOL = 1e-2, 1e-3


def within(got, ref, rtol=RTOL, atol=ATOL):
    got, ref = got.float().cpu(), ref.float().cpu()
    return ((got - ref).abs() <= atol + rtol * ref.abs()).float().mean().item()


def stats(got, ref):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), within(got, ref)


def tokens_close(got, want):
    """bf16 tokens of LayerNorm-ed streams (|x| up to a few units): a bf16 step there is up to 1.6e-2."""
    mx = (got.float().cpu() - want.float().cpu()).abs().max().item()
    frac = within(got, want, rtol=2e-2, atol=2e-2)
    return mx < 0.1 and frac > 0.98, (mx, frac)


# ------------------------------------------------------------------------------------------------------ attention_cls
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("n", [0, 1, 16, 255, 1024, 4096])
@pytest.mark.parametrize("H", [1, 3, 8])
@pytest.mark.parametrize("B", [1, 37])
def test_attention_cls_against_fp32(dh, n, H, B):
    torch.manual_seed(dh * 7 + n * 3 + H + B)
    I = H * dh
    qkv = (2 * torch.randn(B, 3 * I, device=DEV)).bfloat16()
    # strided context: one extra row per image (skipped) and 16 extra columns per row (another layer's k | v)
    rows, ld = n + 1, 2 * I + 16
    ctx = (2 * torch.randn(B * rows, ld, device=DEV)).bfloat16()
    out = torch.full((B, I + 8), 5.0, device=DEV).bfloat16()
    scale = 0.9 * dh ** -0.5
    _lib.attention_cls(qkv, ctx[:, :2 * I] if n else None, out[:, :I], rows, 1, n, H, dh, scale)
    ref, bound = FB.cls_reference(qkv, ctx, rows, 1, n, H, dh, scale)
    Bd.check(out[:, :I], ref, bound, f"attention_cls B{B} H{H} n{n} dh{dh}")
    assert (out[:, I:] == 5.0).all()                     # row stride ldo: the padding columns are untouched
    if n == 0:
        assert torch.equal(out[:, :I], qkv[:, 2 * I:])


# ------------------------------------------------------------------------------------------------------ model
def _eager_bf16(m, x, monkeypatch, *args):
    """The module's own PyTorch graph in bf16 (every submodule, the encoders included)."""
    with monkeypatch.context() as mp:
        mp.setenv("B200VIT_DISABLE_FUSED", "1")
        with torch.inference_mode():
            return m(x, *args)


def test_batch_one(monkeypatch):
    spec = CROSS_VIT_CASES["widths_32_64"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)[:1]
    with torch.inference_mode():
        out = m(x)
        batched = m(FAMILY.input(spec).to(DEV))[:1]
    eager = _eager_bf16(m, x, monkeypatch)
    assert out.shape == (1, 7)
    assert stats(out, eager)[0] < 3e-2 and stats(out, batched)[0] < 3e-2


def test_direct_multi_scale_encoder_and_transformer_calls(monkeypatch):
    spec = CROSS_VIT_CASES["widths_32_64"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    mse = m.multi_scale_encoder
    torch.manual_seed(0)
    sm = torch.randn(3, 65, 32, device=DEV).bfloat16()
    lg = torch.randn(3, 17, 64, device=DEV).bfloat16()
    with torch.inference_mode():
        assert mse.fused_reason(sm, lg) is None
        _lib.reset_launch_count()
        fs, fl = mse(sm, lg)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
    es, el = _eager_bf16(mse, sm, monkeypatch, lg)
    for got, want in ((fs, es), (fl, el)):
        assert got.shape == want.shape and got.dtype == torch.bfloat16
        ok, why = tokens_close(got, want)
        assert ok, why
    t = mse.layers[0][1]
    assert isinstance(t, Transformer)
    with torch.inference_mode():
        assert t.fused_reason(lg) is None
        out = t(lg)
    ok, why = tokens_close(out, _eager_bf16(t, lg, monkeypatch))
    assert ok, why


def test_extractor_on_multi_scale_encoder_stays_fused(monkeypatch):
    spec = CROSS_VIT_CASES["widths_32_64"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        plain = m(x)
    v = Extractor(m, layer_name='multi_scale_encoder')
    with torch.inference_mode():
        v._register_hook()
        assert m.fused_reason(x) is None
        _lib.reset_launch_count()
        logits, (sm, lg) = v(x)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
    assert sm.shape == (3, 65, 32) and lg.shape == (3, 17, 64)
    assert stats(logits, plain)[0] < 2e-2
    v.eject()
    ev = Extractor(m, layer_name='multi_scale_encoder')
    with monkeypatch.context() as mp:
        mp.setenv("B200VIT_DISABLE_FUSED", "1")
        with torch.inference_mode():
            _, (esm, elg) = ev(x)
    for got, want in ((sm, esm), (lg, elg)):
        ok, why = tokens_close(got, want)
        assert ok, why


def test_cuda_graph_replay_is_bit_identical():
    from vit_pytorch_b200.graph import GraphedForward
    spec = CROSS_VIT_CASES["widths_32_64"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    a = FAMILY.input(spec).to(DEV)
    b = torch.randn_like(a.float()).bfloat16()
    with torch.inference_mode():
        ya, yb = m(a).clone(), m(b).clone()
        g = GraphedForward(m, a)
        assert torch.equal(g(b), yb)
        assert torch.equal(g(a), ya)


# ------------------------------------------------------------------------------------------------------ fused_reason
KW = dict(image_size=32, num_classes=5, sm_dim=32, lg_dim=64, sm_patch_size=4, lg_patch_size=8, sm_enc_depth=1,
          sm_enc_heads=2, sm_enc_mlp_dim=64, sm_enc_dim_head=32, lg_enc_depth=1, lg_enc_heads=2, lg_enc_mlp_dim=64,
          lg_enc_dim_head=32, cross_attn_depth=1, cross_attn_heads=2, cross_attn_dim_head=32, depth=1)


def _model(**kw):
    return CrossViT(**dict(KW, **kw)).eval().to(DEV, torch.bfloat16)


def _img(c=3, s=32):
    return torch.randn(2, c, s, s, device=DEV).bfloat16()


def test_reason_eligible():
    with torch.inference_mode():
        assert _model().fused_reason(_img()) is None


def test_reason_not_cuda_or_wrong_dtype():
    m = _model()
    with torch.inference_mode():
        assert m.fused_reason(_img().cpu()) == "input is not on a CUDA device"
        assert "dtype" in m.fused_reason(_img().float())


def test_reason_not_sm90(monkeypatch):
    monkeypatch.setattr(torch.cuda, "get_device_capability", lambda *a: (8, 0))
    with torch.inference_mode():
        assert _model().fused_reason(_img()) == "device is not sm_90"


def test_reason_autograd():
    assert "autograd" in _model().fused_reason(_img())


def test_reason_dropout():
    m = _model(dropout=0.1, emb_dropout=0.1)
    with torch.inference_mode():
        assert m.train().fused_reason(_img()) == "dropout is active"
        assert m.eval().fused_reason(_img()) is None


def test_reason_inner_hooks():
    m = _model()
    h = m.multi_scale_encoder.layers[0][2].layers[0][0].fn.attend.register_forward_hook(lambda *a: None)
    with torch.inference_mode():
        assert m.fused_reason(_img()) == "forward hooks registered inside the model"
        assert m(_img()).shape == (2, 5)
    h.remove()
    h = m.multi_scale_encoder.register_forward_hook(lambda *a: None)
    with torch.inference_mode():
        assert m.fused_reason(_img()) is None
    h.remove()


@pytest.mark.parametrize("which", ["sm_enc_dim_head", "lg_enc_dim_head", "cross_attn_dim_head"])
def test_reason_dim_head(which):
    m = _model(**{which: 96})
    with torch.inference_mode():
        assert "dim_head=96" in m.fused_reason(_img())
        assert m(_img()).shape == (2, 5)


def test_reason_dims_not_multiple_of_8():
    with torch.inference_mode():
        assert "multiples of 8" in _model(sm_dim=36).fused_reason(_img())


def test_reason_image_not_divisible():
    with torch.inference_mode():
        assert "not divisible by the patch size" in _model().fused_reason(_img(s=34))


def test_reason_channel_mismatch():
    with torch.inference_mode():
        assert "channel count" in _model().fused_reason(_img(c=1))


def test_reason_positional_table_overflow():
    with torch.inference_mode():
        assert "exceed the positional table" in _model().fused_reason(_img(s=40))


def test_reason_sequence_too_long():
    m = _model(image_size=516, sm_patch_size=4, lg_patch_size=12)
    with torch.inference_mode():
        assert "16384" in m.fused_reason(_img(s=516))
