"""-m gpu: the shifted-patch tokenizer, the self-masked attention, token assembly without a LayerNorm and the fused
ViT for small datasets on the H100.  Kernels are checked against torch expressions on the same bf16 data; the model's
two host loops against each other (its reference parity is in test_gpu_family_parity.py)."""
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR
from oracle import attention_bounds as AB
from oracle import bounds as Bd
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.vit import Patchify
from vit_pytorch_b200.vit_for_small_dataset import SPT_SHIFTS, Transformer, ViT

sys.path.insert(0, GOLDEN_DIR)
from vit_small_spec import FAMILY, VIT_SMALL_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
RTOL, ATOL = 1e-2, 1e-3


def within(got, ref, rtol=RTOL, atol=ATOL):
    got, ref = got.float().cpu(), ref.float().cpu()
    return ((got - ref).abs() <= atol + rtol * ref.abs()).float().mean().item()


def close(got, want, atol=2e-2, rtol=1e-2):
    """Elementwise |got - want| <= atol + rtol |want|: the outputs are bf16, so the error grows with the value."""
    return bool(((got.float() - want).abs() <= atol + rtol * want.abs()).all())


def stats(got, ref):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    return d.max().item(), within(got, ref)


# ------------------------------------------------------------------------------------------------------ patchify_spt_ln
def spt_reference(img, p, g, b):
    """F.pad x 4 + cat + '(p1 p2 c)' patchify + LayerNorm, fp32 (vit_for_small_dataset.py:92-96 and :86-87)."""
    x = img.float()
    xs = torch.cat([x] + [F.pad(x, s) for s in SPT_SHIFTS], dim=1)
    patches = Patchify(p, p)(xs)
    return F.layer_norm(patches, (patches.shape[-1],), g, b, eps=1e-5).reshape(-1, patches.shape[-1])


@pytest.mark.parametrize("C,H,W,p,extra", [(3, 32, 32, 4, 0), (3, 32, 32, 4, 64), (1, 32, 32, 8, 0), (4, 32, 32, 4, 0),
                                           (3, 32, 32, 16, 0), (4, 32, 48, 16, 0), (3, 24, 32, 4, 0), (3, 48, 16, 8, 0),
                                           (1, 20, 12, 4, 0), (3, 256, 256, 16, 0), (3, 224, 224, 8, 0)])
def test_patchify_spt_ln(C, H, W, p, extra):
    torch.manual_seed(C * 1000 + H + W + p)
    img = torch.randn(2, C, H, W, device=DEV)
    # distinctive borders: a wrong shift direction or a missing zero fill shows up at once
    img[:, :, 0, :] += 3.0
    img[:, :, :, -1] -= 3.0
    img = img.bfloat16()
    pd = 5 * C * p * p
    ldo = (pd + 63) // 64 * 64 + extra
    g, b = 1 + 0.2 * torch.randn(pd, device=DEV), 0.1 * torch.randn(pd, device=DEV)
    out = torch.full((2 * (H // p) * (W // p), ldo), 7.0, device=DEV, dtype=torch.bfloat16)
    _lib.patchify_spt_ln(img, g, b, out, p)
    # within one bf16 ulp (plus the fp32 error of the LayerNorm) of the fp64 LayerNorm of every shifted patch
    xs = torch.cat([img] + [F.pad(img, s) for s in SPT_SHIFTS], dim=1)
    Bd.check(out[:, :pd], *Bd.layernorm_reference(Patchify(p, p)(xs).reshape(-1, pd), g, b), "patchify_spt_ln")
    assert torch.allclose(out[:, :pd].float(), spt_reference(img, p, g, b), rtol=1e-2, atol=2e-2)
    assert (out[:, pd:] == 0).all()


# ------------------------------------------------------------------------------------------------------ masked attention
def masked_reference(qkv, lengths, H, dh, scale):
    """fp32 softmax(q k^T * scale) v per sequence with the diagonal filled with -finfo.max (LSA)."""
    outs, s0 = [], 0
    for n in lengths:
        t = qkv[s0:s0 + n].float().view(n, 3, H, dh).permute(1, 2, 0, 3)
        q, k, v = t[0], t[1], t[2]
        dots = q @ k.transpose(-1, -2) * scale
        dots = dots.masked_fill(torch.eye(n, device=qkv.device, dtype=torch.bool), -torch.finfo(dots.dtype).max)
        outs.append((dots.softmax(-1) @ v).permute(1, 0, 2).reshape(n, H * dh))
        s0 += n
    return torch.cat(outs)


def _ex(qkv, out, B, N, H, dh, scale, flags):
    rc = _lib.lib().b200vit_attention_ex(qkv.data_ptr(), out.data_ptr(), B, N, H, dh, scale, flags,
                                         torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.lib().b200vit_last_error()


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("N", [1, 2, 65, 127, 128, 129, 257, 512])
def test_masked_attention_against_fp32(dh, N):
    torch.manual_seed(dh * 1000 + N)
    B, H = 3, 2
    qkv = (2 * torch.randn(B * N, 3 * H * dh, device=DEV)).bfloat16()
    scale = 0.7 * dh ** -0.5
    out = torch.empty(B * N, H * dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention(qkv, out, B, N, H, dh, scale, mask_self=True)
    want = masked_reference(qkv, [N] * B, H, dh, scale)
    assert torch.isfinite(out.float()).all()
    assert close(out, want), (out.float() - want).abs().max().item()
    Bd.check(out, *AB.qkv_attention_reference(qkv, [N] * B, H, dh, scale, mask_self=True), "MASK_SELF")
    # flags = 0 is the existing entry point, bit for bit
    plain, ex0 = torch.empty_like(out), torch.empty_like(out)
    _lib.attention(qkv, plain, B, N, H, dh, scale)
    Bd.check(plain, *AB.qkv_attention_reference(qkv, [N] * B, H, dh, scale), "flags = 0")
    _ex(qkv, ex0, B, N, H, dh, scale, 0)
    assert torch.equal(plain, ex0)
    if N == 1:                                             # the reference's fill leaves the only key: out = v
        assert torch.equal(out, qkv[:, 2 * H * dh:]) and torch.equal(out, plain)
    else:
        assert not torch.equal(out, plain)


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("lengths", [[513] * 2, [577] * 2, [1025], [1, 513, 2, 130]])
def test_masked_varlen_attention_against_fp32(dh, lengths):
    torch.manual_seed(dh + sum(lengths))
    H = 2
    T = sum(lengths)
    qkv = (2 * torch.randn(T, 3 * H * dh, device=DEV)).bfloat16()
    scale = 1.3 * dh ** -0.5
    cu, tp, tiles = _lib.varlen_index(lengths, DEV)
    out = torch.empty(T, H * dh, device=DEV, dtype=torch.bfloat16)
    _lib.attention_varlen(qkv, out, cu, tp, tiles, H, dh, scale, mask_self=True)
    want = masked_reference(qkv, lengths, H, dh, scale)
    assert torch.isfinite(out.float()).all()
    assert close(out, want), (out.float() - want).abs().max().item()
    Bd.check(out, *AB.qkv_attention_reference(qkv, lengths, H, dh, scale, mask_self=True), "MASK_SELF")
    plain, ex0 = torch.empty_like(out), torch.empty_like(out)
    _lib.attention_varlen(qkv, plain, cu, tp, tiles, H, dh, scale)
    Bd.check(plain, *AB.qkv_attention_reference(qkv, lengths, H, dh, scale), "flags = 0")
    rc = _lib.lib().b200vit_attention_varlen_ex(qkv.data_ptr(), ex0.data_ptr(), cu.data_ptr(), tp.data_ptr(),
                                                len(lengths), T, tiles, H, dh, scale, 0,
                                                torch.cuda.current_stream().cuda_stream)
    assert rc == 0 and torch.equal(plain, ex0)


# ------------------------------------------------------------------------------------------------------ token assembly
@pytest.mark.parametrize("D", [64, 96, 50])
def test_embed_tokens_without_layernorm(D):
    torch.manual_seed(D)
    B, n = 3, 16
    y = torch.randn(B * n, D, device=DEV)
    cls = torch.randn(1, D, device=DEV)
    pos = torch.randn(n + 1, D, device=DEV)
    x = torch.empty(B * (n + 1), D, device=DEV)
    xb = torch.empty(B * (n + 1), D, device=DEV, dtype=torch.bfloat16)
    st = torch.empty(B * (n + 1), 2, device=DEV)
    _lib.embed_tokens(y, None, None, cls, pos, x, B, n, 1, xb=xb, stats=st)
    want = torch.cat((cls.expand(B, 1, D), y.view(B, n, D)), dim=1) + pos
    assert torch.equal(x, want.reshape(-1, D))
    assert torch.equal(xb, x.bfloat16())
    torch.testing.assert_close(st[:, 0], xb.float().sum(1), rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(st[:, 1], (xb.float() ** 2).sum(1), rtol=1e-4, atol=1e-3)


# ------------------------------------------------------------------------------------------------------ model
def _eager_bf16(m, x, monkeypatch):
    """The module's own PyTorch graph in bf16 (every submodule, the Transformer included)."""
    with monkeypatch.context() as mp:
        mp.setenv("B200VIT_DISABLE_FUSED", "1")
        with torch.inference_mode():
            return m(x)


@pytest.mark.parametrize("name", ["c32_p4_cls", "long_577"])
def test_c_and_python_layer_loops_agree(name, monkeypatch):
    """b200vit_encoder_blocks_ex (per-layer scales, self mask) against the per-kernel Python loop: the same launches,
    the same bits."""
    spec = VIT_SMALL_CASES[name]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        m(x)
        _lib.reset_launch_count()
        c_out = m(x).clone()
        torch.cuda.synchronize()
        c_launches = _lib.launch_count()
        monkeypatch.setenv("B200VIT_HOST_LOOP", "python")
        _lib.reset_launch_count()
        py_out = m(x).clone()
        torch.cuda.synchronize()
        py_launches = _lib.launch_count()
    assert torch.equal(c_out, py_out)
    assert c_launches == py_launches


def test_in_place_temperature_change_reaches_the_fused_path(monkeypatch):
    spec = VIT_SMALL_CASES["c32_p4_mean"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        before = m(x).clone()
    with torch.no_grad():
        m.transformer.layers[1][0].temperature.add_(3.0)
    with torch.inference_mode():
        after = m(x).clone()
    eager = _eager_bf16(m, x, monkeypatch)
    assert (after.float() - before.float()).abs().max().item() > 2e-2
    mx_after, mx_before = stats(after, eager)[0], stats(before, eager)[0]
    print(f"vs eager after the change: fused {mx_after:.5f}, fused before it {mx_before:.5f}")
    assert mx_after < 5e-2 and mx_after < mx_before / 2, (mx_after, mx_before)


def test_cuda_graph_replay_is_bit_identical():
    from vit_pytorch_b200.graph import GraphedForward
    spec = VIT_SMALL_CASES["c32_p4_cls"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    a = FAMILY.input(spec).to(DEV)
    b = torch.randn_like(a.float()).bfloat16()
    with torch.inference_mode():
        ya, yb = m(a).clone(), m(b).clone()
        g = GraphedForward(m, a)
        assert torch.equal(g(b), yb)
        assert torch.equal(g(a), ya)


def test_transformer_hook_keeps_the_fused_path():
    """A hook on .transformer (the Extractor pattern) sees the encoder output while the blocks still run fused."""
    spec = VIT_SMALL_CASES["c32_p4_cls"]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    seen = {}
    with torch.inference_mode():
        plain = m(x)
        h = m.transformer.register_forward_hook(lambda _m, _i, o: seen.setdefault("o", o))
        assert m.fused_reason(x) is None
        _lib.reset_launch_count()
        hooked = m(x)
        torch.cuda.synchronize()
        assert _lib.launch_count() >= 3 + 5 * 2
        h.remove()
    assert seen["o"].shape == (3, 65, 64)
    assert (hooked.float() - plain.float()).abs().max() < 2e-2          # tokens passed through bf16 once


def test_direct_transformer_call(monkeypatch):
    torch.manual_seed(3)
    t = Transformer(128, 2, 2, 64, 256).eval()
    with torch.no_grad():
        for i, (attn, _) in enumerate(t.layers):
            attn.temperature.add_(0.4 * (i + 1))
        for p in t.parameters():
            p.copy_(p.bfloat16().float())
    ref = Transformer(128, 2, 2, 64, 256).eval()
    ref.load_state_dict(t.state_dict())
    t = t.to(DEV, torch.bfloat16)
    x = torch.randn(5, 33, 128, device=DEV).bfloat16()
    with torch.inference_mode():
        assert t.fused_reason(x) is None
        _lib.reset_launch_count()
        out = t(x)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = ref(x.float().cpu())
    mx, frac = stats(out, want)
    assert mx < 6e-2 and frac > 0.85, (mx, frac)


def test_fallback_reasons():
    kw = dict(image_size=32, patch_size=4, num_classes=3, dim=64, depth=1, heads=2, mlp_dim=64)
    x = torch.randn(2, 3, 32, 32, device=DEV).bfloat16()
    dh96 = ViT(dim_head=96, **kw).eval().to(DEV, torch.bfloat16)
    with torch.inference_mode():
        assert "dim_head=96" in dh96.fused_reason(x)
        assert dh96(x).shape == (2, 3)                     # eager, like the reference
    drop = ViT(dim_head=32, dropout=0.1, **kw).to(DEV, torch.bfloat16)
    with torch.inference_mode():
        assert drop.train().fused_reason(x) == "dropout is active"
        assert drop.eval().fused_reason(x) is None
        assert "channel count" in drop.fused_reason(torch.randn(2, 1, 32, 32, device=DEV).bfloat16())
        h = drop.transformer.layers[0][0].attend.register_forward_hook(lambda *a: None)
        assert "hooks" in drop.fused_reason(x)
        h.remove()
    assert "autograd" in ViT(dim_head=32, **kw).eval().to(DEV, torch.bfloat16).fused_reason(x)
