"""XCiT (vit_pytorch_b200.xcit) without a GPU: the attribute surface, the seeded layer-dropout case, the BatchNorm /
LayerScale fold of the local patch interaction, the fallback rules, and the argument checks of the cross-covariance
attention, local patch interaction and class attention entry points.  The reference-parity tests are in
test_family_parity.py."""
import ctypes
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR, ROOT, load_golden
from vit_pytorch_b200 import _lib, build
from vit_pytorch_b200.engine import LPIBlock, Norm, lpi_reason, lpi_weights, xca_reason
from vit_pytorch_b200.xcit import (LayerScale, LocalPatchInteraction, XCATransformer, XCAttention, XCiT,
                                   batchnorm_reason)

sys.path.insert(0, GOLDEN_DIR)
from xcit_spec import FAMILY, INIT_KWARGS, XCIT_CASES  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return load_golden("xcit")


def test_layer_scale_init_follows_the_reference_condition():
    """`18 > depth <= 24` is False above depth 18: layers 19 and 20 start at 1e-6, not CaiT's 1e-5."""
    torch.manual_seed(0)
    m = XCiT(**INIT_KWARGS)
    got = [ls.scale[0].item() for ls, _, _ in m.xcit_transformer.layers]
    assert got[:18] == [pytest.approx(0.1)] * 18 and got[18:] == [pytest.approx(1e-6)] * 2


def test_attribute_surface():
    m = XCiT(**INIT_KWARGS)
    assert m.pos_embedding.shape == (1, 16, 64) and m.cls_token.shape == (64,)
    ls = m.xcit_transformer.layers[0][0]
    assert isinstance(ls, LayerScale) and isinstance(ls.fn, XCAttention) and ls.scale.shape == (64,)
    assert ls.fn.temperature.shape == (4, 1, 1)
    lpi = m.xcit_transformer.layers[0][1].fn
    assert isinstance(lpi, LocalPatchInteraction)
    assert [k for k, _ in lpi.named_buffers()] == ["net.3.running_mean", "net.3.running_var",
                                                   "net.3.num_batches_tracked"]
    assert isinstance(m.xcit_transformer, XCATransformer) and not hasattr(m.xcit_transformer, "norm")


def test_layer_dropout_case_drops_layers(golden):
    spec = dict(XCIT_CASES["readme_layer_dropout"])
    m = FAMILY.build(spec)
    m.xcit_transformer.layer_dropout = m.cls_transformer.layer_dropout = 0.0
    with torch.inference_mode():
        out = m(FAMILY.input(spec).float())
    assert (out - golden["cases"]["readme_layer_dropout"]["logits_fp32"]).abs().max() > 1e-3


@pytest.mark.parametrize("k", [1, 3, 5, 7])
@pytest.mark.parametrize("hw", [(1, 1), (1, 5), (2, 2), (6, 8)])
def test_lpi_fold_reproduces_the_module(k, hw):
    """lpi_weights (BatchNorm folded into conv1, LayerScale into conv2, tap-major) applied as depthwise convolutions in
    fp32 torch, with the LayerNorm output zero-padded and the GELU output zero-padded, gives scale * LPI(x)."""
    torch.manual_seed(k)
    D = 16
    ls = LayerScale(D, LocalPatchInteraction(D, k), depth=1).eval()
    net = ls.fn.net
    with torch.no_grad():
        for p in ls.parameters():
            p.add_(0.2 * torch.randn(p.shape))
        net[3].running_mean.normal_(0, 0.3)
        net[3].running_var.uniform_(0.5, 2.0)
    x = torch.randn(2, *hw, D)
    blk = LPIBlock(ln=Norm.of(net[0]), conv1_w=net[2].weight, conv1_b=net[2].bias, bn_w=net[3].weight,
                   bn_b=net[3].bias, bn_mean=net[3].running_mean, bn_var=net[3].running_var, bn_eps=net[3].eps,
                   conv2_w=net[5].weight, conv2_b=net[5].bias, scale=ls.scale, kernel_size=k)
    w1, b1, w2, b2 = lpi_weights(blk)
    assert w1.shape == (k * k, D) and w2.shape == (k * k, D)
    with torch.no_grad():
        z = F.layer_norm(x, (D,), net[0].weight, net[0].bias, net[0].eps).permute(0, 3, 1, 2)
        u = F.gelu(F.conv2d(z, w1.t().reshape(D, 1, k, k), b1, padding=k // 2, groups=D))
        got = F.conv2d(u, w2.t().reshape(D, 1, k, k), b2, padding=k // 2, groups=D).permute(0, 2, 3, 1)
        want = ls(x)
    assert torch.allclose(got, want, atol=1e-5, rtol=1e-5), (got - want).abs().max()


def test_fallback_rules_without_a_gpu():
    assert xca_reason(96) is not None and "dim_head=96" in xca_reason(96)
    assert all(xca_reason(dh) is None for dh in (32, 48, 64, 80, 128))
    assert "local_patch_kernel_size=9" in lpi_reason(9, 8)
    assert all(lpi_reason(k, 56) is None for k in (1, 3, 5, 7))
    assert "too wide" in lpi_reason(7, 400)
    m = XCiT(**INIT_KWARGS).eval()
    assert batchnorm_reason(m) is None
    m.xcit_transformer.layers[1][1].fn.net[3].train()
    assert "BatchNorm2d" in batchnorm_reason(m)
    m.train()
    assert "BatchNorm2d" in batchnorm_reason(m)
    assert m.fused_reason(torch.randn(2, 3, 32, 32)) is not None       # CPU input


def test_graph_reason_refuses_layer_dropout():
    assert XCiT(**INIT_KWARGS).graph_reason() is None
    assert "layer_dropout" in XCiT(**{**INIT_KWARGS, "layer_dropout": 0.1}).graph_reason()


def test_direct_transformer_call_on_cpu():
    torch.manual_seed(5)
    t = XCATransformer(64, 2, 4, 32, 96).eval()
    x = torch.randn(2, 3, 5, 64)
    with torch.inference_mode():
        out = t(x)
        want = x
        for a, lpi, ff in t.layers:
            want = a(want) + want
            want = lpi(want) + want
            want = ff(want) + want
    assert torch.equal(out, want)


def test_eager_graph_keeps_hooks_observable():
    m = XCiT(**INIT_KWARGS).eval()
    seen = []
    m.xcit_transformer.layers[0][1].fn.net[2].register_forward_hook(lambda mod, i, o: seen.append(o.shape))
    with torch.inference_mode():
        m(torch.randn(2, 3, 32, 32))
    assert seen == [(2, 64, 4, 4)]


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_attention_xca_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    f = ctypes.c_void_p(260)
    def call(*, qkv=p, tau=f, out=p, B=2, N=196, H=8, dh=48):
        rc = lib.b200vit_attention_xca(qkv, tau, out, B, N, H, dh, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(qkv=None), dict(tau=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    rc, msg = call(dh=96)
    assert rc == -1 and b"dim_head=96" in msg and b"32, 48, 64, 80 or 128" in msg
    rc, msg = call(N=16385)
    assert rc == -1 and b"16384" in msg
    rc, msg = call(N=0)
    assert rc == -1 and b"bad shape" in msg
    rc, msg = call(B=0)
    assert rc == -1 and b"bad shape" in msg
    rc, msg = call(out=ctypes.c_void_p(264))
    assert rc == -1 and b"16-byte aligned" in msg
    rc, msg = call(tau=ctypes.c_void_p(262))
    assert rc == -1 and b"4-byte aligned" in msg


def test_local_patch_interaction_rejects_bad_arguments(lib):
    x, y = 1 << 20, 1 << 30
    f = ctypes.c_void_p(260)
    def call(*, x=ctypes.c_void_p(x), y=ctypes.c_void_p(y), yb=ctypes.c_void_p(1 << 34), ys=f, B=2, h=14, w=14,
             D=384, k=3, g=f):
        rc = lib.b200vit_local_patch_interaction(x, y, yb, ys, f, g, f, 1e-5, f, f, f, f, B, h, w, D, k, None)
        return rc, lib.b200vit_last_error()
    rc, msg = call(g=None)
    assert rc == -1 and b"null" in msg
    rc, msg = call(yb=None)
    assert rc == -1 and b"both" in msg
    for k in (0, 2, 9):
        rc, msg = call(k=k)
        assert rc == -1 and f"kernel size {k}".encode() in msg
    rc, msg = call(D=386)
    assert rc == -1 and b"multiple of 4" in msg
    rc, msg = call(h=0)
    assert rc == -1 and b"bad shape" in msg
    rc, msg = call(y=ctypes.c_void_p(x + 4096))
    assert rc == -1 and b"overlaps" in msg
    rc, msg = call(y=ctypes.c_void_p(y + 8))
    assert rc == -1 and b"16-byte aligned" in msg
    rc, msg = call(w=2000, k=7)
    assert rc == -1 and b"shared memory" in msg


def test_attention_cls_accepts_dim_head_48(lib):
    """dh 48 passes the width check, which comes before the row-stride and alignment checks: a call whose only fault
    is a later one fails on that fault, not on the width (a build without the dh 48 instance fails on the width)."""
    p = ctypes.c_void_p(256)
    def call(*, out=p, ldo=96, dh=48):                     # B = 3 images, H = 2 heads
        rc = lib.b200vit_attention_cls(p, p, 2 * 2 * dh, 17, 1, 16, out, ldo, 3, 2, dh, 0.125, None)
        return rc, lib.b200vit_last_error()
    rc, msg = call(ldo=88)
    assert rc == -1 and b"ldo=88" in msg, msg
    rc, msg = call(out=ctypes.c_void_p(264))
    assert rc == -1 and b"16-byte aligned" in msg, msg
    rc, msg = call(dh=40, ldo=80)
    assert rc == -1 and b"dim_head=40" in msg and b"32, 48, 64, 80 or 128" in msg, msg


def test_train_mode_forward_rebuilds_the_folded_batchnorm():
    """A train-mode forward updates BatchNorm's running statistics in place without bumping their version counters;
    the prepared conv1 weights must still follow them (the batch counter is part of the key)."""
    torch.manual_seed(7)
    m = XCiT(**INIT_KWARGS).eval()
    eng = m.xcit_transformer.engine()
    bn = m.xcit_transformer.layers[0][1].fn.net[3]
    before = eng.prepared()["0.lpi.w1"].clone()
    m.train()
    with torch.no_grad():
        m(torch.randn(4, 3, 32, 32))
    m.eval()
    after = eng.prepared()["0.lpi.w1"]
    want = lpi_weights(eng.layers[0].lpi)[0]
    assert not torch.equal(after, before) and torch.equal(after, want)
    assert torch.equal(want, (m.xcit_transformer.layers[0][1].fn.net[2].weight.detach().reshape(64, 9)
                              * (bn.weight / torch.sqrt(bn.running_var + bn.eps))[:, None]).t())


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in ("b200vit_attention_xca", "b200vit_local_patch_interaction"):
        assert f"int {name}(" in h and name in _lib.SYMBOLS
