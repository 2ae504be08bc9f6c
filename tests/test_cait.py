"""CaiT (vit_pytorch_b200.cait) without a GPU: the attribute surface, the seeded cases' layer dropout and mixing-matrix
orientation, the eager graph's hooks, and the argument checks of the two talking-heads attention entry points.  The
reference-parity tests are in test_family_parity.py."""
import ctypes
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT, load_golden
from vit_pytorch_b200 import _lib, build
from vit_pytorch_b200.cait import Attention, CaiT, LayerScale, Transformer

sys.path.insert(0, GOLDEN_DIR)
from cait_spec import CAIT_CASES, FAMILY, INIT_KWARGS  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return load_golden("cait")


def test_layer_scale_init_follows_the_layer_index():
    torch.manual_seed(0)
    m = CaiT(**INIT_KWARGS)
    got = [ls.scale.flatten()[0].item() for ls, _ in m.patch_transformer.layers]
    assert got[:18] == [pytest.approx(0.1)] * 18 and got[18:] == [pytest.approx(1e-5)] * 2


def test_attribute_surface():
    m = CaiT(**INIT_KWARGS)
    assert m.pos_embedding.shape == (1, 16, 64) and m.cls_token.shape == (1, 1, 64)
    ls = m.patch_transformer.layers[0][0]
    assert isinstance(ls, LayerScale) and isinstance(ls.fn, Attention) and ls.scale.shape == (1, 1, 64)
    assert [k for k, _ in ls.named_parameters()][0] == "scale"
    names = [k for k, _ in ls.fn.named_parameters()]
    assert names[:2] == ["mix_heads_pre_attn", "mix_heads_post_attn"]
    assert isinstance(m.cls_transformer, Transformer) and not hasattr(m.patch_transformer, "norm")


def test_layer_dropout_case_drops_layers(golden):
    """The seeded layer-dropout case runs a strict subset: with every layer it gives other logits."""
    spec = dict(CAIT_CASES["readme_layer_dropout"])
    m = FAMILY.build(spec)
    m.patch_transformer.layer_dropout = m.cls_transformer.layer_dropout = 0.0
    with torch.inference_mode():
        out = m(FAMILY.input(spec).float())
    assert (out - golden["cases"]["readme_layer_dropout"]["logits_fp32"]).abs().max() > 1e-3


@pytest.mark.parametrize("which", ["mix_heads_pre_attn", "mix_heads_post_attn"])
def test_transposed_mixing_matrix_changes_the_logits(golden, which):
    """The einsums 'b h i j, h g -> b g i j' index both matrices [input head][output head]: a transpose is a different
    model, so the goldens pin the orientation of each."""
    spec = CAIT_CASES["dh32_n64"]
    m = FAMILY.build(spec)
    with torch.no_grad():
        for t in (m.patch_transformer, m.cls_transformer):
            for ls, _ in t.layers:
                w = getattr(ls.fn, which)
                w.copy_(w.t().contiguous())
    with torch.inference_mode():
        out = m(FAMILY.input(spec).float())
    assert (out - golden["cases"]["dh32_n64"]["logits_fp32"]).abs().max() > 1e-3


def test_eager_graph_keeps_hooks_observable():
    m = CaiT(**INIT_KWARGS).eval()
    seen = []
    m.cls_transformer.layers[0][0].fn.to_kv.register_forward_hook(lambda mod, i, o: seen.append(o.shape))
    assert m.fused_reason(torch.randn(2, 3, 32, 32)) is not None
    with torch.inference_mode():
        m(torch.randn(2, 3, 32, 32))
    assert seen == [(2, 17, 256)]                          # [LN(cls); 16 patch rows] -> k | v


def test_direct_transformer_call_on_cpu():
    torch.manual_seed(5)
    t = Transformer(64, 2, 4, 32, 96).eval()
    x = torch.randn(2, 9, 64)
    with torch.inference_mode():
        out = t(x)
        want = x
        for attn, ff in t.layers:
            want = attn(want) + want
            want = ff(want) + want
    assert torch.equal(out, want)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_attention_headmix_ex_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    f = ctypes.c_void_p(260)
    def call(*, qkv=p, out=p, B=2, N=16, H=4, dh=48, pre=f, post=f, g=None, b=None, eps=1e-5):
        rc = lib.b200vit_attention_headmix_ex(qkv, out, B, N, H, dh, 0.125, pre, post, g, b, eps, None)
        return rc, lib.b200vit_last_error()
    rc, msg = call(post=None)
    assert rc == -1 and b"null" in msg
    rc, msg = call(pre=ctypes.c_void_p(262))
    assert rc == -1 and b"4-byte aligned" in msg
    rc, msg = call(dh=96)
    assert rc == -1 and b"dim_head=96" in msg
    rc, msg = call(H=17, dh=32)
    assert rc == -1 and b"H=17" in msg
    rc, msg = call(N=16385)
    assert rc == -1 and b"16384" in msg


def test_attention_cls_headmix_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    f = ctypes.c_void_p(260)
    def call(*, q=p, ctx=p, ld=512, rows=197, first=0, n=196, out=p, ldo=192, B=2, H=4, dh=48, pre=f, post=f):
        rc = lib.b200vit_attention_cls_headmix(q, ctx, ld, rows, first, n, out, ldo, B, H, dh, 0.125, pre, post,
                                               None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(pre=None), dict(post=None), dict(ctx=None), dict(q=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    rc, msg = call(dh=96)
    assert rc == -1 and b"dim_head=96" in msg
    rc, msg = call(H=17, dh=32, ld=2 * 17 * 32, ldo=17 * 32)
    assert rc == -1 and b"H=17" in msg
    rc, msg = call(H=16, dh=80, ld=2560, ldo=1280)
    assert rc == -1 and b"H*dim_head=1280" in msg
    rc, msg = call(n=16385, rows=20000)
    assert rc == -1 and b"16384" in msg
    rc, msg = call(first=2, n=196)
    assert rc == -1 and b"rows per image" in msg
    rc, msg = call(ldo=100)
    assert rc == -1 and b"ldo" in msg
    rc, msg = call(ld=200)
    assert rc == -1 and b"ctx_ld" in msg
    rc, msg = call(out=ctypes.c_void_p(264))
    assert rc == -1 and b"16-byte aligned" in msg
    rc, msg = call(post=ctypes.c_void_p(262))
    assert rc == -1 and b"4-byte aligned" in msg
    rc, msg = call(B=0)
    assert rc == -1 and b"bad shape" in msg


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in ("b200vit_attention_headmix_ex", "b200vit_attention_cls_headmix"):
        assert f"int {name}(" in h and name in _lib.SYMBOLS
