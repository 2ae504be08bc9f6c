"""DeepViT (vit_pytorch_b200.deepvit) without a GPU: the attribute surface, the mixing-matrix orientation, the eager
graph's hooks, and the argument checks of the head-mixing attention entry point.  The reference-parity tests are in
test_family_parity.py."""
import ctypes
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT, load_golden
from vit_pytorch_b200 import _lib, build
from vit_pytorch_b200.deepvit import Attention, DeepViT, Transformer

sys.path.insert(0, GOLDEN_DIR)
from deepvit_spec import DEEPVIT_CASES, FAMILY, INIT_KWARGS  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return load_golden("deepvit")


def test_attribute_surface():
    m = DeepViT(**INIT_KWARGS)
    n = (32 // 8) ** 2
    assert m.pos_embedding.shape == (1, n + 1, 64) and m.cls_token.shape == (1, 1, 64)
    assert isinstance(m.transformer, Transformer) and not hasattr(m.transformer, "norm")
    attn = m.transformer.layers[0][0]
    assert isinstance(attn, Attention) and attn.reattn_weights.shape == (4, 4)
    assert attn.reattn_norm[1].normalized_shape == (4,)
    names = [k for k, _ in attn.named_parameters()]
    assert names[:2] == ["reattn_weights", "norm.weight"]


def test_transposed_mixing_matrix_changes_the_logits(golden):
    """The einsum 'b h i j, h g -> b g i j' indexes the matrix [input head][output head]: its transpose is a different
    model, so the goldens pin the orientation."""
    spec = DEEPVIT_CASES["dh32_n65"]
    m = FAMILY.build(spec)
    with torch.no_grad():
        for attn, _ in m.transformer.layers:
            attn.reattn_weights.copy_(attn.reattn_weights.t().contiguous())
    with torch.inference_mode():
        out = m(FAMILY.input(spec).float())
    assert (out - golden["cases"]["dh32_n65"]["logits_fp32"]).abs().max() > 1e-2


def test_eager_graph_keeps_hooks_observable():
    m = DeepViT(**INIT_KWARGS).eval()
    seen = []
    m.transformer.layers[0][0].reattn_norm[1].register_forward_hook(lambda mod, i, o: seen.append(o.shape))
    assert m.fused_reason(torch.randn(2, 3, 32, 32)) is not None
    with torch.inference_mode():
        m(torch.randn(2, 3, 32, 32))
    assert seen == [(2, 17, 17, 4)]                        # b i j h: the LayerNorm runs over the heads


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


def test_attention_headmix_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    f = ctypes.c_void_p(260)
    def call(*, qkv=p, out=p, B=2, N=16, H=4, dh=64, post=f, g=None, b=None, eps=1e-5):
        rc = lib.b200vit_attention_headmix(qkv, out, B, N, H, dh, 0.125, post, g, b, eps, None)
        return rc, lib.b200vit_last_error()
    rc, msg = call(post=None)
    assert rc == -1 and b"null" in msg
    rc, msg = call(g=f)
    assert rc == -1 and b"both gamma and beta" in msg
    rc, msg = call(dh=96)
    assert rc == -1 and b"dim_head=96" in msg
    rc, msg = call(H=17, dh=32)
    assert rc == -1 and b"H=17" in msg
    rc, msg = call(H=16, dh=80)
    assert rc == -1 and b"H*dim_head=1280" in msg
    rc, msg = call(N=16385)
    assert rc == -1 and b"16384" in msg
    rc, msg = call(N=0)
    assert rc == -1 and b"bad shape" in msg
    rc, msg = call(qkv=ctypes.c_void_p(264))
    assert rc == -1 and b"16-byte aligned" in msg
    rc, msg = call(post=ctypes.c_void_p(262))
    assert rc == -1 and b"4-byte aligned" in msg
    rc, msg = call(g=f, b=f, eps=0.0)
    assert rc == -1 and b"eps" in msg


def test_header_declares_the_new_entry_point():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    assert "int b200vit_attention_headmix(" in h and "b200vit_attention_headmix" in _lib.SYMBOLS
