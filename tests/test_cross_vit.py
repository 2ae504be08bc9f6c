"""CrossViT (vit_pytorch_b200.cross_vit) without a GPU: the attribute surface, the eager graph's hooks, and the
argument checks of b200vit_attention_cls.  The reference-parity tests are in test_family_parity.py."""
import ctypes
import os
import sys

import pytest
import torch
from torch import nn

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build
from vit_pytorch_b200.cross_vit import (Attention, CrossTransformer, CrossViT, ImageEmbedder, MultiScaleEncoder,
                                        ProjectInOut, Transformer)

sys.path.insert(0, GOLDEN_DIR)
from cross_vit_spec import CROSS_VIT_CASES, FAMILY, INIT_KWARGS  # noqa: E402


def test_attribute_surface():
    m = CrossViT(**INIT_KWARGS)
    se, le = m.sm_image_embedder, m.lg_image_embedder
    assert isinstance(se, ImageEmbedder) and isinstance(m.multi_scale_encoder, MultiScaleEncoder)
    assert se.pos_embedding.shape == (1, 64 + 1, 32) and se.cls_token.shape == (1, 1, 32)
    assert le.pos_embedding.shape == (1, 16 + 1, 64) and le.cls_token.shape == (1, 1, 64)
    sm_enc, lg_enc, cross = m.multi_scale_encoder.layers[0]
    assert isinstance(sm_enc, Transformer) and isinstance(cross, CrossTransformer)
    assert [k for k, _ in sm_enc.named_parameters()][-2:] == ["norm.weight", "norm.bias"]   # layers before norm
    pio = cross.layers[0][0]
    assert isinstance(pio, ProjectInOut) and isinstance(pio.fn, Attention)
    assert [k.split(".")[0] for k, _ in pio.named_parameters()] == ["fn"] * 6 + ["project_in"] * 2 + \
        ["project_out"] * 2
    assert pio.project_in.weight.shape == (64, 32) and pio.fn.to_kv.weight.shape == (128, 64)
    eq = CrossViT(**dict(INIT_KWARGS, lg_dim=32))
    for pio in eq.multi_scale_encoder.layers[0][2].layers[0]:
        assert isinstance(pio.project_in, nn.Identity) and isinstance(pio.project_out, nn.Identity)
    assert m.sm_mlp_head[1].out_features == 7 and m.lg_mlp_head[0].normalized_shape == (64,)


def test_eager_graph_keeps_hooks_observable():
    """Recorder-style hooks on the cross-attention softmax fire on the PyTorch graph: one query row over the query
    token itself plus the other stream's patch tokens."""
    spec = CROSS_VIT_CASES["widths_32_64"]
    m = FAMILY.build(spec)
    seen = []
    for mse_layer in m.multi_scale_encoder.layers:
        for sm_lg, lg_sm in mse_layer[2].layers:
            sm_lg.fn.attend.register_forward_hook(lambda mod, i, o: seen.append(("sm", o)))
            lg_sm.fn.attend.register_forward_hook(lambda mod, i, o: seen.append(("lg", o)))
    with torch.inference_mode():
        m(FAMILY.input(spec).float())
    assert len(seen) == 2 * 2 * 2
    assert seen[0][0] == "sm" and seen[0][1].shape == (3, 2, 1, 1 + 16)     # self + 16 lg patches
    assert seen[1][0] == "lg" and seen[1][1].shape == (3, 2, 1, 1 + 64)     # self + 64 sm patches
    torch.testing.assert_close(seen[0][1].sum(-1), torch.ones(3, 2, 1))


def test_direct_calls_on_cpu():
    torch.manual_seed(0)
    t = Transformer(32, 2, 2, 16, 64).eval()
    mse = CrossViT(**INIT_KWARGS).eval().multi_scale_encoder
    with torch.inference_mode():
        assert t(torch.randn(2, 5, 32)).shape == (2, 5, 32)
        sm, lg = mse(torch.randn(2, 65, 32), torch.randn(2, 17, 64))
    assert sm.shape == (2, 65, 32) and lg.shape == (2, 17, 64)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_attention_cls_rejects_bad_arguments(lib):
    """Checks run before any device work: every one fails with dummy device pointers."""
    p = ctypes.c_void_p(256)
    call = lib.b200vit_attention_cls
    rc = call(None, p, 128, 17, 1, 16, p, 64, 3, 1, 64, 0.125, None)
    assert rc == -1 and b"null pointer" in lib.b200vit_last_error()
    rc = call(p, None, 128, 17, 1, 16, p, 64, 3, 1, 64, 0.125, None)
    assert rc == -1 and b"null pointer" in lib.b200vit_last_error()
    rc = call(p, p, 192, 17, 1, 16, p, 96, 3, 1, 96, 0.125, None)
    assert rc == -1 and b"dim_head=96" in lib.b200vit_last_error()
    rc = call(p, p, 128, 16390, 1, 16385, p, 64, 3, 1, 64, 0.125, None)
    assert rc == -1 and b"n=16385" in lib.b200vit_last_error()
    rc = call(p, p, 128, 17, 1, -1, p, 64, 3, 1, 64, 0.125, None)
    assert rc == -1 and b"n=-1" in lib.b200vit_last_error()
    rc = call(p, p, 128, 17, 1, 17, p, 64, 3, 1, 64, 0.125, None)
    assert rc == -1 and b"exceed the 17 rows per image" in lib.b200vit_last_error()
    rc = call(p, p, 132, 17, 1, 16, p, 64, 3, 1, 64, 0.125, None)
    assert rc == -1 and b"ctx_ld=132" in lib.b200vit_last_error()
    rc = call(p, p, 120, 17, 1, 16, p, 64, 3, 1, 64, 0.125, None)
    assert rc == -1 and b"ctx_ld=120" in lib.b200vit_last_error()
    rc = call(p, p, 128, 17, 1, 16, p, 68, 3, 1, 64, 0.125, None)
    assert rc == -1 and b"ldo=68" in lib.b200vit_last_error()
    rc = call(p, p, 128, 17, 1, 16, ctypes.c_void_p(264), 64, 3, 1, 64, 0.125, None)
    assert rc == -1 and b"16-byte aligned" in lib.b200vit_last_error()
    rc = call(p, p, 128, 17, 1, 16, p, 64, 0, 1, 64, 0.125, None)
    assert rc == -1 and b"bad shape" in lib.b200vit_last_error()


def test_header_declares_the_new_entry_point():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    assert "int b200vit_attention_cls(" in h and "b200vit_attention_cls" in _lib.SYMBOLS
