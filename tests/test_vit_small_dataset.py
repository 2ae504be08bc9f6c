"""ViT for small datasets (vit_pytorch_b200.vit_for_small_dataset) without a GPU: the attribute surface, the seeded
cases' temperatures, the eager graph's hooks, and the argument checks of the new C entry points (shifted-patch
tokenization, self-masked attention, the per-layer-scale encoder and token assembly without a LayerNorm).  The
reference-parity tests are in test_family_parity.py."""
import ctypes
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build
from vit_pytorch_b200.vit_for_small_dataset import LSA, SPT, Transformer, ViT

sys.path.insert(0, GOLDEN_DIR)
from vit_small_spec import FAMILY, INIT_KWARGS, VIT_SMALL_CASES  # noqa: E402


def test_attribute_surface():
    m = ViT(**INIT_KWARGS)
    n = (32 // 4) ** 2
    assert m.pos_embedding.shape == (1, n + 1, 64) and m.cls_token.shape == (1, 1, 64)
    assert isinstance(m.to_patch_embedding, SPT) and isinstance(m.transformer, Transformer)
    assert m.to_patch_embedding.to_patch_tokens[1].normalized_shape == (5 * 3 * 4 * 4,)
    attn = m.transformer.layers[0][0]
    assert isinstance(attn, LSA) and attn.temperature.dim() == 0
    assert torch.allclose(attn.temperature.exp(), torch.tensor(32 ** -0.5))
    assert not hasattr(m.transformer, "norm")              # the reference's Transformer has no final LayerNorm
    names = [k for k, _ in m.transformer.layers[0][0].named_parameters()]
    assert names[:2] == ["temperature", "norm.weight"]


@pytest.mark.parametrize("name", sorted(VIT_SMALL_CASES))
def test_seeded_cases_move_every_temperature_off_its_default(name):
    """The recipe perturbs every layer's temperature (its default is exactly log(dim_head ** -0.5), so a fused path
    that ignored it would still match the reference's logits)."""
    m = FAMILY.build(VIT_SMALL_CASES[name])
    temps = [layer[0].temperature.item() for layer in m.transformer.layers]
    assert all(abs(t - torch.tensor(m.transformer.layers[0][0].dim_head ** -0.5).log().item()) > 0.1 for t in temps)


def test_eager_graph_keeps_hooks_observable():
    """Recorder-style hooks on the LSA softmax fire on the PyTorch graph, with the self mask visible in the weights."""
    spec = VIT_SMALL_CASES["c32_p4_cls"]
    m = FAMILY.build(spec)
    seen = []
    for attn, _ in m.transformer.layers:
        attn.attend.register_forward_hook(lambda mod, i, o: seen.append(o))
    with torch.inference_mode():
        m(FAMILY.input(spec).float())
    assert len(seen) == 2 and seen[0].shape == (3, 2, 65, 65)
    assert (seen[0].diagonal(dim1=-2, dim2=-1) == 0).all()


def test_single_token_attends_to_itself():
    """N = 1: every key is masked and the reference's -finfo.max fill gives that key weight 1, so LSA returns
    to_out(v) -- the case the fused kernel keeps by not masking a sequence of one token."""
    torch.manual_seed(0)
    a = LSA(32, heads=2, dim_head=16).eval()
    x = torch.randn(2, 1, 32)
    with torch.no_grad():
        v = a.to_qkv(a.norm(x)).chunk(3, dim=-1)[2]
        torch.testing.assert_close(a(x), a.to_out(v))


def test_direct_transformer_call_on_cpu():
    t = Transformer(32, 2, 2, 16, 64).eval()
    with torch.inference_mode():
        assert t(torch.randn(2, 5, 32)).shape == (2, 5, 32)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_patchify_spt_ln_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_patchify_spt_ln(p, p, p, p, 256, 1, 3, 30, 32, 4, 1e-5, None)
    assert rc == -1 and b"divisible" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_spt_ln(p, p, p, p, 232, 1, 3, 32, 32, 4, 1e-5, None)
    assert rc == -1 and b"ldo=232 must be >= 5*C*p*p=240" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_spt_ln(p, p, p, p, 244, 1, 3, 32, 32, 4, 1e-5, None)
    assert rc == -1 and b"multiple of 8" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_spt_ln(p, p, p, ctypes.c_void_p(264), 256, 1, 3, 32, 32, 4, 1e-5, None)
    assert rc == -1 and b"16-byte aligned" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_spt_ln(p, None, p, p, 256, 1, 3, 32, 32, 4, 1e-5, None)
    assert rc == -1 and b"null" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_spt_ln(p, p, p, p, 3840, 1, 3, 16, 16384, 16, 1e-5, None)
    assert rc == -1 and b"exceeds shared memory" in lib.b200vit_last_error()


def test_attention_ex_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_attention_ex(p, p, 1, 16, 1, 64, 0.1, 2, None)
    assert rc == -1 and b"unknown flags 0x2" in lib.b200vit_last_error()
    rc = lib.b200vit_attention_ex(p, p, 1, 16, 1, 96, 0.1, 1, None)
    assert rc == -1 and b"dim_head=96" in lib.b200vit_last_error()
    rc = lib.b200vit_attention_ex(p, p, 1, 513, 1, 64, 0.1, 1, None)
    assert rc == -1 and b"512" in lib.b200vit_last_error()
    rc = lib.b200vit_attention_varlen_ex(p, p, p, p, 1, 16, 1, 1, 64, 0.1, 4, None)
    assert rc == -1 and b"unknown flags 0x4" in lib.b200vit_last_error()
    rc = lib.b200vit_attention_varlen_ex(p, p, None, p, 1, 16, 1, 1, 64, 0.1, 1, None)
    assert rc == -1 and b"null" in lib.b200vit_last_error()


def test_encoder_blocks_ex_rejects_bad_arguments(lib):
    """Checks run before any device work: a bad flag or a non-finite layer scale fails with dummy device pointers."""
    layers = (_lib.Layer * 2)()
    full = _lib.EncoderWs(*([256] * 7))
    x = ctypes.c_void_p(256)
    ok = (ctypes.c_float * 2)(0.1, 0.2)
    rc = lib.b200vit_encoder_blocks_ex(layers, 2, x, ctypes.byref(full), 1, 16, 64, 1, 64, 128, 0.125, 1, None, None,
                                       0, None, 0, ok, 2, None)
    assert rc == -1 and b"unknown attention flags 0x2" in lib.b200vit_last_error()
    bad = (ctypes.c_float * 2)(0.1, float("nan"))
    rc = lib.b200vit_encoder_blocks_ex(layers, 2, x, ctypes.byref(full), 1, 16, 64, 1, 64, 128, 0.125, 1, None, None,
                                       0, None, 0, bad, 1, None)
    assert rc == -1 and b"layer 1 has a non-finite scale" in lib.b200vit_last_error()
    rc = lib.b200vit_encoder_blocks_ex(layers, 2, x, ctypes.byref(_lib.EncoderWs()), 1, 16, 64, 1, 64, 128, 0.125, 1,
                                       None, None, 0, None, 0, ok, 1, None)
    assert rc == -1 and b"workspace" in lib.b200vit_last_error()
    rc = lib.b200vit_encoder_blocks_ex(layers, 2, x, ctypes.byref(full), 1, 600, 64, 1, 64, 128, 0.125, 1, None, None,
                                       0, None, 0, ok, 1, None)
    assert rc == -1 and b"varlen" in lib.b200vit_last_error()
    # valid flags and scales get as far as the layers' weights (all NULL here), still before any launch
    rc = lib.b200vit_encoder_blocks_ex(layers, 2, x, ctypes.byref(full), 1, 16, 64, 1, 64, 128, 0.125, 1, None, None,
                                       0, None, 0, ok, 1, None)
    assert rc == -1 and b"layer 0 has a null weight" in lib.b200vit_last_error()


def test_embed_tokens_without_layernorm_checks_beta_only_with_gamma(lib):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_embed_tokens(p, p, None, None, p, None, p, None, None, 2, 4, 0, 0, 64, 1e-5, None)
    assert rc == -1 and b"null pointer" in lib.b200vit_last_error()
    rc = lib.b200vit_embed_tokens(p, None, None, None, p, None, p, None, None, 2, 4, 1, 0, 64, 1e-5, None)
    assert rc == -1 and b"ncls=1 without cls" in lib.b200vit_last_error()   # gamma NULL passes the pointer check


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for sym in ("b200vit_patchify_spt_ln", "b200vit_attention_ex", "b200vit_attention_varlen_ex",
                "b200vit_encoder_blocks_ex"):
        assert f"int {sym}(" in h and sym in _lib.SYMBOLS
    assert "#define B200VIT_ATTN_MASK_SELF 1" in h and _lib.ATTN_MASK_SELF == 1
