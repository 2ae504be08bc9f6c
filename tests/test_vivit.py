"""ViViT (vit_pytorch_b200.vivit) without a GPU: the attribute surface, the stored logits of a fully masked clip, the
state_dict round trip with the reference package, the eager graph's hooks, and the argument checks of the new C entry
points.  The reference-parity tests are in test_family_parity.py."""
import ctypes
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT, import_reference, load_golden, reference_available
from vit_pytorch_b200 import _lib, build
from vit_pytorch_b200.vivit import FactorizedTransformer, Transformer, ViViT

sys.path.insert(0, GOLDEN_DIR)
from vivit_spec import FAMILY, INIT_KWARGS, VARIANTS, VIVIT_CASES  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return load_golden("vivit")


@pytest.mark.parametrize("pool", ["cls", "mean"])
def test_attribute_surface(pool):
    fe = ViViT(variant="factorized_encoder", pool=pool, **INIT_KWARGS)
    fsa = ViViT(variant="factorized_self_attention", pool=pool, **INIT_KWARGS)
    assert fe.pos_embedding.shape == (1, 4, 6, INIT_KWARGS["dim"])
    assert fe.global_average_pool == (pool == "mean") and fe.variant == "factorized_encoder"
    for m in (fe, fsa):
        assert (m.spatial_cls_token is None) == (pool == "mean")
    assert (fe.temporal_cls_token is None) == (pool == "mean")
    assert isinstance(fe.spatial_transformer, Transformer) and isinstance(fsa.factorized_transformer,
                                                                          FactorizedTransformer)


def test_fully_masked_clip_modes_differ(golden):
    """The reference's two attention paths disagree on a clip whose frames are all masked (SDPA returns zeros, the
    masked_fill softmax averages every value); the stored logits keep both."""
    c = golden["cases"]
    for v in ("fe_mean", "fsa_cls", "fsa_mean"):
        a, b = c[f"{v}_sdpa"]["logits_fp32"]["full"][1], c[f"{v}_softmax"]["logits_fp32"]["full"][1]
        assert not torch.allclose(a, b, atol=1e-3)


@pytest.mark.skipif(not reference_available(), reason="reference package not installed (oracle/_ref)")
@pytest.mark.parametrize("variant", VARIANTS)
def test_state_dict_round_trip_with_reference(variant):
    ref_mod = import_reference()
    import importlib
    vivit_ref = importlib.import_module("vit_pytorch.vivit")
    torch.manual_seed(5)
    ref = vivit_ref.ViViT(variant=variant, **INIT_KWARGS).eval()
    ours = ViViT(variant=variant, **INIT_KWARGS).eval()
    ours.load_state_dict(ref.state_dict())
    ref.load_state_dict(ours.state_dict())
    x = torch.randn(2, 3, 8, 16, 24)
    mask = torch.ones(2, 8, dtype=torch.bool)
    mask[1, 2:] = False
    with torch.inference_mode():
        torch.testing.assert_close(ours(x, mask=mask), ref(x, mask=mask), rtol=0, atol=1e-5)
    assert ref_mod is not None


def test_eager_graph_keeps_hooks_observable():
    """Recorder-style hooks on the attention softmax fire on the PyTorch graph: spatial and temporal, every layer."""
    spec = VIVIT_CASES["fsa_cls_softmax"]
    m = FAMILY.build(spec)
    seen = []
    for sa, ta, _ in m.factorized_transformer.layers:
        for a in (sa, ta):
            a.attend.register_forward_hook(lambda mod, i, o: seen.append(tuple(o.shape)))
    with torch.inference_mode():
        m(FAMILY.input(spec).float())
    n, f = 6 + 1, 4
    assert seen[0] == (3 * f, 2, n, n) and seen[1] == (3 * n, 2, f, f) and len(seen) == 4


def test_direct_transformer_calls_take_masks():
    t = Transformer(32, 1, 2, 16, 64, use_flash_attn=False).eval()
    ft = FactorizedTransformer(32, 1, 2, 16, 64).eval()
    mask = torch.tensor([[True, True, False], [False, False, False]])
    with torch.inference_mode():
        assert t(torch.randn(2, 3, 32), mask).shape == (2, 3, 32)
        assert ft(torch.randn(2, 3, 5, 32), mask).shape == (2, 3, 5, 32)


def test_positional_table_overflow_raises_like_the_reference():
    m = FAMILY.build(VIVIT_CASES["fe_cls_sdpa"])
    with pytest.raises(RuntimeError):
        m(torch.randn(1, 3, 8, 32, 24))                   # more patches per frame than the table holds


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_attention_axial_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_attention_axial(p, p, None, 2, 8, 3, 2, 96, 0.1, 1, None)
    assert rc == -1 and b"dim_head=96 not supported by this build (32, 64, 80 or 128)" in lib.b200vit_last_error()
    rc = lib.b200vit_attention_axial(p, p, None, 2, 65, 3, 2, 64, 0.1, 1, None)
    assert rc == -1 and b"L=65 > 64" in lib.b200vit_last_error()
    rc = lib.b200vit_attention_axial(p, p, None, 0, 8, 3, 2, 64, 0.1, 1, None)
    assert rc == -1 and b"bad shape" in lib.b200vit_last_error()
    rc = lib.b200vit_attention_axial(p, ctypes.c_void_p(264), None, 2, 8, 3, 2, 64, 0.1, 1, None)
    assert rc == -1 and b"16-byte aligned" in lib.b200vit_last_error()
    rc = lib.b200vit_attention_axial(None, p, None, 2, 8, 3, 2, 64, 0.1, 0, None)
    assert rc == -1 and b"null" in lib.b200vit_last_error()


def test_embed_tokens_grouped_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    args = [p, p, p, None, p, None, p, None, None]
    rc = lib.b200vit_embed_tokens_grouped(*args, 4, 6, 0, 0, 64, 1e-5, 0, 6, 0, None)
    assert rc == -1 and b"positional period 0" in lib.b200vit_last_error()
    rc = lib.b200vit_embed_tokens_grouped(*args, 4, 6, 0, 0, 64, 1e-5, 2, -1, 0, None)
    assert rc == -1 and b"stride -1" in lib.b200vit_last_error()
    rc = lib.b200vit_embed_tokens_grouped(*args, 4, 6, 1, 0, 64, 1e-5, 2, 6, 0, None)
    assert rc == -1 and b"ncls=1 without cls" in lib.b200vit_last_error()
    rc = lib.b200vit_embed_tokens_grouped(*args, 0, 6, 0, 0, 64, 1e-5, 2, 6, 0, None)
    assert rc == -1 and b"bad shape" in lib.b200vit_last_error()


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for sym in ("b200vit_attention_axial", "b200vit_embed_tokens_grouped"):
        assert f"int {sym}(" in h and sym in _lib.SYMBOLS
