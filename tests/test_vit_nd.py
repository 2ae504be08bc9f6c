"""The N-dimensional ViTs (vit_pytorch_b200.vit_nd / vit_nd_rotary) without a GPU: the shared rotary buffer, the eager
graph's hooks, and the argument checks of the new C entry points.  The reference-parity tests are in
test_family_parity.py."""
import ctypes
import sys

import pytest
import torch

from conftest import GOLDEN_DIR
from vit_pytorch_b200 import _lib, build
from vit_pytorch_b200.vit_nd_rotary import ViTND as RotaryViTND

sys.path.insert(0, GOLDEN_DIR)
from vit_nd_spec import FAMILY, INIT_KWARGS, VIT_ND_CASES  # noqa: E402


def test_rotary_buffer_is_shared_and_muon_parameters():
    kw = INIT_KWARGS
    m = RotaryViTND(**kw)
    sd = m.state_dict()
    depth = kw["depth"]
    keys = [k for k in sd if k.endswith("rotary_emb.freqs")]
    assert keys == ["rotary_emb.freqs"] + [f"transformer.layers.{i}.0.rotary_emb.freqs" for i in range(depth)]
    assert all(attn.rotary_emb is m.rotary_emb for attn, _ in m.transformer.layers)
    mp = m.muon_parameters()
    assert len(mp) == 4 * depth
    assert mp[0] is m.transformer.layers[0][0].to_v.weight and mp[1] is m.transformer.layers[0][0].to_out[0].weight


def test_eager_graph_keeps_hooks_observable():
    """Recorder-style hooks on the attention softmax fire on the PyTorch graph, once per layer."""
    spec = VIT_ND_CASES["rot_r2"]
    m = FAMILY.build(spec)
    seen = []
    for attn, _ in m.transformer.layers:
        attn.attend.register_forward_hook(lambda mod, i, o: seen.append(o.shape))
    with torch.inference_mode():
        m(FAMILY.input(spec).float())
    assert len(seen) == len(m.transformer.layers) and seen[0][-1] == seen[0][-2]


def test_positional_table_overflow_raises_like_the_reference():
    m = FAMILY.build(VIT_ND_CASES["nd_r2_cls"])
    big = torch.randn(1, 3, 32, 24)                       # more patches than the learned table holds
    with pytest.raises(RuntimeError):
        m(big)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def _ints(*v):
    return (ctypes.c_int * len(v))(*v)


def test_patchify_nd_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_patchify_nd(p, p, 64, 1, 3, 8, _ints(*[2] * 8), _ints(*[1] * 8), None)
    assert rc == -1 and b"rank 8" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_nd(p, p, 64, 1, 3, 0, _ints(1), _ints(1), None)
    assert rc == -1 and b"rank 0" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_nd(p, p, 64, 1, 3, 2, _ints(30, 32), _ints(4, 4), None)
    assert rc == -1 and b"not divisible" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_nd(p, p, 52, 1, 3, 2, _ints(32, 32), _ints(4, 4), None)
    assert rc == -1 and b"multiple of 8" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_nd(p, p, 40, 1, 3, 2, _ints(32, 32), _ints(4, 4), None)     # ldo < patch_dim 48
    assert rc == -1 and b"patch_dim" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_nd(p, ctypes.c_void_p(264), 64, 1, 3, 2, _ints(32, 32), _ints(4, 4), None)
    assert rc == -1 and b"misaligned" in lib.b200vit_last_error()
    rc = lib.b200vit_patchify_nd(None, p, 64, 1, 3, 2, _ints(32, 32), _ints(4, 4), None)
    assert rc == -1 and b"null" in lib.b200vit_last_error()


def test_rope_qk_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_rope_qk(p, p, 16, 16, 2, 96, None)
    assert rc == -1 and b"dim_head=96" in lib.b200vit_last_error()
    rc = lib.b200vit_rope_qk(p, p, 0, 16, 2, 64, None)
    assert rc == -1 and b"R=0" in lib.b200vit_last_error()
    rc = lib.b200vit_rope_qk(p, ctypes.c_void_p(260), 16, 16, 2, 64, None)
    assert rc == -1 and b"aligned" in lib.b200vit_last_error()
    rc = lib.b200vit_rope_qk(None, p, 16, 16, 2, 64, None)
    assert rc == -1 and b"null" in lib.b200vit_last_error()


def test_encoder_blocks_rope_rejects_bad_arguments(lib):
    layers = (_lib.Layer * 1)()
    full = _lib.EncoderWs(*([256] * 7))
    rc = lib.b200vit_encoder_blocks_rope(layers, 1, ctypes.c_void_p(256), ctypes.byref(full), 1, 16, 64, 1, 64, 128,
                                         0.125, 1, None, None, 0, ctypes.c_void_p(256), 0, None)
    assert rc == -1 and b"rope table" in lib.b200vit_last_error()
    rc = lib.b200vit_encoder_blocks_rope(layers, 1, ctypes.c_void_p(256), ctypes.byref(_lib.EncoderWs()), 1, 16, 64,
                                         1, 64, 128, 0.125, 1, None, None, 0, ctypes.c_void_p(256), 16, None)
    assert rc == -1 and b"workspace" in lib.b200vit_last_error()
