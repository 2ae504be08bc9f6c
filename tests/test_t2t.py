"""T2T-ViT without a GPU: the fused dataflow of t2t.py (the padded soft-split weights and widths, the layer schedule of
soft_split_layer, the int(sqrt(n)) maps) emulated in fp64 against the module's own PyTorch graph, the dispatch rules,
the argument checks of the new C ABI entry points (every call below fails its checks before it touches a device) and
the header declaring them."""
import ctypes
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR
from vit_pytorch_b200 import _lib, build
from vit_pytorch_b200.pit import pool_grid
from vit_pytorch_b200.t2t import T2TViT, round8, soft_split_width, split_weights

sys.path.insert(0, GOLDEN_DIR)
from t2t_spec import FAMILY, T2T_CASES  # noqa: E402

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200vit.h")
NEW = ("b200vit_t2t_unfold_image", "b200vit_t2t_unfold_tokens", "b200vit_attention_wide",
       "b200vit_attention_wide_workspace")


def _layernorm(x, ln):
    g, b, eps = ln
    return F.layer_norm(x, (x.shape[-1],), g.double(), b.double(), eps)


def emulate(model: T2TViT, img: torch.Tensor) -> torch.Tensor:
    """forward_fused's dataflow in fp64: padded buffers, the prepared (padded) weights, attention at width dp."""
    B = img.shape[0]
    geo = model.stage_geometry(img.shape[2], img.shape[3])
    src, width = img.double(), img.shape[1]
    for i, ((k, s), t, (h, w_, oh, ow)) in enumerate(zip(model.t2t_layers, model.soft_splits(), geo)):
        w, n = width * k * k, oh * ow
        if i > 0:
            src = src[:, :width].reshape(B, h, w_, width).permute(0, 3, 1, 2)
        x = torch.zeros(B * n, round8(w), dtype=torch.float64)
        x[:, :w] = F.unfold(src, k, padding=s // 2, stride=s).transpose(1, 2).reshape(B * n, w)
        if t is not None:
            p = split_weights(t)
            dp = p["dp"]
            xa = _layernorm(x[:, :w], p["ln1"])
            qkv = xa @ p["qkv"].double()[:, :w].t()
            q, kk, v = qkv.view(B, n, 3, dp).unbind(2)
            assert (qkv.view(B * n, 3, dp)[:, :, w:] == 0).all()       # the padding is zero
            a = torch.softmax(q @ kk.transpose(1, 2) * p["scale"], -1) @ v
            o = a.reshape(B * n, dp)
            assert (o[:, w:] == 0).all()
            x[:, :w] += (o[:, :w] @ p["eye"].double()[:, :w].t())[:, :w] if dp <= 160 else o[:, :w]
            h1 = F.gelu(_layernorm(x[:, :w], p["ln2"]) @ p["w1"].double()[:, :w].t() + p["b1"].double())
            assert (h1[:, w:] == 0).all()
            x += h1[:, :w] @ p["w2"].double()[:, :w].t() + p["b2"].double()
            assert (x[:, w:] == 0).all()                                # the stream's padding stays zero
            src = _layernorm(x[:, :w], p["norm"])
        else:
            src = x
        width = w
    lin = model.to_patch_embedding[-1]
    y = src[:, :width] @ lin.weight.double().t() + lin.bias.double()
    tok = torch.cat([model.cls_token.double().expand(B, -1, -1), y.view(B, n, -1)], 1)
    tok = tok + model.pos_embedding.double()[:, :n + 1]
    out = model.transformer.double()(tok)
    pooled = out.mean(1) if model.pool == 'mean' else out[:, 0]
    return model.mlp_head.double()(pooled)


@pytest.mark.parametrize("name", ["pool_mean", "channels1", "two_stage", "k3_small", "isqrt_4x16", "smaller_input"])
def test_fused_dataflow_in_fp64_matches_the_module(name):
    spec = T2T_CASES[name]
    m = FAMILY.build(spec).double()
    x = FAMILY.input(spec).double()
    with torch.inference_mode():
        want = m.forward_eager(x)
        got = emulate(m, x)
    torch.testing.assert_close(got, want, rtol=1e-9, atol=1e-9)


def test_soft_split_widths():
    assert [soft_split_width(w) for w in (9, 27, 49, 64, 81, 128, 147, 160)] == [32, 32, 64, 64, 128, 128, 160, 160]
    assert [soft_split_width(w) for w in (161, 243, 441, 1323)] == [192, 256, 448, 1344]


def test_stage_geometry_follows_the_reference():
    m = T2TViT(image_size=224, num_classes=3, dim=32, depth=1, heads=1, mlp_dim=32)
    assert m.stage_geometry(224, 224) == [(224, 224, 56, 56), (56, 56, 28, 28), (28, 28, 14, 14)]
    # a 4 x 16 first map is read as 8 x 8
    assert m.stage_geometry(16, 64)[1] == (8, 8, 4, 4)
    # 5 tokens cannot be read as a map of 2 rows: einops raises, so does the module
    assert m.stage_geometry(20, 20) is not None and pool_grid(5) is None and pool_grid(20) == (4, 5)


def test_dispatch_reasons_on_cpu():
    m = T2TViT(image_size=32, num_classes=3, dim=32, depth=1, heads=1, mlp_dim=32).eval()
    assert m.fused_reason(torch.zeros(1, 3, 32, 32)) == "input is not on a CUDA device"
    assert m.fused_reason(torch.zeros(3, 32, 32)) == "input is not (B, C, H, W)"
    assert "channel count" in m.fused_reason(torch.zeros(1, 1, 32, 32))
    other = T2TViT(image_size=32, num_classes=3, dim=32, transformer=torch.nn.Identity())
    assert "transformer=" in other.fused_reason(torch.zeros(1, 3, 32, 32))


def test_padded_weights():
    m = T2TViT(image_size=32, num_classes=3, dim=32, depth=1, heads=1, mlp_dim=32)
    p = split_weights(m.to_patch_embedding[3])
    w = 147
    assert p["dp"] == 160 and p["qkv"].shape == (480, 152) and p["w1"].shape == (152, 152)
    wq = m.to_patch_embedding[3].layers[0][0].to_qkv.weight.bfloat16()
    for j in range(3):
        assert torch.equal(p["qkv"][160 * j:160 * j + w, :w], wq[w * j:w * (j + 1)])
        assert (p["qkv"][160 * j + w:160 * (j + 1)] == 0).all()
    assert (p["qkv"][:, w:] == 0).all() and (p["w2"][w:] == 0).all() and (p["b2"][w:] == 0).all()
    assert p["scale"] == w ** -0.5


# ---------------------------------------------------------------------------------------------------- C ABI
P_ = ctypes.c_void_p
GOOD = P_(256)        # 16-byte aligned, never dereferenced: the calls fail their argument checks first
ODD = P_(258)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def _err(lib) -> str:
    return lib.b200vit_last_error().decode()


def test_header_declares_the_new_entry_points():
    text = open(HEADER).read()
    for s in NEW:
        assert f"{s}(" in text and s in _lib.SYMBOLS, s
    assert "B200VIT_ATTN_WIDE_MAX_TOKENS 1024" in text and "B200VIT_ATTN_WIDE_MAX_WIDTH 4096" in text


def test_library_exports_them(lib):
    for s in NEW:
        assert hasattr(lib, s), s


def test_unfold_argument_checks(lib):
    img = lib.b200vit_t2t_unfold_image
    assert img(GOOD, GOOD, GOOD, 152, 1, 3, 32, 32, 7, 4, 2, None) == -1
    assert "exactly one of" in _err(lib)
    assert img(GOOD, GOOD, None, 148, 1, 3, 32, 32, 7, 4, 2, None) == -1
    assert "ldo=148 must be a multiple of 8" in _err(lib)
    assert img(GOOD, GOOD, None, 144, 1, 3, 32, 32, 7, 4, 2, None) == -1
    assert ">= C*k*k=147" in _err(lib)
    assert img(GOOD, GOOD, None, 152, 1, 3, 32, 32, 3, 8, 4, None) == -1
    assert "bad shape" in _err(lib)
    assert img(GOOD, GOOD, None, 152, 1, 3, 2, 2, 7, 4, 2, None) == -1
    assert "smaller than one 7 x 7 window" in _err(lib)
    assert img(GOOD, ODD, None, 152, 1, 3, 32, 32, 7, 4, 2, None) == -1
    assert "16-byte aligned" in _err(lib)
    tok = lib.b200vit_t2t_unfold_tokens
    assert tok(GOOD, 152, 2, 5, 147, GOOD, None, 1328, 3, 2, 1, None) == -1
    assert "5 tokens cannot be read as a map of 2 rows" in _err(lib)
    assert tok(GOOD, 100, 2, 64, 147, GOOD, None, 1328, 3, 2, 1, None) == -1
    assert "ldx=100 < C=147" in _err(lib)
    assert tok(GOOD, 152, 2, 64, 147, GOOD, None, 1320, 3, 2, 1, None) == -1
    assert ">= C*k*k=1323" in _err(lib)


def test_wide_attention_argument_checks(lib):
    wide = lib.b200vit_attention_wide
    ws = _lib.attention_wide_workspace(784, 1344, 1)
    assert ws > 784 * 784 * 4
    assert wide(GOOD, GOOD, None, 0, 0, 2, 1025, 1344, 0.03, GOOD, ws, None) == -1
    assert "n=1025 tokens per image (1 .. 1024)" in _err(lib)
    assert wide(GOOD, GOOD, None, 0, 0, 2, 784, 1330, 0.03, GOOD, ws, None) == -1
    assert "multiple of 64" in _err(lib)
    assert wide(GOOD, GOOD, None, 0, 0, 2, 784, 4160, 0.03, GOOD, ws, None) == -1
    assert "<= 4096" in _err(lib)
    assert wide(GOOD, GOOD, GOOD, 1328, 1345, 2, 784, 1344, 0.03, GOOD, ws, None) == -1
    assert "n_resid=1345" in _err(lib)
    assert wide(GOOD, ODD, None, 0, 0, 2, 784, 1344, 0.03, GOOD, ws, None) == -1
    assert "16-byte aligned" in _err(lib)
    assert wide(GOOD, GOOD, None, 0, 0, 2, 784, 1344, 0.03, GOOD, ws - 1024, None) == -1
    assert "holds no image" in _err(lib)
    assert wide(GOOD, None, None, 0, 0, 2, 784, 1344, 0.03, GOOD, ws, None) == -1
    assert "null pointer" in _err(lib)


def test_varlen_takes_dh_160_without_self_masking(lib):
    assert lib.b200vit_attention_varlen(ODD, GOOD, GOOD, GOOD, 1, 16, 1, 1, 160, 0.1, None) == -1
    assert "16-byte aligned" in _err(lib) and "dim_head" not in _err(lib)
    assert lib.b200vit_attention_varlen_ex(GOOD, GOOD, GOOD, GOOD, 1, 16, 1, 1, 160, 0.1, _lib.ATTN_MASK_SELF,
                                           None) == -1
    assert "dim_head=160" in _err(lib)
    assert lib.b200vit_attention(GOOD, GOOD, 1, 16, 1, 160, 0.1, None) == -1
    assert "dim_head=160" in _err(lib)


# ---------------------------------------------------------------------------------------------------- launch sequence
import json  # noqa: E402

import make_t2t_schedule as TS  # noqa: E402


@pytest.fixture(scope="module")
def schedule():
    with open(TS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [TS.run_name(m, h) for m, h in TS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", TS.RUNS)
def test_fused_forward_schedule_matches_fixture(lib, schedule, ln_mode, host_loop):
    """Every launch of T2TViT.forward_fused, recorded on CPU: its entry point, its scalars, the buffer (and offset,
    shape, stride) of every tensor and the digest of every prepared weight, against tests/golden/t2t_schedule.json."""
    name = TS.run_name(ln_mode, host_loop)
    got, want = TS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
def test_soft_split_launch_lists(lib, ln_mode):
    """The narrow soft split runs the key-block attention and the identity to_out as a residual GEMM; the wide one
    runs b200vit_attention_wide, whose epilogue adds into the stream; every soft-split GEMM reads K = w."""
    names = [c["call"] for c in TS.record(ln_mode, "python")]
    layer = ["layernorm", "gemm", "attention_varlen", "gemm", "layernorm", "gemm", "gemm", "layernorm"]
    wide = ["layernorm", "gemm", "attention_wide", "layernorm", "gemm", "gemm", "layernorm"]
    assert names[:17] == ["t2t_unfold_image"] + layer + ["t2t_unfold_tokens"] + wide
    assert names[17:20] == ["t2t_unfold_tokens", "gemm", "embed_tokens"]
    calls = TS.record(ln_mode, "python")
    assert [c["k"] for c in calls[:17] if c["call"] == "gemm"] == [27] * 4 + [243] * 3
    assert calls[12]["n_resid"] == 243 and calls[12]["dp"] == 256 and calls[12]["x"]["role"] == calls[9]["out"]["role"]
    assert calls[18]["k"] == 2187
