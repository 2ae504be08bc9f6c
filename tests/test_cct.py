"""CCT (vit_pytorch_b200.cct) without a GPU: the sine table and presets, the fallback rules, the prepared conv-weight
layout, the argument checks of the im2col, ReLU max-pool and sequence-pooling entry points, the post-norm layer's
schedule and the launch sequence of the whole fused forward (tests/golden/cct_schedule.json, made by
make_cct_schedule.py).  The reference-parity tests are in test_family_parity.py."""
import ctypes
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build, cct as cct_mod
from vit_pytorch_b200.cct import CCT, conv_weights, sinusoidal_embedding

sys.path.insert(0, GOLDEN_DIR)
import make_cct_schedule as CS  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_sine_table_and_presets():
    t = sinusoidal_embedding(5, 8)
    assert t.shape == (1, 5, 8) and t.dtype == torch.float32
    assert torch.equal(t[0, 0], torch.tensor([0., 1.] * 4))
    m = cct_mod.cct_7(img_size=32, num_classes=10, n_conv_layers=1)
    conv = m.tokenizer.conv_layers[0][0]
    assert conv.kernel_size == (3, 3) and conv.stride == (1, 1) and conv.padding == (1, 1)
    assert len(m.classifier.blocks) == 7 and m.classifier.embedding_dim == 256
    assert m.classifier.sequence_length == 256 and m.classifier.blocks[0].linear1.out_features == 512


@pytest.fixture
def eligible(monkeypatch):
    """fused_reason with the device / dtype / autograd part passed, so its shape rules can be checked on CPU."""
    monkeypatch.setattr(cct_mod, "common_reason", lambda *a, **k: None)


KW = dict(img_size=32, embedding_dim=64, n_conv_layers=1, kernel_size=3, stride=1, padding=1, num_layers=1,
          num_heads=1, num_classes=3)


def test_fused_reason_rules(eligible):
    img = lambda c, h, w: torch.zeros(2, c, h, w)                       # noqa: E731
    m = CCT(**KW).eval()
    assert m.fused_reason(img(3, 32, 32)) is None
    assert "not (B, C, H, W)" in m.fused_reason(torch.zeros(3, 32, 32))
    assert "channel count" in m.fused_reason(img(1, 32, 32))
    assert "positional table" in m.fused_reason(img(3, 36, 32))          # sine / learnable: n must equal the table
    assert "positional table" in CCT(**{**KW, "positional_embedding": "learnable"}).fused_reason(img(3, 30, 32))
    none = CCT(**{**KW, "positional_embedding": "none"}).eval()
    assert none.fused_reason(img(3, 40, 40)) is None                    # more tokens than sequence_length: fused
    assert "fewer than sequence_length" in none.fused_reason(img(3, 24, 32))
    assert "not divisible" in CCT(**{**KW, "num_heads": 5, "embedding_dim": 72}).fused_reason(img(3, 32, 32))
    assert "dim_head=48" in CCT(**{**KW, "num_heads": 2, "embedding_dim": 96}).fused_reason(img(3, 32, 32))
    assert "multiples of 8" in CCT(**{**KW, "mlp_ratio": 1.1}).fused_reason(img(3, 32, 32))
    assert "kernel 17" in CCT(**{**KW, "kernel_size": 17, "padding": 8}).fused_reason(img(3, 32, 32))
    assert "padding 3" in CCT(**{**KW, "padding": 3}).fused_reason(img(3, 32, 32))
    assert "MaxPool2d" in CCT(**{**KW, "pooling_kernel_size": 20, "pooling_padding": 0}).fused_reason(img(3, 64, 64))
    assert "embedding_dim=1088" in CCT(**{**KW, "embedding_dim": 1088, "num_heads": 17}).fused_reason(img(3, 32, 32))
    assert "num_layers == 0" in CCT(**{**KW, "num_layers": 0}).fused_reason(img(3, 32, 32))
    big = CCT(**{**KW, "img_size": 264, "pooling_stride": 1}).eval()     # 264 x 264 tokens
    assert "16384" in big.fused_reason(img(3, 264, 264))


def test_fused_reason_on_cpu_input_and_training():
    m = CCT(**KW).eval()
    assert "CUDA" in m.fused_reason(torch.zeros(2, 3, 32, 32))
    r = cct_mod.common_reason(m.train(), torch.zeros(2, 3, 32, 32), dropout_p=m.classifier.dropout_p)
    assert r is not None
    assert m.classifier.dropout_p == 0.1                  # attention_dropout and stochastic_depth_rate count too


def test_reference_errors_are_reproduced():
    """A table whose length differs from the token count raises in the eager graph, as the reference's add does; with
    'none' a shorter sequence raises (the reference pads to an attribute it never sets)."""
    m = CCT(**KW).eval()
    with torch.inference_mode(), pytest.raises(RuntimeError):
        m(torch.randn(2, 3, 36, 32))
    none = CCT(**{**KW, "positional_embedding": "none"}).eval()
    with torch.inference_mode(), pytest.raises(AttributeError):
        none(torch.randn(2, 3, 24, 32))
    with torch.inference_mode():
        assert none(torch.randn(2, 3, 40, 40)).shape == (2, 3)


@pytest.mark.parametrize("k,s,p,C", [(3, 1, 1, 3), (7, 2, 3, 3), (1, 1, 0, 8), (5, 3, 2, 16)])
def test_conv_weights_reproduce_the_convolution(k, s, p, C):
    """The prepared weight times an fp32 im2col of either column order gives Conv2d's output."""
    torch.manual_seed(k * 10 + s)
    conv = torch.nn.Conv2d(C, 16, k, s, p, bias=False)
    with torch.no_grad():
        conv.weight.copy_(conv.weight.bfloat16().float())
    x = torch.randn(2, C, 13, 11)
    want = conv(x).permute(0, 2, 3, 1).reshape(-1, 16)
    oh, ow = (13 + 2 * p - k) // s + 1, (11 + 2 * p - k) // s + 1
    # (cin, ky, kx): F.unfold
    w0 = conv_weights(conv, False).float()
    K = C * k * k
    assert w0.shape == (16, (K + 7) // 8 * 8) and (w0[:, K:] == 0).all()
    a0 = F.unfold(x, k, padding=p, stride=s).transpose(1, 2).reshape(-1, K)
    assert torch.allclose(a0 @ w0[:, :K].t(), want, atol=1e-4, rtol=1e-4)
    # (ky, kx, cin): the channels-last gather
    w1 = conv_weights(conv, True).float()
    a1 = F.unfold(x, k, padding=p, stride=s).reshape(2, C, k * k, oh * ow).permute(0, 3, 2, 1).reshape(-1, K)
    assert torch.allclose(a1 @ w1[:, :K].t(), want, atol=1e-4, rtol=1e-4)


def test_classifier_describes_post_norm_layers():
    m = CCT(**{**KW, "num_layers": 2, "num_heads": 2})
    layers, norm = m.classifier.encoder_layers()
    assert len(layers) == 2 and all(L.post_norm for L in layers)
    blk = m.classifier.blocks[1]
    L = layers[1]
    assert L.ln2.gamma is blk.norm1.weight and L.ln1.gamma is blk.pre_norm.weight
    assert L.qkv_w is blk.self_attn.qkv.weight and L.out_b is blk.self_attn.proj.bias
    assert L.heads == 2 and L.dim_head == 32 and L.scale == 32 ** -0.5 and norm.gamma is m.classifier.norm.weight
    assert m.classifier.engine().prepared()["c_layers"] is None       # the per-kernel loop runs them


# ------------------------------------------------------------------------------------------------ argument checks
def _err(lib):
    return lib.b200vit_last_error()


def test_conv_im2col_nchw_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    def call(*, img=p, out=p, ldo=152, B=2, C=3, H=32, W=32, k=7, s=2, pad=3):
        return lib.b200vit_conv_im2col_nchw(img, out, ldo, B, C, H, W, k, s, pad, None), _err(lib)
    for kw in (dict(img=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw in (dict(k=0), dict(k=17, pad=3), dict(s=0), dict(pad=-1), dict(pad=7), dict(H=0), dict(B=0), dict(C=0),
               dict(H=2, pad=1, k=5)):
        rc, msg = call(**kw)
        assert rc == -1 and b"bad shape" in msg, kw
    rc, msg = call(ldo=144)
    assert rc == -1 and b"ldo=144" in msg
    rc, msg = call(ldo=150)
    assert rc == -1 and b"multiple of 8" in msg
    rc, msg = call(out=ctypes.c_void_p(264))
    assert rc == -1 and b"16-byte aligned" in msg


def test_conv_im2col_nhwc_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    def call(*, x=p, M=2 * 28 * 56, out=p, ldo=3136, B=2, H=28, W=56, C=64, k=7, s=2, pad=3):
        return lib.b200vit_conv_im2col_nhwc(x, M, out, ldo, B, H, W, C, k, s, pad, None), _err(lib)
    for kw in (dict(x=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw in (dict(k=0), dict(s=0), dict(pad=7), dict(W=0), dict(B=0)):
        rc, msg = call(**kw)
        assert rc == -1 and b"bad shape" in msg, kw
    rc, msg = call(C=60, ldo=2944)
    assert rc == -1 and b"multiple of 8" in msg
    rc, msg = call(M=100)
    assert rc == -1 and b"100 rows" in msg
    rc, msg = call(ldo=3128)
    assert rc == -1 and b"ldo=3128" in msg
    for kw in (dict(x=ctypes.c_void_p(264)), dict(out=ctypes.c_void_p(264))):
        rc, msg = call(**kw)
        assert rc == -1 and b"16-byte aligned" in msg, kw


def test_relu_maxpool_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    def call(*, y=p, M=2 * 16 * 16, B=2, H=16, W=16, C=64, pk=3, ps=2, pp=1, ob=p, of=None, ldo=64):
        return lib.b200vit_relu_maxpool(y, M, B, H, W, C, pk, ps, pp, ob, of, ldo, None), _err(lib)
    for kw in (dict(y=None), dict(ob=None), dict(of=p)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw in (dict(pk=0), dict(pk=17), dict(ps=0), dict(pp=2), dict(H=0), dict(H=1, pp=0)):
        rc, msg = call(**kw)
        assert rc == -1 and b"bad shape" in msg, kw
    rc, msg = call(C=12, ldo=16)
    assert rc == -1 and b"multiple of 8" in msg
    rc, msg = call(M=5)
    assert rc == -1 and b"5 rows" in msg
    rc, msg = call(ldo=60)
    assert rc == -1 and b"ldo=60" in msg
    rc, msg = call(ob=None, of=p, ldo=66)
    assert rc == -1 and b"multiple of 4" in msg
    for kw in (dict(y=ctypes.c_void_p(264)), dict(ob=ctypes.c_void_p(264))):
        rc, msg = call(**kw)
        assert rc == -1 and b"16-byte aligned" in msg, kw


def test_seq_pool_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    def call(*, x=p, B=2, n=256, D=256, g=p, b=p, w=p, bias=p, out=p, ldo=256):
        return lib.b200vit_seq_pool(x, B, n, D, g, b, 1e-5, w, bias, out, ldo, None), _err(lib)
    for kw in (dict(x=None), dict(g=None), dict(b=None), dict(w=None), dict(bias=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw in (dict(B=0), dict(n=0), dict(D=0)):
        rc, msg = call(**kw)
        assert rc == -1 and b"bad shape" in msg, kw
    for kw in (dict(D=260, ldo=264), dict(D=1032, ldo=1032)):
        rc, msg = call(**kw)
        assert rc == -1 and b"multiple of 8 and <= 1024" in msg, kw
    rc, msg = call(B=70000)
    assert rc == -1 and b"too many" in msg
    rc, msg = call(ldo=248)
    assert rc == -1 and b"ldo=248" in msg
    for kw in (dict(x=ctypes.c_void_p(264)), dict(out=ctypes.c_void_p(264)), dict(w=ctypes.c_void_p(264))):
        rc, msg = call(**kw)
        assert rc == -1 and b"16-byte aligned" in msg, kw


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in ("b200vit_conv_im2col_nchw", "b200vit_conv_im2col_nhwc", "b200vit_relu_maxpool", "b200vit_seq_pool"):
        assert f"int {name}(" in h and name in _lib.SYMBOLS
    for name, value in (("CONV_MAX_KERNEL", cct_mod.CONV_MAX_KERNEL), ("POOL_MAX_KERNEL", cct_mod.POOL_MAX_KERNEL),
                        ("SEQ_POOL_MAX_DIM", cct_mod.SEQ_POOL_MAX_DIM)):
        assert f"#define B200VIT_{name} {value} " in h


# ------------------------------------------------------------------------------------------------ launch sequence
@pytest.fixture(scope="module")
def schedule():
    with open(CS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [CS.run_name(m, h) for m, h in CS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", CS.RUNS)
def test_fused_forward_schedule_matches_fixture(lib, schedule, ln_mode, host_loop):
    name = CS.run_name(ln_mode, host_loop)
    got, want = CS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
def test_post_norm_layer_sequence(lib, ln_mode):
    """After the out-projection (which writes no bf16 copy): layernorm into ws.y and ws.xn, the plain fc1 GEMM on
    ws.xn, and fc2 onto ws.y written to the stream; fold mode adds the copy and statistics the next QKV reads."""
    calls = CS.record(ln_mode, "python")
    names = [c["call"] for c in calls]
    assert names[:7] == ["conv_im2col_nchw", "gemm", "relu_maxpool", "conv_im2col_nhwc", "gemm", "relu_maxpool",
                         "embed_tokens"]
    assert names[-2:] == ["seq_pool", "gemm"]
    lns = [i for i, c in enumerate(calls) if c["call"] == "layernorm" and c["out_f32"] is not None]
    assert len(lns) == 2
    for i in lns:
        out, ln, fc1, fc2 = calls[i - 1], calls[i], calls[i + 1], calls[i + 2]
        assert out["out_bf16"] is None and out["stats_out"] is None
        assert ln["out_f32"]["role"] == "ws.y" and ln["out_bf16"]["role"] == "ws.xn" and ln["x"] == out["out_f32"]
        assert fc1["a"]["role"] == "ws.xn" and fc1["gelu"] and fc1["ln_sums"] is None
        assert fc1["w"]["key"].endswith("fc1.w")
        assert fc2["resid"]["role"] == "ws.y" and fc2["out_f32"] == ln["x"]
        assert (fc2["stats_out"] is not None) == (ln_mode == "fold")
    seq = calls[-2]
    assert seq["x"] == calls[lns[-1] + 2]["out_f32"] and calls[-1]["a"] == seq["out_bf16"]
