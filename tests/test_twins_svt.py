"""Twins-SVT (vit_pytorch_b200.twins_svt) without a GPU: the attribute surface, the fallback rules and that the eager
graph raises where the reference does, the prepared weights in fp32 (the permuted key / value convolution weight
against F.conv2d, the permuted patch-merge LayerNorm and GEMM against PatchEmbedding, the tap-major PEG weights), the
argument checks of the four entry points, and the launch sequence of the whole fused forward
(tests/golden/twins_svt_schedule.json, made by make_twins_svt_schedule.py).  The reference-parity tests are in
test_twins_svt_parity.py."""
import ctypes
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build, twins_svt as tw
from vit_pytorch_b200.engine import StridedKV, Windows, attention_kernel
from vit_pytorch_b200.twins_svt import PEG, PatchEmbedding, Transformer, TwinsSVT, merge_weights, peg_weights

sys.path.insert(0, GOLDEN_DIR)
from twins_svt_spec import INIT_KWARGS  # noqa: E402
import make_twins_svt_schedule as TS  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_attribute_surface():
    m = TwinsSVT(**INIT_KWARGS)
    kinds = [type(t).__name__ for t in m.layers]
    assert kinds == ["Sequential"] * 4 + ["AdaptiveAvgPool2d", "_Squeeze", "Linear"]
    assert [type(t).__name__ for t in m.layers[0]] == ["PatchEmbedding", "Transformer", "PEG", "Transformer"]
    assert not list(m.layers[5].parameters()) and m.layers[6].in_features == 40
    pe = m.layers[1][0]
    assert pe.proj[0].g.shape == (1, 64, 1, 1) and pe.proj[1].weight.shape == (24, 64, 1, 1)
    local, ff1, glob, ff2 = m.layers[0][1].layers[0]
    # 8 heads of 64 whatever the stage's width; to_q / to_kv without bias, to_out with one
    assert local.fn.to_q.weight.shape == (512, 16, 1, 1) and local.fn.to_q.bias is None
    assert glob.fn.to_kv.weight.shape == (1024, 16, 7, 7) and glob.fn.to_kv.bias is None and glob.fn.to_kv.stride == (7, 7)
    assert local.fn.to_out[0].bias.shape == (16,) and ff1.fn.net[1].weight.shape == (64, 16, 1, 1)
    last = m.layers[3][3]
    assert len(last.layers) == 2 and all(isinstance(l[0], torch.nn.Identity) and isinstance(l[1], torch.nn.Identity)
                                         for l in last.layers)
    assert m.layers[2][2].proj.fn.groups == 32 and m.layers[2][2].proj.fn.padding == (1, 1)
    keys = list(m.state_dict())
    assert keys[:4] == ["layers.0.0.proj.0.g", "layers.0.0.proj.0.b", "layers.0.0.proj.1.weight",
                        "layers.0.0.proj.1.bias"]
    assert keys[-2:] == ["layers.6.weight", "layers.6.bias"]
    assert "layers.3.3.layers.1.2.fn.to_kv.weight" in keys and not any(".layers.0.0.fn" in k for k in keys
                                                                       if k.startswith("layers.3."))


def test_encoder_layers_carry_window_and_strided_kv_records():
    t = Transformer(16, 2, local_patch_size=4, global_k=3).eval()
    layers, norm = t.encoder_layers()
    assert norm is None and [attention_kernel(L) for L in layers] == ["window", "kv", "window", "kv"]
    assert layers[0].attention == Windows(4) and layers[0].qkv_w.shape == (3 * 512, 16)
    assert isinstance(layers[1].attention, StridedKV) and layers[1].attention.stride == 3
    assert layers[1].qkv_w.shape == (512, 16) and layers[1].attention.kv_w.shape == (1024, 16, 3, 3)
    assert torch.equal(layers[0].qkv_w[512:], t.layers[0][0].fn.to_kv.weight.reshape(1024, 16))
    assert [attention_kernel(L) for L in Transformer(16, 1, has_local=False).encoder_layers()[0]] == ["kv"]
    with pytest.raises(ValueError):
        attention_kernel(layers[0], axial=True)
    with pytest.raises(ValueError):
        attention_kernel(layers[1], packed=True)


@pytest.fixture
def eligible(monkeypatch):
    """fused_reason with the device / dtype / autograd part passed, so its shape rules can be checked on CPU."""
    monkeypatch.setattr(tw, "common_reason", lambda *a, **k: None)


SMALL = dict(INIT_KWARGS, s1_local_patch_size=4, s1_global_k=2, s2_local_patch_size=2, s2_global_k=2,
             s3_local_patch_size=2, s3_global_k=1, s4_global_k=1)          # 32 x 32: 16 x 16 -> 8 x 8 -> 4 x 4 -> 2 x 2


def test_fused_reason_rules(eligible):
    m = TwinsSVT(**SMALL).eval()
    img = lambda h, w, c=3: torch.zeros(2, c, h, w)                      # noqa: E731
    assert m.fused_reason(img(32, 32)) is None and m.fused_reason(img(64, 32)) is None
    assert "not (B, 3, H, W)" in m.fused_reason(torch.zeros(3, 32, 32))
    assert "not (B, 3, H, W)" in m.fused_reason(img(32, 32, c=1))
    assert "stage 1" in m.fused_reason(img(33, 32)) and "patch_size=2" in m.fused_reason(img(33, 32))
    r = m.fused_reason(img(24, 32))                                        # 12 x 16 -> 6 x 8 -> 3 x 4
    assert "stage 3" in r and "local_patch_size=2" in r
    r = TwinsSVT(**dict(SMALL, s3_local_patch_size=1)).fused_reason(img(24, 32))
    assert "stage 4" in r and "patch_size=2" in r
    assert "local_patch_size=4" in m.fused_reason(img(36, 32))                                          # an 18 x 16 grid
    assert "smaller than global_k=5" in TwinsSVT(**dict(SMALL, s3_global_k=5)).fused_reason(img(32, 32))
    assert "is even" in TwinsSVT(**dict(SMALL, peg_kernel_size=4)).fused_reason(img(32, 32))
    assert "peg_kernel_size=9" in TwinsSVT(**dict(SMALL, peg_kernel_size=9)).fused_reason(img(32, 32))
    r = TwinsSVT(**dict(SMALL, s1_patch_size=1, s1_local_patch_size=9)).fused_reason(img(72, 72))
    assert "local_patch_size=9" in r and "81 tokens" in r
    assert "multiples of 8" in TwinsSVT(**dict(SMALL, s2_emb_dim=20)).fused_reason(img(32, 32))
    big = TwinsSVT(**dict(SMALL, s1_patch_size=1, s1_global_k=1))
    assert "sequence length 32768" in big.fused_reason(img(256, 128)) and big.fused_reason(img(128, 128)) is None


def test_fused_reason_on_cpu_input_and_dropout():
    assert "CUDA" in TwinsSVT(**SMALL).eval().fused_reason(torch.zeros(2, 3, 32, 32))
    assert "depth == 0" in TwinsSVT(**dict(SMALL, s2_depth=0)).eval().fused_reason(torch.zeros(2, 3, 32, 32))


@pytest.mark.parametrize("kw,hw", [({}, (33, 32)), ({}, (40, 32)), (dict(s3_global_k=5), (32, 32)),
                                   (dict(peg_kernel_size=4), (32, 32))])
def test_eager_graph_raises_where_the_reference_does(kw, hw):
    """An indivisible map (einops in the reference), a grid smaller than global_k (the convolution) and an even PEG
    kernel (the residual add) all raise a RuntimeError, in the reference too when it is installed."""
    from conftest import import_reference, reference_available
    mods = [TwinsSVT]
    if reference_available():
        import_reference()
        import importlib
        mods.append(importlib.import_module("vit_pytorch.twins_svt").TwinsSVT)
    for cls in mods:
        torch.manual_seed(0)
        m = cls(**dict(SMALL, **kw)).eval()
        with torch.inference_mode(), pytest.raises(RuntimeError):
            m(torch.randn(2, 3, *hw))


def _rounded(module):
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(torch.randn(p.shape).bfloat16().float() if p.dim() == 4 and p.shape[2] == 1 and p.shape[0] == 1
                    else p.bfloat16().float())
    return module.eval()


@pytest.mark.parametrize("p,hw,C", [(1, (3, 5), 8), (2, (4, 6), 8), (4, (8, 4), 3)])
def test_merge_weights_reproduce_the_module(p, hw, C):
    """The (p1 p2 c) merge, LayerNorm with the permuted affine and the permuted GEMM in fp32 torch give
    PatchEmbedding(x) up to its second LayerNorm."""
    torch.manual_seed(p * 10 + C)
    pe = _rounded(PatchEmbedding(dim=C, dim_out=16, patch_size=p))
    t = merge_weights(pe)
    K = C * p * p
    assert t["g"].shape == (K,) and t["w"].shape == (16, t["kp"]) and t["kp"] % 64 == 0
    assert (t["w"][:, K:] == 0).all()
    B, (h, w) = 2, hw
    x = torch.randn(B, C, h, w)
    with torch.no_grad():
        tokens = x.permute(0, 2, 3, 1)                                                   # b h w c
        merged = tokens.reshape(B, h // p, p, w // p, p, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, K)
        normed = F.layer_norm(merged, (K,), t["g"], t["b"], eps=1e-5)
        y = normed @ t["w"][:, :K].float().t() + t["bias"]
        got = F.layer_norm(y, (16,), t["g2"], t["b2"], eps=1e-5)
        want = pe(x).permute(0, 2, 3, 1).reshape(-1, 16)
    assert torch.allclose(got, want, atol=2e-5, rtol=1e-5), (got - want).abs().max()


@pytest.mark.parametrize("k,hw", [(1, (4, 4)), (2, (5, 7)), (3, (6, 6)), (7, (7, 9))])
def test_permuted_kv_weight_times_im2col_rows_is_the_convolution(k, hw):
    """The engine's prepared key / value weight applied to rows in b200vit_conv_im2col_nhwc's column order
    ((tap row, tap column, channel), stride k, no padding) equals F.conv2d with the module's weight."""
    torch.manual_seed(k)
    t = _rounded(Transformer(8, 1, global_k=k, has_local=False))
    prep = t.engine().prepared()
    w = prep["0.kv.w"].float()
    conv = t.layers[0][2].fn.to_kv
    assert w.shape == (1024, k * k * 8) and prep["0.qkv.w"].shape == (512, 8)
    h, wd = hw
    x = torch.randn(2, 8, h, wd).bfloat16().float()
    with torch.no_grad():
        tokens = x.permute(0, 2, 3, 1)
        oh, ow = h // k, wd // k
        rows = tokens[:, :oh * k, :ow * k].reshape(2, oh, k, ow, k, 8).permute(0, 1, 3, 2, 4, 5).reshape(-1, k * k * 8)
        got = rows @ w.t()
        want = conv(x).permute(0, 2, 3, 1).reshape(-1, 1024)
    assert torch.allclose(got, want, atol=1e-4, rtol=1e-5), (got - want).abs().max()


def test_peg_weights_are_tap_major():
    torch.manual_seed(3)
    peg = PEG(8, kernel_size=5).eval()
    t = peg_weights(peg)
    assert t["w"].shape == (25, 8) and t["b"].shape == (8,)
    assert torch.equal(t["w"][7], peg.proj.fn.weight[:, 0, 1, 2]) and torch.equal(t["b"], peg.proj.fn.bias)


# ------------------------------------------------------------------------------------------------ argument checks
def test_attention_window_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    def call(*, qkv=p, out=p, B=2, h=14, w=14, win=7, H=8, dh=64):
        rc = lib.b200vit_attention_window(qkv, out, B, h, w, win, H, dh, 0.125, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(qkv=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw in (dict(B=0), dict(h=0), dict(win=0), dict(H=0)):
        rc, msg = call(**kw)
        assert rc == -1 and b"bad shape" in msg, kw
    rc, msg = call(dh=48)
    assert rc == -1 and b"dim_head=48" in msg
    rc, msg = call(win=9, h=18, w=18)
    assert rc == -1 and b"81 tokens" in msg
    rc, msg = call(h=15)
    assert rc == -1 and b"not divisible" in msg
    rc, msg = call(out=ctypes.c_void_p(264))
    assert rc == -1 and b"16-byte aligned" in msg


def test_attention_kv_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    def call(*, q=p, ldq=512, kv=p, ldkv=1024, out=p, B=2, Nq=3136, Nk=64, H=8, dh=64):
        rc = lib.b200vit_attention_kv(q, ldq, kv, ldkv, out, B, Nq, Nk, H, dh, 0.125, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(q=None), dict(kv=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw in (dict(B=0), dict(Nq=0), dict(Nk=0), dict(H=0)):
        rc, msg = call(**kw)
        assert rc == -1 and b"bad shape" in msg, kw
    rc, msg = call(dh=48)
    assert rc == -1 and b"dim_head=48" in msg
    rc, msg = call(Nk=16385)
    assert rc == -1 and b"Nk=16385" in msg
    rc, msg = call(ldq=504)
    assert rc == -1 and b"ldq=504" in msg
    rc, msg = call(ldkv=1028)
    assert rc == -1 and b"ldkv=1028" in msg
    rc, msg = call(kv=ctypes.c_void_p(264))
    assert rc == -1 and b"16-byte aligned" in msg


def test_merge_patches_ln_and_peg_reject_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    def merge(*, x=p, M=2 * 56 * 56, g=p, b=p, out=p, ldo=256, B=2, h=56, w=56, C=64, win=2):
        rc = lib.b200vit_merge_patches_ln(x, M, g, b, out, ldo, B, h, w, C, win, 1e-5, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(x=None), dict(g=None), dict(b=None), dict(out=None)):
        rc, msg = merge(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(B=0), b"bad shape"), (dict(h=55), b"not divisible"), (dict(M=100), b"100 rows"),
                     (dict(C=62, ldo=248), b"multiple of 4"), (dict(ldo=248), b"ldo=248"), (dict(ldo=260), b"ldo=260"),
                     (dict(out=ctypes.c_void_p(264)), b"16-byte aligned")):
        rc, msg = merge(**kw)
        assert rc == -1 and what in msg, (kw, msg)

    def peg(*, x=p, M=2 * 49, w=p, b=p, y=ctypes.c_void_p(512), B=2, gh=7, gw=7, C=512, k=3):
        rc = lib.b200vit_peg(x, M, w, b, y, B, gh, gw, C, k, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(x=None), dict(w=None), dict(b=None), dict(y=None)):
        rc, msg = peg(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(B=0), b"bad shape"), (dict(k=4), b"kernel size 4"), (dict(k=9), b"kernel size 9"),
                     (dict(M=99), b"99 rows"), (dict(C=510), b"multiple of 4"), (dict(y=p), b"must not be x"),
                     (dict(y=ctypes.c_void_p(520)), b"16-byte aligned")):
        rc, msg = peg(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in ("b200vit_attention_window", "b200vit_attention_kv", "b200vit_merge_patches_ln", "b200vit_peg"):
        assert f"int {name}(" in h and name in _lib.SYMBOLS


# ------------------------------------------------------------------------------------------------ launch sequence
@pytest.fixture(scope="module")
def schedule():
    with open(TS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [TS.run_name(m, h) for m, h in TS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", TS.RUNS)
def test_fused_forward_schedule_matches_fixture(lib, schedule, ln_mode, host_loop):
    name = TS.run_name(ln_mode, host_loop)
    got, want = TS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
def test_global_sub_block_sequence(lib, ln_mode):
    """The sub-sampled-key sub-block is the same in both LayerNorm modes: layernorm into the bf16 rows, the query GEMM
    on them into the q columns of the qkv buffer, conv_im2col_nhwc of them (none for k = 1), the key / value GEMM,
    attention_kv, then the out-projection with the residual."""
    calls = TS.record(ln_mode, "python")
    names = [c["call"] for c in calls]
    assert names[:3] == ["patchify_ln", "gemm", "embed_tokens"] and names[-3:] == ["mean_pool", "cast_f32_bf16", "gemm"]
    assert names.count("merge_patches_ln") == 3 and names.count("peg") == 4
    assert names.count("attention_window") == 2 + 3 + 2 and names.count("attention_kv") == 2 + 3 + 2 + 2
    kv = [i for i, n in enumerate(names) if n == "attention_kv"]
    for i in kv:
        a = calls[i]
        j = i - 1
        assert calls[j]["call"] == "gemm" and calls[j]["out_bf16"] == a["kv"] and calls[j]["w"]["key"].endswith(".kv.w")
        if calls[j - 1]["call"] == "conv_im2col_nhwc":
            assert calls[j - 1]["out_bf16"] == calls[j]["a"] and calls[j - 1]["k"] == calls[j - 1]["s"] > 1
            j -= 1
        q, ln = calls[j - 1], calls[j - 2]
        assert q["call"] == "gemm" and q["out_bf16"] == a["q"] and q["out_bf16"]["stride"][0] == 3 * 512
        assert ln["call"] == "layernorm" and ln["out_bf16"] == q["a"] and ln["out_bf16"]["role"].endswith(".ws.xn")
        out = calls[i + 1]
        assert out["call"] == "gemm" and out["a"] == a["out"] and out["resid"] is not None
    assert sum(calls[i - 2]["call"] == "conv_im2col_nhwc" for i in kv) == 2 + 3       # stages 1 and 2 (k 3 and 2)
