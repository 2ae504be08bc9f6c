"""LeViT (vit_pytorch_b200.levit) without a GPU: the attribute and state_dict surface, the BatchNorm folding in fp64,
the bias table and the kernel's coordinate-based index against the module's pos_indices buffer, the fallback rules and
that the eager graph raises where the reference does, the argument checks of b200vit_attention_posbias and of the
Hardswish GEMM flag, and the launch sequence of the whole fused forward (tests/golden/levit_schedule.json, made by
make_levit_schedule.py).  The reference-parity tests are in test_levit_parity.py."""
import ctypes
import json
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build, levit as lv
from vit_pytorch_b200.levit import Attention, LeViT, attention_weights, bias_table, fold_bn

sys.path.insert(0, GOLDEN_DIR)
from levit_spec import INIT_KWARGS, SMALL  # noqa: E402
import make_levit_schedule as LS  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_attribute_surface():
    m = LeViT(**INIT_KWARGS)
    assert [type(t).__name__ for t in m.backbone] == ["Transformer"] * 5
    assert [t.attn_residual for t in m.backbone] == [True, False, True, False, True]
    ds = m.backbone[1].layers[0][0]
    assert ds.heads == 4 and ds.to_q[0].stride == (2, 2) and ds.to_out[1].out_channels == 48
    assert ds.pos_bias.weight.shape == (16, 4) and ds.pos_indices.shape == (4, 16)
    keys = list(m.state_dict())
    assert keys[:2] == ["conv_embedding.0.weight", "conv_embedding.0.bias"]
    assert keys[-4:] == ["distill_head.weight", "distill_head.bias", "mlp_head.weight", "mlp_head.bias"]
    assert "backbone.0.layers.0.0.pos_indices" in keys and "backbone.0.layers.0.0.to_q.1.running_var" in keys
    assert m.backbone[1].layers[0][1].net[0].out_channels == 96                # mlp_mult 2 of dim_out 48
    assert LeViT(**SMALL, image_size=64).distill_head(torch.zeros(1)) is None


def test_to_out_batchnorm_starts_at_zero():
    a = Attention(16, 4)
    assert torch.equal(a.to_out[2].weight.detach(), torch.zeros(16))


def _perturbed_bn(bn, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        bn.weight.copy_(torch.randn(bn.weight.shape, generator=g))
        bn.bias.copy_(torch.randn(bn.bias.shape, generator=g))
        bn.running_mean.copy_(torch.randn(bn.running_mean.shape, generator=g))
        bn.running_var.copy_(0.2 + torch.rand(bn.running_var.shape, generator=g))
    return bn.eval()


@pytest.mark.parametrize("which", ["to_q", "to_k", "to_v", "to_out"])
def test_folded_batchnorm_reproduces_the_module_in_fp64(which):
    torch.manual_seed(3)
    a = Attention(16, 4, heads=2, dim_key=16, dim_value=32).double().eval()
    seq = getattr(a, which)
    conv, bn = (seq[1], seq[2]) if which == "to_out" else (seq[0], seq[1])
    _perturbed_bn(bn, 7)
    x = torch.randn(2, conv.in_channels, 4, 4, dtype=torch.float64)
    w, b = fold_bn(conv.weight, conv.bias, bn)
    with torch.no_grad():
        want = bn(conv(x))
        # fold_bn computes in fp32 (what the kernels get); in fp64 the same formula is exact up to rounding
        got = torch.einsum("oc,bchw->bohw", w.double(), x) + b.double()[None, :, None, None]
    assert torch.allclose(got, want, atol=1e-5, rtol=1e-5), (got - want).abs().max()


def test_prepared_qkv_rows_are_q_k_v():
    torch.manual_seed(4)
    m = LeViT(**dict(SMALL, image_size=64)).eval()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            _perturbed_bn(mod, 11)
    a, ff = m.backbone[1].layers[0]
    t = attention_weights(a, ff)
    x = torch.randn(2, 32, 4, 4)
    with torch.no_grad():
        tokens = x.permute(0, 2, 3, 1).reshape(-1, 32)
        got = tokens @ t["qkv.w"].float().t() + t["qkv.b"]
        full = torch.cat([torch.nn.functional.conv2d(x, s[0].weight) for s in (a.to_q, a.to_k, a.to_v)], 1)
        bns = [s[1] for s in (a.to_q, a.to_k, a.to_v)]
        want = torch.cat([bn(full[:, o:o + bn.num_features]) for bn, o in
                          zip(bns, (0, bns[0].num_features, 2 * bns[0].num_features))], 1)
        want = want.permute(0, 2, 3, 1).reshape(-1, want.shape[1])
    assert t["qkv.w"].shape == (2 * 4 * 32 + 4 * 64, 32)
    assert torch.allclose(got, want, atol=3e-2, rtol=3e-2)       # the bf16-rounded folded rows


@pytest.mark.parametrize("F,downsample", [(1, False), (4, False), (7, False), (7, True), (14, True), (5, True),
                                          (32, False)])
def test_bias_table_and_coordinate_index_reproduce_pos_indices(F, downsample):
    """The kernel's index |s i - ky| * F + |s j - kx| into bias_table (= pos_bias.weight^T / scale) gives the module's
    pos_bias(pos_indices) / scale for every (query, key, head)."""
    torch.manual_seed(F)
    a = Attention(16, F, heads=3, dim_key=32, downsample=downsample)
    s = 2 if downsample else 1
    Fq = -(-F // s)
    n = torch.arange(Fq * Fq)
    qy, qx = s * (n // Fq), s * (n % Fq)
    m = torch.arange(F * F)
    ky, kx = m // F, m % F
    idx = (qy[:, None] - ky[None, :]).abs() * F + (qx[:, None] - kx[None, :]).abs()
    assert torch.equal(idx, a.pos_indices)
    t = bias_table(a)
    assert t.shape == (3, F * F)
    want = a.pos_bias(a.pos_indices).permute(2, 0, 1) / a.scale
    assert torch.allclose(t[:, idx], want.detach(), rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------------ fallback rules
@pytest.fixture
def eligible(monkeypatch):
    """fused_reason with the device / dtype / autograd part passed, so its shape rules can be checked on CPU."""
    monkeypatch.setattr(lv, "common_reason", lambda *a, **k: None)


def test_fused_reason_rules(eligible):
    m = LeViT(**dict(SMALL, image_size=64)).eval()
    img = lambda h, w, c=3: torch.zeros(2, c, h, w)                      # noqa: E731
    assert m.fused_reason(img(64, 64)) is None and m.fused_reason(img(61, 57)) is None       # both give 4 x 4
    assert "not (B, 3, H, W)" in m.fused_reason(torch.zeros(3, 64, 64))
    assert "not (B, 3, H, W)" in m.fused_reason(img(64, 64, c=1))
    assert "5 x 4 grid" in m.fused_reason(img(72, 64))
    assert "dim_key=48" in LeViT(**dict(SMALL, image_size=64, dim_key=48)).eval().fused_reason(img(64, 64))
    assert "dim_value=16" in LeViT(**dict(SMALL, image_size=64, dim_value=16)).eval().fused_reason(img(64, 64))
    big = LeViT(**dict(SMALL, image_size=1040)).eval()                  # 65 x 65 = 4225 keys
    assert "4225 keys" in big.fused_reason(img(1040, 1040))
    assert "multiples of 8" in LeViT(**dict(SMALL, image_size=64, dim=(32, 44, 64))).eval().fused_reason(img(64, 64))
    assert "36 -> 64 channels" in LeViT(**dict(SMALL, image_size=64, dim=(36, 48, 64))).eval().fused_reason(img(64, 64))
    t = LeViT(**dict(SMALL, image_size=64))
    t.train()
    assert "BatchNorm2d is in training mode" in t.fused_reason(img(64, 64))
    t.eval()
    t.backbone[0].layers[0][0].to_k[1].running_var = None
    assert "no running statistics" in t.fused_reason(img(64, 64))


def test_fused_reason_on_cpu_input_and_depth_zero():
    assert "CUDA" in LeViT(**dict(SMALL, image_size=64)).eval().fused_reason(torch.zeros(2, 3, 64, 64))
    m = LeViT(**dict(SMALL, image_size=64, depth=(1, 0, 1))).eval()
    assert "depth == 0" in m.fused_reason(torch.zeros(2, 3, 64, 64))


@pytest.mark.parametrize("image_size,hw", [(200, (200, 200)), (64, (80, 64)), (224, (256, 256))])
def test_eager_graph_raises_where_the_reference_does(image_size, hw):
    """A conv grid other than image_size // 16 square fails the bias add, in the reference too when it is
    installed."""
    from conftest import import_reference, reference_available
    mods = [LeViT]
    if reference_available():
        import_reference()
        import importlib
        mods.append(importlib.import_module("vit_pytorch.levit").LeViT)
    for cls in mods:
        torch.manual_seed(0)
        m = cls(**dict(SMALL, image_size=image_size)).eval()
        with torch.inference_mode(), pytest.raises(RuntimeError):
            m(torch.randn(1, 3, *hw))


# ------------------------------------------------------------------------------------------------ argument checks
def test_attention_posbias_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)

    def call(*, qkv=p, ld=2 * 4 * 32 + 4 * 64, out=p, table=p, B=2, F=14, s=1, H=4, dk=32, dv=64, flags=4):
        rc = lib.b200vit_attention_posbias(qkv, ld, out, table, B, F, s, H, dk, dv, 0.17, flags, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(qkv=None), dict(out=None), dict(table=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(B=0), b"bad shape"), (dict(F=0), b"bad shape"), (dict(H=0), b"bad shape"),
                     (dict(s=3), b"s=3"), (dict(dk=48), b"dim_key=48"), (dict(dk=128), b"dim_key=128"),
                     (dict(dv=16), b"dim_value=16"), (dict(dv=80), b"dim_value=80"), (dict(F=65), b"4225 keys"),
                     (dict(ld=504), b"ld=504"), (dict(ld=516), b"ld=516"), (dict(flags=1), b"unknown flags"),
                     (dict(flags=8), b"unknown flags"), (dict(out=ctypes.c_void_p(264)), b"16-byte aligned"),
                     (dict(table=ctypes.c_void_p(260)), b"16-byte aligned"), (dict(B=65536), b"exceed the grid")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_other_attention_entry_points_reject_gelu_out(lib):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_attention_ex(p, p, 2, 64, 4, 64, 0.125, _lib.ATTN_GELU_OUT, None)
    assert rc == -1 and b"unknown flags" in lib.b200vit_last_error()


def test_gemm_rejects_gelu_with_hardswish(lib):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_gemm_bf16(p, 64, p, 64, p, None, 64, None, None, None, 0, 1e-5, None, None, 64, 64, 64,
                               _lib.EPI_GELU | _lib.EPI_HARDSWISH, None)
    assert rc == -1 and b"exclusive" in lib.b200vit_last_error()


def test_header_declares_the_new_entry_point_and_flags():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    assert "int b200vit_attention_posbias(" in h and "b200vit_attention_posbias" in _lib.SYMBOLS
    assert "#define B200VIT_EPI_HARDSWISH 32" in h and "#define B200VIT_ATTN_GELU_OUT 4" in h
    assert f"#define B200VIT_ATTN_POSBIAS_MAX_KEYS {_lib.ATTN_POSBIAS_MAX_KEYS}" in h


# ------------------------------------------------------------------------------------------------ launch sequence
@pytest.fixture(scope="module")
def schedule():
    with open(LS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [LS.run_name(m, h) for m, h in LS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", LS.RUNS)
def test_fused_forward_schedule_matches_fixture(lib, schedule, ln_mode, host_loop):
    name = LS.run_name(ln_mode, host_loop)
    got, want = LS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"


def test_both_layernorm_settings_give_one_sequence(schedule):
    a, b = (schedule[LS.run_name(m, h)] for m, h in LS.RUNS)
    assert a == b


def test_five_launches_per_layer(lib):
    calls = LS.record("fold", "python")
    names = [c["call"] for c in calls]
    assert names[:8] == ["conv_im2col_nchw", "gemm"] + ["conv_im2col_nhwc", "gemm"] * 3
    assert names[-3:] == ["mean_pool", "cast_f32_bf16", "gemm"]
    layers = names[8:-3]
    assert layers == ["gemm", "attention_posbias", "gemm", "gemm_hardswish", "gemm"] * 6
    att = [c for c in calls if c["call"] == "attention_posbias"]
    assert [(c["F"], c["s"], c["H"]) for c in att] == [(7, 1, 2), (7, 2, 4), (4, 1, 3), (4, 1, 3), (4, 2, 6),
                                                      (2, 1, 4)]
    assert all(c["gelu_out"] for c in att)
    # the downsampling layers' to_out GEMM starts a fresh stream (no residual); every other to_out GEMM adds it
    outs = [calls[i + 1] for i, c in enumerate(calls) if c["call"] == "attention_posbias"]
    assert [o["resid"] is None for o in outs] == [False, True, False, False, True, False]
    head = calls[-1]
    assert head["w"]["key"] == "head.w" and head["w"]["shape"][0] == 5 + 3
