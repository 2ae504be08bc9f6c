"""MobileViT (vit_pytorch_b200.mobile_vit) without a GPU: the module surface, that the eager graph raises where the
reference does, the fallback rules, the engine description of the README config, the BatchNorm folds against
convolution + BatchNorm in fp64, the kernel's group address map against the module's rearrangement, the argument checks
of the new entry points, and the launch sequence of the whole fused forward (tests/golden/mobile_vit_schedule.json, made
by make_mobile_vit_schedule.py).  The reference-parity tests are in test_mobile_vit_parity.py."""
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build, mobile_vit as mvit
from vit_pytorch_b200.engine import PatchGroups, attention_kernel
from vit_pytorch_b200.mobile_vit import MobileViT, conv_bn_weights, from_groups, to_groups

sys.path.insert(0, GOLDEN_DIR)
from mobile_vit_spec import SMALL  # noqa: E402
import make_engine_schedule as S  # noqa: E402
import make_mobile_vit_schedule as MS  # noqa: E402

README = dict(image_size=(256, 256), dims=[96, 120, 144], channels=[16, 32, 48, 48, 64, 64, 80, 80, 96, 96, 384],
              num_classes=1000)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def small(**kw):
    torch.manual_seed(0)
    return MobileViT(**dict(SMALL, image_size=(64, 64), **kw)).eval()


# ------------------------------------------------------------------------------------------------ surface
def test_module_surface():
    for name in ("conv_1x1_bn", "conv_nxn_bn", "FeedForward", "Attention", "Transformer", "MV2Block",
                 "MobileViTBlock", "MobileViT"):
        assert hasattr(mvit, name), name
    m = small()
    names = [n for n, _ in m.named_parameters()]
    assert names[0] == "conv1.0.weight" and names[-1] == "to_logits.2.weight"
    assert m.stem[3].conv[0].in_channels == SMALL["channels"][2]
    assert m.to_logits[2].bias is None


def test_eager_graph_raises_where_the_reference_does():
    m = small()
    with torch.inference_mode():
        assert m(torch.randn(1, 3, 64, 64)).shape == (1, 7)
        with pytest.raises(RuntimeError, match="not divisible"):
            m(torch.randn(1, 3, 96, 64))               # 96 -> blocks 12, 6, 3: 3 is odd
    with pytest.raises(RuntimeError):
        with torch.inference_mode():
            small(kernel_size=5)(torch.randn(1, 3, 64, 64))
    bad = dict(SMALL, image_size=(64, 64), channels=[16, 16, 24, 32, 32, 32, 40, 40, 48, 48, 96])
    with pytest.raises(RuntimeError):
        with torch.inference_mode():
            MobileViT(**bad).eval()(torch.randn(1, 3, 64, 64))


@pytest.mark.parametrize("ph,pw,h,w", [(2, 2, 8, 8), (2, 4, 16, 32), (1, 1, 13, 9), (4, 2, 8, 6)])
def test_group_address_map_reproduces_the_rearrangement(ph, pw, h, w):
    """Token t of group (b, i, j) in the module's rearrangement is map row (b*h + y'*ph + i)*w + x'*pw + j."""
    B, d = 2, 3
    x = torch.arange(B * d * h * w, dtype=torch.float64).reshape(B, d, h, w)
    g = to_groups(x, ph, pw)                                          # b, (ph pw), (h w), d
    rows = x.permute(0, 2, 3, 1).reshape(B * h * w, d)
    hh, ww = h // ph, w // pw
    for b in range(B):
        for i in range(ph):
            for j in range(pw):
                for t in range(hh * ww):
                    y, xx = divmod(t, ww)
                    assert torch.equal(g[b, i * pw + j, t], rows[(b * h + y * ph + i) * w + xx * pw + j])
    assert torch.equal(from_groups(g, hh, ww, ph, pw), x)


# ------------------------------------------------------------------------------------------------ fused_reason
def test_fused_reason_rules():
    x = torch.zeros(2, 3, 64, 64, dtype=torch.bfloat16)
    m = small().bfloat16()
    assert m.fused_reason(x) == "input is not on a CUDA device"
    # shape rules, checked without a device: the common checks pass once they are stubbed
    orig = mvit.common_reason
    try:
        mvit.common_reason = lambda *a, **k: None
        assert m.fused_reason(x) is None
        assert "(B, 3, H, W)" in m.fused_reason(torch.zeros(2, 1, 64, 64))
        assert "not divisible" in m.fused_reason(torch.zeros(2, 3, 96, 64))
        assert "tokens per group" in small(patch_size=(1, 1)).bfloat16().fused_reason(
            torch.zeros(1, 3, 1040, 512))
        assert "kernel_size=5" in small(kernel_size=5).bfloat16().fused_reason(x)
        assert "channels[2]" in MobileViT(**dict(SMALL, image_size=(64, 64), channels=[
            16, 16, 24, 32, 32, 32, 40, 40, 48, 48, 96])).eval().fused_reason(x)
        assert "multiples of 8" in MobileViT(**dict(SMALL, image_size=(64, 64), channels=[
            16, 16, 24, 24, 36, 36, 40, 40, 48, 48, 96])).eval().fused_reason(x)
        assert "multiples of 8" in small(expansion=1.5).fused_reason(x)
        assert "to_logits" in MobileViT(**dict(SMALL, image_size=(64, 64), channels=[
            16, 16, 24, 24, 32, 32, 40, 40, 48, 48, 100])).eval().fused_reason(x)
        assert "multiples of 8" in MobileViT(**dict(SMALL, image_size=(64, 64), dims=(36, 40, 48))).eval() \
            .fused_reason(x)
        bn = small()
        bn.trunk[1][1].conv3[1].train()
        assert "BatchNorm2d" in bn.fused_reason(x)
    finally:
        mvit.common_reason = orig


def test_fused_reason_hooks(monkeypatch):
    m = small()
    monkeypatch.setattr(mvit, "batchnorm_reason", lambda mod: None)
    h = m.trunk[0][1].transformer.layers[0][0].to_qkv.register_forward_hook(lambda *a: None)
    import vit_pytorch_b200.engine as E
    monkeypatch.setattr(E, "why_not_fused", lambda *a, **k: None)
    assert "hooks" in m.fused_reason(torch.zeros(2, 3, 64, 64))
    h.remove()


# ------------------------------------------------------------------------------------------------ engine description
def test_patch_group_records_of_the_readme_config():
    torch.manual_seed(0)
    m = MobileViT(**README).eval()
    for (_, blk), depth, dim, mlp in zip(m.trunk, (2, 4, 3), (96, 120, 144), (192, 480, 576)):
        layers, norm = blk.transformer.encoder_layers()
        assert norm is None and len(layers) == depth
        for L in layers:
            assert (L.heads, L.dim_head, L.ff_act, L.attention) == (4, 8, "silu", PatchGroups())
            assert L.scale == 8 ** -0.5 and L.qkv_w.shape == (96, dim) and L.fc1_w.shape == (mlp, dim)
            assert attention_kernel(L) == "groups"
            with pytest.raises(ValueError):
                attention_kernel(L, axial=True)
        assert (blk.ph, blk.pw) == (2, 2)
        eng = blk.transformer.engine()
        assert eng.unsupported_reason(256, grid=(16, 16), groups=(2, 2)) is None
        assert eng.prepared()["c_layers"] is None                 # the per-kernel loop
    assert m.block_maps(256, 256) == [(32, 32), (16, 16), (8, 8)]


# ------------------------------------------------------------------------------------------------ BatchNorm folds
def _perturb(m):
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.weight.add_(0.5 * torch.randn(mod.weight.shape, generator=g))
                mod.bias.add_(0.1 * torch.randn(mod.bias.shape, generator=g))
                mod.running_mean.add_(0.2 * torch.randn(mod.running_mean.shape, generator=g))
                mod.running_var.mul_(0.5 + torch.rand(mod.running_var.shape, generator=g))


def _check_fold(conv, bn, w, b, rel, channels_last=True):
    """The folded (w, b) of conv + bn, applied as a convolution in fp64, against bn(conv(x)) in fp64: within `rel` of
    the magnitude sum (the rounding of the folded weights; the fold itself is exact algebra)."""
    g = torch.Generator().manual_seed(conv.out_channels)
    x = torch.randn(2, conv.in_channels, 9, 7, dtype=torch.float64, generator=g)
    kh, kw = conv.kernel_size
    cin = conv.in_channels // conv.groups
    if w.shape[0] == conv.out_channels and w.shape[1] >= cin * kh * kw:           # a GEMM weight [out, K (padded)]
        w = w.double()[:, :cin * kh * kw]
        w = (w.reshape(-1, kh, kw, cin).permute(0, 3, 1, 2) if channels_last else w.reshape(-1, cin, kh, kw))
    else:                                                                          # depthwise, tap-major [9, C]
        w = w.double().t().reshape(-1, 1, kh, kw)
    kw_ = dict(stride=conv.stride, padding=conv.padding, groups=conv.groups)
    with torch.no_grad():
        want = bn(conv(x))
        got = torch.nn.functional.conv2d(x, w, b.double(), **kw_)
        mag = torch.nn.functional.conv2d(x.abs(), w.abs(), b.double().abs(), **kw_)
    assert ((got - want).abs() <= rel * mag + 1e-12).all()


@pytest.mark.parametrize("expansion", [1, 2])
def test_folded_batchnorms_reproduce_conv_and_batchnorm_in_fp64(expansion):
    """Every BatchNorm fold of the prepared weights, conv by conv: bf16 GEMM weights within half a bf16 ulp (2^-8
    relative, with the fp32 bias), the fp32 depthwise taps within a few fp32 ulps."""
    m = small(expansion=expansion).double()
    _perturb(m)
    t = m._build()
    bf, f32 = 2.0 ** -8, 2.0 ** -20
    _check_fold(m.conv1[0], m.conv1[1], t["conv1.w"], t["conv1.b"], bf, channels_last=False)
    for name, mv2 in [(f"stem{i}.", v) for i, v in enumerate(m.stem)] + \
            [(f"trunk{i}.", v) for i, (v, _) in enumerate(m.trunk)]:
        c = mv2.conv
        if expansion != 1:
            _check_fold(c[0], c[1], t[name + "w1"], t[name + "b1"], bf)
            dw, bn2, pw, bn3 = c[3], c[4], c[6], c[7]
        else:
            assert name + "w1" not in t
            dw, bn2, pw, bn3 = c[0], c[1], c[3], c[4]
        _check_fold(dw, bn2, t[name + "w9"], t[name + "b9"], f32)
        _check_fold(pw, bn3, t[name + "w3"], t[name + "b3"], bf)
    for i, (_, blk) in enumerate(m.trunk):
        for j, conv in enumerate((blk.conv1, blk.conv2, blk.conv3, blk.conv4), 1):
            _check_fold(conv[0], conv[1], t[f"block{i}.c{j}.w"], t[f"block{i}.c{j}.b"], bf)
    _check_fold(m.to_logits[0][0], m.to_logits[0][1], t["head.w"], t["head.b"], bf)


def test_conv_bn_weights_column_orders():
    conv = torch.nn.Conv2d(8, 16, 3, 1, 1, bias=False).double()
    bn = torch.nn.BatchNorm2d(16).double().eval()
    _perturb(torch.nn.Sequential(bn))
    x = torch.randn(1, 8, 5, 6, dtype=torch.float64)
    with torch.no_grad():
        want = bn(conv(x))
        for cl in (False, True):
            w, b = conv_bn_weights(conv, bn, channels_last=cl)
            assert w.dtype == torch.bfloat16 and w.shape == (16, 72)
            wf = w.double().reshape(16, 3, 3, 8).permute(0, 3, 1, 2) if cl else w.double().reshape(16, 8, 3, 3)
            got = torch.nn.functional.conv2d(x, wf, b.double(), padding=1)
            assert (got - want).abs().max().item() < 2e-2 * want.abs().max().item()


# ------------------------------------------------------------------------------------------------ argument checks
def test_attention_groups_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)

    def call(*, qkv=p, out=p, B=2, gh=8, gw=8, ph=2, pw=2, H=4, dh=8):
        rc = lib.b200vit_attention_groups(qkv, out, B, gh, gw, ph, pw, H, dh, 0.35, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(qkv=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(dh=16), b"dim_head=16"), (dict(dh=32), b"dim_head=32"), (dict(B=0), b"bad shape"),
                     (dict(H=0), b"bad shape"), (dict(ph=0), b"bad shape"), (dict(gh=7), b"not divisible"),
                     (dict(gw=9), b"not divisible"), (dict(gh=128, gw=64, ph=1, pw=1), b"tokens per group"),
                     (dict(H=65536), b"exceeds the grid"), (dict(out=ctypes.c_void_p(264)), b"16-byte aligned")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_mbconv_dwconv_ex_rejects_bad_arguments(lib):
    p, q = ctypes.c_void_p(256), ctypes.c_void_p(4096)

    def call(*, x=p, M=2 * 9 * 11, w9=p, bias=p, y=q, part=None, B=2, h=9, w=11, C=64, stride=2, act=_lib.EPI_SILU):
        rc = lib.b200vit_mbconv_dwconv_ex(x, M, w9, bias, y, part, B, h, w, C, stride, act, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(x=None), dict(w9=None), dict(bias=None), dict(y=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(act=_lib.EPI_SIGMOID), b"act="), (dict(act=0), b"act="), (dict(stride=3), b"stride=3"),
                     (dict(C=60), b"C=60"), (dict(y=p), b"must not be x"), (dict(M=100), b"100 rows")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)
    # the plain entry point still requires the channel sums
    rc = lib.b200vit_mbconv_dwconv(p, 2 * 9 * 11, p, p, q, None, 2, 9, 11, 64, 2, None)
    assert rc == -1 and b"null" in lib.b200vit_last_error()


def test_conv_im2col_nhwc_ex_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)

    def call(*, x=p, ldx=64, M=2 * 9 * 11, out=p, ldo=288, B=2, H=9, W=11, C=32):
        rc = lib.b200vit_conv_im2col_nhwc_ex(x, ldx, M, out, ldo, B, H, W, C, 3, 1, 1, None)
        return rc, lib.b200vit_last_error()
    assert call(x=None)[0] == -1 and b"null" in call(x=None)[1]
    for kw, what in ((dict(ldx=16), b"ldx=16"), (dict(ldx=36), b"ldx=36"), (dict(M=100), b"100 rows"),
                     (dict(x=ctypes.c_void_p(264)), b"16-byte aligned"), (dict(ldo=100), b"ldo=100")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_gemm_act_binding_rejects_other_activations():
    with pytest.raises(_lib.B200VitError, match="act="):
        _lib.gemm_act(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16),
                      act="sigmoid", out_bf16=torch.zeros(8, 8, dtype=torch.bfloat16))


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in ("attention_groups", "mbconv_dwconv_ex", "conv_im2col_nhwc_ex"):
        assert f"int b200vit_{name}(" in h and f"b200vit_{name}" in _lib.SYMBOLS
    assert f"#define B200VIT_ATTN_GROUPS_MAX_TOKENS {_lib.ATTN_GROUPS_MAX_TOKENS}" in h


def test_library_exports_the_new_entry_points(lib):
    for name in ("b200vit_attention_groups", "b200vit_mbconv_dwconv_ex", "b200vit_conv_im2col_nhwc_ex"):
        assert hasattr(lib, name)


# ------------------------------------------------------------------------------------------------ launch sequence
@pytest.fixture(scope="module")
def schedule():
    with open(MS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [MS.run_name(m, h) for m, h in MS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", MS.RUNS)
def test_fused_forward_schedule_matches_fixture(lib, schedule, ln_mode, host_loop):
    name = MS.run_name(ln_mode, host_loop)
    got, want = MS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"


@pytest.mark.parametrize("ln_mode,host_loop", MS.RUNS)
def test_group_attention_and_depthwise_launches(lib, ln_mode, host_loop):
    calls = MS.record(ln_mode, host_loop)
    names = [c["call"] for c in calls]
    assert names[:2] == ["conv_im2col_nchw", "gemm_act"]
    assert names[-4:] == ["gemm_act", "mean_pool", "cast_f32_bf16", "gemm"]
    att = [c for c in calls if c["call"] == "attention_groups"]
    assert [(c["gh"], c["gw"], c["ph"], c["pw"]) for c in att] == [(8, 8, 2, 2), (4, 4, 2, 2), (2, 2, 2, 2)]
    assert names.count("mbconv_dwconv_ex") == 7
    # every feed-forward fc1 takes SiLU, never GELU
    assert not any(c.get("gelu") for c in calls)
    assert sum(c["call"] == "gemm_act" and c["ln_sums"] is not None for c in calls) == (3 if ln_mode == "fold" else 0)
    # each block's concatenation: the MV2Block's projection writes its right half and conv3 its left half, once each;
    # conv1's im2col reads the right half in place and conv4's im2col the whole buffer
    cats = [c["x"] for c in calls if c["call"] == "conv_im2col_nhwc" and c["x"]["offset"] == 0]
    assert len(cats) == 3
    for cat in cats:
        role, half = cat["role"], cat["shape"][1] // 2
        writes = [(c["call"], c["out_bf16"]["offset"]) for c in calls
                  if isinstance(c.get("out_bf16"), dict) and c["out_bf16"].get("role") == role]
        assert writes == [("gemm", 2 * half), ("gemm_act", 0)], writes
        reads = [c["x"]["offset"] for c in calls if c["call"] == "conv_im2col_nhwc" and c["x"]["role"] == role]
        assert reads == [2 * half, 0]


def test_other_families_schedule_fixtures_are_unchanged(lib):
    """Every other family's pinned launch sequence, regenerated, is byte-identical to its fixture."""
    for mod in ("make_engine_schedule", "make_cct_schedule", "make_pit_schedule", "make_levit_schedule",
                "make_twins_svt_schedule", "make_max_vit_schedule", "make_cvt_schedule",
                "make_crossformer_schedule"):
        g = importlib.import_module(mod)
        with open(g.FIXTURE) as f:
            assert S.dumps(g.generate()) == f.read(), mod
