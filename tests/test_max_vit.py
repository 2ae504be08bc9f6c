"""MaxViT (vit_pytorch_b200.max_vit) without a GPU: the attribute and state_dict surface, the three BatchNorm folds of
an MBConv in fp64, the kernel's block and grid address maps and bias index against the module's rearrangements and
rel_pos_indices buffer, the fallback rules and that the eager graph raises where the reference does, the argument
checks of the new entry points and GEMM flags, and the launch sequence of the whole fused forward
(tests/golden/max_vit_schedule.json, made by make_max_vit_schedule.py).  The reference-parity tests are in
test_max_vit_parity.py."""
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build, max_vit as mv
from vit_pytorch_b200.max_vit import Attention, MaxViT, MBConv, MBConvResidual, mbconv_weights

sys.path.insert(0, GOLDEN_DIR)
from max_vit_spec import INIT_KWARGS, SMALL  # noqa: E402
import make_engine_schedule as S  # noqa: E402
import make_max_vit_schedule as MS  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_attribute_surface():
    m = MaxViT(**INIT_KWARGS)
    assert len(m.layers) == 3
    assert [isinstance(b[0], MBConvResidual) for b in m.layers] == [False, True, False]
    a = m.layers[0][2].fn
    assert isinstance(a, Attention) and a.heads == 1 and a.rel_pos_bias.weight.shape == (9, 1)
    assert a.rel_pos_indices.shape == (4, 4)
    keys = list(m.state_dict())
    assert keys[:4] == ["conv_stem.0.weight", "conv_stem.0.bias", "conv_stem.1.weight", "conv_stem.1.bias"]
    assert keys[-4:] == ["mlp_head.1.weight", "mlp_head.1.bias", "mlp_head.2.weight", "mlp_head.2.bias"]
    assert "layers.0.2.fn.rel_pos_bias.weight" in keys and "layers.1.0.fn.6.gate.3.weight" in keys
    assert "layers.0.0.4.running_var" in keys and "layers.0.6.fn.to_out.0.weight" in keys
    assert not any(k.endswith("rel_pos_indices") for k in keys)          # a non-persistent buffer
    assert m.layers[0][0][6].gate[1].weight.shape == (32, 128)          # hidden 4 * 32, squeeze 0.25


def test_seeded_init_is_deterministic():
    torch.manual_seed(5)
    a = MaxViT(**SMALL).state_dict()
    torch.manual_seed(5)
    b = MaxViT(**SMALL).state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


def _perturbed_bn(bn, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        bn.weight.copy_(torch.randn(bn.weight.shape, generator=g))
        bn.bias.copy_(torch.randn(bn.bias.shape, generator=g))
        bn.running_mean.copy_(torch.randn(bn.running_mean.shape, generator=g))
        bn.running_var.copy_(0.2 + torch.rand(bn.running_var.shape, generator=g))
    return bn.eval()


@pytest.mark.parametrize("which", ["expand", "depthwise", "project"])
@pytest.mark.parametrize("downsample", [False, True])
def test_folded_batchnorms_reproduce_the_module_in_fp64(which, downsample):
    torch.manual_seed(3)
    mb = MBConv(16, 16, downsample=downsample, expansion_rate=2).double().eval()
    net = mb.fn if isinstance(mb, MBConvResidual) else mb
    for i, bn in enumerate((net[1], net[4], net[8])):
        _perturbed_bn(bn, 7 + i)
    t = mbconv_weights(mb)
    s = 2 if downsample else 1
    with torch.no_grad():
        if which == "expand":
            x = torch.randn(2, 16, 5, 7, dtype=torch.float64)
            want = net[1](net[0](x))
            got = torch.einsum("oc,bchw->bohw", t["w1"].double(), x) + t["b1"].double()[None, :, None, None]
            tol = 3e-2                                             # the bf16-rounded folded rows
        elif which == "depthwise":
            x = torch.randn(2, 32, 5, 7, dtype=torch.float64)
            want = net[4](net[3](x))
            w = t["w9"].double().t().reshape(32, 1, 3, 3)
            got = torch.nn.functional.conv2d(x, w, t["b9"].double(), stride=s, padding=1, groups=32)
            tol = 1e-5                                             # fp32, what b200vit_mbconv_dwconv gets
        else:
            x = torch.randn(2, 32, 5, 7, dtype=torch.float64)
            want = net[8](net[7](x))
            got = torch.einsum("oc,bchw->bohw", t["w3"].double(), x) + t["b3"].double()[None, :, None, None]
            tol = 3e-2
    assert torch.allclose(got, want, atol=tol, rtol=tol), (got - want).abs().max()
    assert t["w9"].shape == (9, 32) and t["se1"].shape == (8, 32) and t["se2"].shape == (32, 8)


# ------------------------------------------------------------------------------------------------ address maps
def kernel_rows(B, gh, gw, w, grid):
    """b200vit_attention_window_relpos's map: [windows, w*w] map rows, window (b, i, j), local token r = u*w + v."""
    X, Y = gh // w, gw // w
    b, i, j, u, v = torch.meshgrid(torch.arange(B), torch.arange(X), torch.arange(Y), torch.arange(w),
                                   torch.arange(w), indexing="ij")
    y = u * X + i if grid else i * w + u
    x = v * Y + j if grid else j * w + v
    return ((b * gh + y) * gw + x).reshape(B * X * Y, w * w)


@pytest.mark.parametrize("gh,gw,w", [(8, 8, 2), (6, 12, 3), (16, 8, 8), (14, 28, 7), (7, 7, 7)])
@pytest.mark.parametrize("grid", [False, True])
def test_kernel_address_map_reproduces_the_window_rearrangements(gh, gw, w, grid):
    """The rows the kernel gathers for each window are the tokens the module's (and einops') rearrangement puts in
    it, in the same local order."""
    B = 2
    idx = torch.arange(B * gh * gw).reshape(B, gh, gw)[:, None]            # b d h w, d = 1: the row of each token
    win = mv._ToWindows(w, grid)(idx)                                      # b x y w1 w2 d
    want = win.reshape(-1, w * w)
    assert torch.equal(kernel_rows(B, gh, gw, w, grid), want)
    try:
        einops = importlib.import_module("einops")
    except ImportError:
        einops = None
    if einops is not None:
        pat = "b d (w1 x) (w2 y) -> b x y w1 w2 d" if grid else "b d (x w1) (y w2) -> b x y w1 w2 d"
        assert torch.equal(einops.rearrange(idx, pat, w1=w, w2=w), win)
    back = mv._FromWindows(grid)(win)
    assert torch.equal(back, idx)


@pytest.mark.parametrize("w", [1, 2, 3, 7, 8])
def test_kernel_bias_index_reproduces_rel_pos_indices(w):
    a = Attention(32, 32, window_size=w)
    r = torch.arange(w * w)
    u, v = r // w, r % w
    idx = (u[:, None] - u[None, :] + w - 1) * (2 * w - 1) + (v[:, None] - v[None, :] + w - 1)
    assert torch.equal(idx, a.rel_pos_indices)


def test_window_records_describe_block_then_grid_windows():
    m = MaxViT(**INIT_KWARGS).eval()
    layers, norm = m._encoders()[1].encoder_layers()
    assert norm is None and [L.attention.dilated for L in layers] == [False, True]
    a = m.layers[1][2].fn
    L = layers[0]
    assert L.attention.size == 2 and L.attention.rel_pos_bias is a.rel_pos_bias.weight
    assert L.out_b is None and L.scale == a.scale
    from vit_pytorch_b200.engine import attention_kernel
    assert [attention_kernel(L) for L in layers] == ["window_relpos"] * 2
    engines = [e.engine() for e in m._encoders()]
    assert engines[1].slot is engines[0].slot and engines[2].slot is not engines[0].slot


# ------------------------------------------------------------------------------------------------ fallback rules
@pytest.fixture
def eligible(monkeypatch):
    """fused_reason with the device / dtype / autograd part passed, so its shape rules can be checked on CPU."""
    monkeypatch.setattr(mv, "common_reason", lambda *a, **k: None)


def test_fused_reason_rules(eligible):
    m = MaxViT(**SMALL).eval()                                             # window 2
    img = lambda h, w, c=3: torch.zeros(2, c, h, w)                        # noqa: E731
    assert m.fused_reason(img(32, 32)) is None and m.fused_reason(img(32, 48)) is None
    assert m.fused_reason(img(29, 31)) is None                             # 15 x 16 -> 8 x 8 -> 4 x 4
    assert "not (B, 3, H, W)" in m.fused_reason(torch.zeros(3, 32, 32))
    assert "not (B, 3, H, W)" in m.fused_reason(img(32, 32, c=1))
    assert "not divisible into 2 x 2 windows" in m.fused_reason(img(32, 40))   # 16 x 20 -> 8 x 10 -> 4 x 5
    assert "dim_head=48" in MaxViT(**dict(SMALL, dim=48, dim_head=48)).eval().fused_reason(img(32, 32))
    assert "window_size=9" in MaxViT(**dict(SMALL, window_size=9)).eval().fused_reason(img(144, 144))
    assert MaxViT(**dict(SMALL, window_size=8)).eval().fused_reason(img(64, 64)) is None
    assert "dim_conv_stem=12" in MaxViT(**dict(SMALL, dim_conv_stem=12)).eval().fused_reason(img(32, 32))
    assert "multiples of 8" in MaxViT(**dict(SMALL, mbconv_expansion_rate=1.5)).eval().fused_reason(img(32, 32))
    assert "multiples of 8" in MaxViT(**dict(SMALL, mbconv_shrinkage_rate=0.2)).eval().fused_reason(img(32, 32))
    assert "depth == 0" in MaxViT(**dict(SMALL, depth=(1, 0))).eval().fused_reason(img(32, 32))
    assert MaxViT(**dict(SMALL, dropout=0.1)).eval().fused_reason(img(32, 32)) is None
    t = MaxViT(**SMALL)
    t.train()
    assert "BatchNorm2d is in training mode" in t.fused_reason(img(32, 32))
    t.eval()
    t.layers[0][0][4].running_var = None
    assert "no running statistics" in t.fused_reason(img(32, 32))


def test_fused_reason_on_cpu_input_hooks_and_dropout_in_training():
    m = MaxViT(**SMALL).eval()
    assert "CUDA" in m.fused_reason(torch.zeros(2, 3, 32, 32))
    assert "CUDA" in MaxViT(**dict(SMALL, channels=1)).eval().fused_reason(torch.zeros(2, 1, 32, 32))


@pytest.mark.parametrize("kwargs,hw", [(SMALL, (30, 22)), (dict(SMALL, window_size=7), (64, 64)),
                                       (dict(SMALL, depth=(1, 0)), (32, 32))])
def test_eager_graph_raises_where_the_reference_does(kwargs, hw):
    """A map not divisible by the window (30 x 22: 15 x 11 -> 8 x 6 -> 4 x 3), or a stage of depth 0 (the next stage's
    MBConv expects the skipped stage's width) fail in the reference too when it is installed."""
    from conftest import import_reference, reference_available
    mods = [MaxViT]
    if reference_available():
        import_reference()
        mods.append(importlib.import_module("vit_pytorch.max_vit").MaxViT)
    for cls in mods:
        torch.manual_seed(0)
        m = cls(**kwargs).eval()
        with torch.inference_mode(), pytest.raises(RuntimeError):
            m(torch.randn(1, 3, *hw))


# ------------------------------------------------------------------------------------------------ argument checks
def test_attention_window_relpos_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)

    def call(*, qkv=p, out=p, table=p, B=2, gh=14, gw=28, w=7, grid=1, H=2, dh=32):
        rc = lib.b200vit_attention_window_relpos(qkv, out, table, B, gh, gw, w, grid, H, dh, 0.17, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(qkv=None), dict(out=None), dict(table=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(B=0), b"bad shape"), (dict(gh=0), b"bad shape"), (dict(w=0), b"bad shape"),
                     (dict(H=0), b"bad shape"), (dict(dh=48), b"dim_head=48"), (dict(dh=16), b"dim_head=16"),
                     (dict(w=9, gh=18, gw=18), b"window=9"), (dict(gh=15), b"not divisible"),
                     (dict(gw=27), b"not divisible"), (dict(grid=2), b"grid=2"),
                     (dict(out=ctypes.c_void_p(264)), b"16-byte aligned"),
                     (dict(table=ctypes.c_void_p(260)), b"16-byte aligned"), (dict(H=65536), b"exceeds the grid")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_mbconv_dwconv_rejects_bad_arguments(lib):
    p, q = ctypes.c_void_p(256), ctypes.c_void_p(4096)

    def call(*, x=p, M=2 * 9 * 11, w9=p, bias=p, y=q, part=p, B=2, h=9, w=11, C=64, stride=2):
        rc = lib.b200vit_mbconv_dwconv(x, M, w9, bias, y, part, B, h, w, C, stride, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(x=None), dict(w9=None), dict(bias=None), dict(y=None), dict(part=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(B=0), b"bad shape"), (dict(h=0), b"bad shape"), (dict(C=0), b"bad shape"),
                     (dict(stride=3), b"stride=3"), (dict(M=100), b"100 rows"), (dict(C=60), b"C=60"),
                     (dict(y=p), b"must not be x"), (dict(part=ctypes.c_void_p(260)), b"16-byte aligned"),
                     (dict(B=65536, M=65536 * 99), b"exceed the grid")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_se_pool_and_scale_reject_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    for args, what in (((None, p, 2, 3, 64, 0.5), b"null"), ((p, p, 0, 3, 64, 0.5), b"bad shape"),
                       ((p, p, 2, 0, 64, 0.5), b"bad shape"), ((p, p, 2, 3, 60, 0.5), b"C=60"),
                       ((p, ctypes.c_void_p(258), 2, 3, 64, 0.5), b"16-byte aligned"),
                       ((p, p, 65536, 3, 64, 0.5), b"exceeds the grid")):
        rc = lib.b200vit_se_pool(*args, None)
        assert rc == -1 and what in lib.b200vit_last_error(), args
    for args, what in (((None, p, 2, 9, 64), b"null"), ((p, None, 2, 9, 64), b"null"), ((p, p, 2, 0, 64), b"bad shape"),
                       ((p, p, 2, 9, 20), b"C=20"), ((ctypes.c_void_p(264), p, 2, 9, 64), b"16-byte aligned")):
        rc = lib.b200vit_se_scale(*args, None)
        assert rc == -1 and what in lib.b200vit_last_error(), args


@pytest.mark.parametrize("flags", [
    _lib.EPI_SILU | _lib.EPI_SIGMOID, _lib.EPI_GELU | _lib.EPI_SILU, _lib.EPI_HARDSWISH | _lib.EPI_SIGMOID,
    _lib.EPI_GELU | _lib.EPI_SIGMOID, _lib.EPI_HARDSWISH | _lib.EPI_SILU])
def test_gemm_rejects_two_activations(lib, flags):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_gemm_bf16(p, 64, p, 64, p, None, 64, None, None, None, 0, 1e-5, None, None, 64, 64, 64, flags, None)
    assert rc == -1 and b"exclusive" in lib.b200vit_last_error()


@pytest.mark.parametrize("act", [_lib.EPI_SILU, _lib.EPI_SIGMOID])
def test_gemm_rejects_silu_and_sigmoid_with_a_residual(lib, act):
    p = ctypes.c_void_p(256)
    rc = lib.b200vit_gemm_bf16(p, 64, p, 64, None, p, 64, None, p, None, 0, 1e-5, None, None, 64, 64, 64,
                               act | _lib.EPI_RESIDUAL, None)
    assert rc == -1 and b"EPI_RESIDUAL" in lib.b200vit_last_error()


def test_headnorm_gemm_rejects_the_new_flags(lib):
    p = ctypes.c_void_p(256)
    for f in (_lib.EPI_SILU, _lib.EPI_SIGMOID):
        rc = lib.b200vit_gemm_headnorm_bf16(p, 64, p, 64, p, 64, None, None, 0, 1e-5, None, p, 1, 64, 0.0, 64, 64,
                                            64, f, None)
        assert rc == -1


def test_header_declares_the_new_entry_points_and_flags():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in ("attention_window_relpos", "mbconv_dwconv", "se_pool", "se_scale"):
        assert f"int b200vit_{name}(" in h and f"b200vit_{name}" in _lib.SYMBOLS
    assert "#define B200VIT_EPI_SILU 128" in h and "#define B200VIT_EPI_SIGMOID 256" in h
    assert f"#define B200VIT_MBCONV_PART_ROWS {_lib.MBCONV_PART_ROWS}" in h


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
def test_mbconv_and_attention_launches(lib, ln_mode, host_loop):
    names = [c["call"] for c in MS.record(ln_mode, host_loop)]
    assert names[:4] == ["conv_im2col_nchw", "gemm", "conv_im2col_nhwc", "gemm"]
    assert names[-3:] == ["mean_pool", "layernorm", "gemm"]
    mb = ["gemm", "mbconv_dwconv", "se_pool", "gemm_silu", "gemm_sigmoid", "se_scale", "gemm"]
    starts = [i for i, n in enumerate(names) if n == "mbconv_dwconv"]
    assert len(starts) == 3 and all(names[i - 1:i + 6] == mb for i in starts)
    att = [c for c in MS.record(ln_mode, host_loop) if c["call"] == "attention_window_relpos"]
    assert [(c["gh"], c["gw"], c["w"], c["grid"]) for c in att] == [(8, 4, 2, False), (8, 4, 2, True)] * 2 + \
        [(4, 2, 2, False), (4, 2, 2, True)]
    # the stage's second block adds its MBConv into the stream; the first blocks start fresh streams
    projs = [c for i, c in enumerate(MS.record(ln_mode, host_loop)) if c["call"] == "gemm" and
             i > 0 and names[i - 1] == "se_scale"]
    assert [p["resid"] is None for p in projs] == [True, False, True]


def test_other_families_schedule_fixtures_are_unchanged(lib):
    """Every other family's pinned launch sequence, regenerated, is byte-identical to its fixture."""
    for mod in ("make_engine_schedule", "make_cct_schedule", "make_pit_schedule", "make_levit_schedule",
                "make_twins_svt_schedule"):
        g = importlib.import_module(mod)
        with open(g.FIXTURE) as f:
            assert S.dumps(g.generate()) == f.read(), mod
