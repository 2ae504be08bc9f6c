"""CvT (vit_pytorch_b200.cvt) without a GPU: the attribute and state_dict surface, the BatchNorm folds of the
convolutional projections in fp64, the query and key / value map geometry against the convolutions' output shapes,
the engine's description of a CvT layer and its prepared-weight refresh, the fallback rules and that the eager graph
raises where the reference does, the argument checks of b200vit_conv_proj_dw, and the launch sequence of the whole
fused forward (tests/golden/cvt_schedule.json, made by make_cvt_schedule.py).  The reference-parity tests are in
test_cvt_parity.py."""
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build, cvt as cv
from vit_pytorch_b200.cvt import CvT, DepthWiseConv2d
from vit_pytorch_b200.engine import ConvProj, attention_kernel, conv_proj_weights

sys.path.insert(0, GOLDEN_DIR)
from cvt_spec import INIT_KWARGS, SMALL  # noqa: E402
import make_cvt_schedule as CS  # noqa: E402
import make_engine_schedule as S  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def reference_cvt():
    """The reference's cvt module when it is installed, else None."""
    from conftest import import_reference, reference_available
    if not reference_available():
        return None
    import_reference()
    return importlib.import_module("vit_pytorch.cvt")


def test_attribute_surface():
    m = CvT(**INIT_KWARGS)
    assert len(m.layers) == 3 and [len(s[2].layers) for s in m.layers] == [1, 2, 2]
    keys = list(m.state_dict())
    assert keys[:4] == ["layers.0.0.weight", "layers.0.0.bias", "layers.0.1.g", "layers.0.1.b"]
    assert keys[-2:] == ["to_logits.2.weight", "to_logits.2.bias"]
    for k in ("layers.0.2.layers.0.0.to_q.net.0.weight", "layers.0.2.layers.0.0.to_q.net.1.running_var",
              "layers.1.2.layers.1.0.to_kv.net.2.weight", "layers.2.2.layers.0.1.net.4.bias",
              "layers.2.2.layers.0.0.to_out.0.weight"):
        assert k in keys, k
    a = m.layers[2][2].layers[0][0]
    assert a.to_q.net[0].bias is None and a.to_q.net[2].bias is None and a.to_kv.net[2].weight.shape == (256, 48, 1, 1)


def test_seeded_init_is_deterministic():
    torch.manual_seed(5)
    a = CvT(**SMALL).state_dict()
    torch.manual_seed(5)
    b = CvT(**SMALL).state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


def _perturbed_bn(bn, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        bn.weight.copy_(torch.randn(bn.weight.shape, generator=g))
        bn.bias.copy_(torch.randn(bn.bias.shape, generator=g))
        bn.running_mean.copy_(torch.randn(bn.running_mean.shape, generator=g))
        bn.running_var.copy_(0.2 + torch.rand(bn.running_var.shape, generator=g))
    return bn.eval()


def _conv_proj(q: DepthWiseConv2d, kv: DepthWiseConv2d) -> ConvProj:
    dq, bq, _ = q.net
    dkv, bkv, _ = kv.net
    return ConvProj(dq.weight, bq.weight, bq.bias, bq.running_mean, bq.running_var, bq.eps, dkv.weight, bkv.weight,
                    bkv.bias, bkv.running_mean, bkv.running_var, bkv.eps, dq.kernel_size[0], dkv.stride[0])


@pytest.mark.parametrize("k,s", [(1, 1), (3, 2), (5, 3), (7, 2)])
def test_folded_batchnorms_reproduce_the_module_in_fp64(k, s):
    """The folded tap-major weights of conv_proj_weights, as a depthwise convolution with bias followed by the 1 x 1
    convolution, reproduce the (reference, when installed) DepthWiseConv2d in eval mode."""
    ref = reference_cvt()
    make = ref.DepthWiseConv2d if ref is not None else DepthWiseConv2d
    torch.manual_seed(k * 10 + s)
    q = make(16, 32, k, padding=k // 2, stride=1, bias=False).double().eval()
    kv = make(16, 64, k, padding=k // 2, stride=s, bias=False).double().eval()
    _perturbed_bn(q.net[1], 3)
    _perturbed_bn(kv.net[1], 4)
    wq, bq, wkv, bkv = conv_proj_weights(_conv_proj(q, kv))
    assert wq.dtype == torch.float32 and wq.shape == (k * k, 16) and bq.shape == (16,) and wkv.shape == (k * k, 16)
    x = torch.randn(2, 16, 9, 7, dtype=torch.float64)
    F = torch.nn.functional
    with torch.no_grad():
        for mod, w, b, stride in ((q, wq, bq, 1), (kv, wkv, bkv, s)):
            want = mod(x)
            dw = F.conv2d(x, w.double().t().reshape(16, 1, k, k), b.double(), stride=stride, padding=k // 2, groups=16)
            got = F.conv2d(dw, mod.net[2].weight)
            assert torch.allclose(got, want, atol=1e-5, rtol=1e-5), (got - want).abs().max()


@pytest.mark.parametrize("k", [1, 3, 5, 7])
@pytest.mark.parametrize("s", [1, 2, 3])
@pytest.mark.parametrize("h,w", [(1, 1), (2, 3), (7, 5), (13, 10), (25, 19), (56, 56)])
def test_map_geometry_matches_the_convolutions(k, s, h, w):
    """The query map is the token grid and the key / value map (h - 1) // s + 1 by (w - 1) // s + 1: the output shapes
    of the projections' depthwise convolutions."""
    torch.manual_seed(0)
    q = DepthWiseConv2d(8, 8, k, padding=k // 2, stride=1, bias=False).eval()
    kv = DepthWiseConv2d(8, 16, k, padding=k // 2, stride=s, bias=False).eval()
    x = torch.zeros(1, 8, h, w)
    with torch.no_grad():
        assert q(x).shape[2:] == (h, w)
        assert tuple(kv(x).shape[2:]) == _conv_proj(q, kv).grid(h, w)


# ------------------------------------------------------------------------------------------------ engine
def test_encoder_layers_carry_conv_projection_records():
    m = CvT(**INIT_KWARGS).eval()
    layers, norm = m.layers[2][2].encoder_layers()
    assert norm is None and len(layers) == 2
    a = m.layers[2][2].layers[0][0]
    L = layers[0]
    assert attention_kernel(L) == "kv" and isinstance(L.attention, ConvProj)
    assert L.qkv_w.shape == (128, 48) and L.attention.kv_proj_w.shape == (256, 48) and L.out_w.shape == (48, 128)
    assert L.attention.kernel_size == 3 and L.attention.stride == 2
    assert L.attention.q_bn_var is a.to_q.net[1].running_var
    assert L.heads == 2 and L.dim_head == 64 and L.scale == a.scale
    eng = m.layers[2][2].engine()
    assert eng.unsupported_reason(49, grid=(7, 7)) is None
    t = eng.prepared()
    assert t["0.cpq.w"].shape == (9, 48) and t["0.cpkv.b"].shape == (48,) and t["0.kv.w"].shape == (256, 48)
    assert t["0.kv.w"].dtype == torch.bfloat16 and t["c_layers"] is None
    assert torch.equal(t["0.kv.w"], a.to_kv.net[2].weight.detach().reshape(256, 48).bfloat16())


def test_running_statistics_rebuild_the_prepared_weights():
    m = CvT(**SMALL).eval()
    eng = m.layers[0][2].engine()
    bn = m.layers[0][2].layers[0][0].to_kv.net[1]
    assert any(b is bn.running_var for b in m.layers[0][2].prepared_buffers())
    before = eng.prepared()["0.cpkv.w"]
    with torch.no_grad():
        bn.running_var.mul_(4.0)                       # in place: the version counter moves
    after = eng.prepared()["0.cpkv.w"]
    assert torch.allclose(after, before / 2, rtol=1e-3, atol=1e-6)


@pytest.mark.parametrize("k", [2, 4, 9])
def test_engine_rejects_unbuilt_projection_kernels(k):
    m = CvT(**dict(SMALL, s2_proj_kernel=k)).eval()
    assert f"proj_kernel={k}" in m.layers[1][2].engine().unsupported_reason(64)


@pytest.mark.parametrize("grid", [(1, 1), (7, 5), (3, 17)])
def test_run_blocks_accepts_any_grid_for_conv_projections(grid):
    """No divisibility rule: the layer reaches its first launch for any h, w >= 1 (recorded, nothing computes)."""
    m = CvT(**SMALL).eval()
    eng = m.layers[1][2].engine()
    h, w = grid
    x = torch.zeros(2 * h * w, 32)
    with S.recording(eng, S.caller_buffers(eng, x, {}), "fold", "python", ("conv_proj_dw", "attention_kv")) as rec:
        eng.run_blocks(x, 2, h * w, grid=grid)
        kv = [c for c in rec.calls if c["call"] == "attention_kv"]
        assert [(c["Nq"], c["Nk"]) for c in kv] == [(h * w, ((h - 1) // 2 + 1) * ((w - 1) // 2 + 1))]
        with pytest.raises(ValueError, match="h \\* w == N"):
            eng.run_blocks(x, 2, h * w + 1, grid=grid)


# ------------------------------------------------------------------------------------------------ fallback rules
@pytest.fixture
def eligible(monkeypatch):
    """fused_reason with the device / dtype / autograd part passed, so its shape rules can be checked on CPU."""
    monkeypatch.setattr(cv, "common_reason", lambda *a, **k: None)


def test_fused_reason_rules(eligible):
    m = CvT(**SMALL).eval()
    img = lambda h, w, c=3: torch.zeros(2, c, h, w)                        # noqa: E731
    assert m.fused_reason(img(64, 64)) is None and m.fused_reason(img(100, 75)) is None
    assert m.fused_reason(img(16, 16)) is None and m.fused_reason(img(1, 1)) is None     # 1 x 1 maps throughout
    assert "not (B, 3, H, W)" in m.fused_reason(torch.zeros(3, 64, 64))
    assert "not (B, 3, H, W)" in m.fused_reason(img(64, 64, c=1))
    assert "not (B, 1, H, W)" in CvT(**dict(SMALL, channels=1)).eval().fused_reason(img(64, 64))
    assert "emb_dim=20" in CvT(**dict(SMALL, s2_emb_dim=20)).eval().fused_reason(img(64, 64))
    assert "emb_kernel=17" in CvT(**dict(SMALL, s1_emb_kernel=17)).eval().fused_reason(img(64, 64))
    assert CvT(**dict(SMALL, s1_emb_kernel=4, s1_emb_stride=4)).eval().fused_reason(img(64, 64)) is None
    assert "proj_kernel=2" in CvT(**dict(SMALL, s1_proj_kernel=2)).eval().fused_reason(img(64, 64))
    assert "proj_kernel=4" in CvT(**dict(SMALL, s3_proj_kernel=4)).eval().fused_reason(img(64, 64))
    assert "proj_kernel=9" in CvT(**dict(SMALL, s3_proj_kernel=9)).eval().fused_reason(img(64, 64))
    assert "empty" in m.fused_reason(img(0, 64))
    assert "16641 > 16384" in m.fused_reason(img(516, 516))                  # 129 x 129 at stage 1
    assert m.fused_reason(img(512, 512)) is None                            # 128 x 128
    assert CvT(**dict(SMALL, dropout=0.1)).eval().fused_reason(img(64, 64)) is None
    t = CvT(**SMALL)
    t.train()
    assert "BatchNorm2d is in training mode" in t.fused_reason(img(64, 64))
    t.eval()
    t.layers[1][2].layers[0][0].to_kv.net[1].running_var = None
    assert "no running statistics" in t.fused_reason(img(64, 64))


def test_fused_reason_common_rules():
    m = CvT(**SMALL).eval()
    assert "CUDA" in m.fused_reason(torch.zeros(2, 3, 64, 64))
    assert "depth == 0" in CvT(**dict(SMALL, s2_depth=0)).eval().fused_reason(torch.zeros(2, 3, 64, 64))


@pytest.mark.parametrize("kwargs,hw", [(dict(SMALL, s2_proj_kernel=2), (64, 64)),
                                       (dict(SMALL, s1_proj_kernel=4), (40, 24)),
                                       (dict(SMALL, s1_proj_kernel=2), (64, 4))])
def test_eager_graph_raises_where_the_reference_does(kwargs, hw):
    """An even proj_kernel grows the query map by one, and the rearrangement after the attention fails (or, on a
    one-token-wide map, the residual add), in the reference too when it is installed."""
    ref = reference_cvt()
    mods = [CvT] + ([ref.CvT] if ref is not None else [])
    for cls in mods:
        torch.manual_seed(0)
        m = cls(**kwargs).eval()
        with torch.inference_mode(), pytest.raises(RuntimeError):
            m(torch.randn(1, 3, *hw))


# ------------------------------------------------------------------------------------------------ argument checks
def test_conv_proj_dw_rejects_bad_arguments(lib):
    p, q, r = ctypes.c_void_p(256), ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 21)

    def call(*, x=p, M=2 * 9 * 11, wq=p, bq=p, wkv=p, bkv=p, qo=q, kvo=r, B=2, h=9, w=11, C=64, k=3, s=2):
        rc = lib.b200vit_conv_proj_dw(x, M, wq, bq, wkv, bkv, qo, kvo, B, h, w, C, k, s, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(x=None), dict(wq=None), dict(bq=None), dict(wkv=None), dict(bkv=None), dict(qo=None),
               dict(kvo=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(B=0), b"bad shape"), (dict(h=0), b"bad shape"), (dict(w=0), b"bad shape"),
                     (dict(C=0), b"bad shape"), (dict(k=2), b"kernel size 2"), (dict(k=9), b"kernel size 9"),
                     (dict(k=0), b"kernel size 0"), (dict(s=0), b"s=0"), (dict(s=-1), b"s=-1"), (dict(C=60), b"C=60"),
                     (dict(M=100), b"100 rows"), (dict(x=ctypes.c_void_p(264)), b"16-byte aligned"),
                     (dict(bkv=ctypes.c_void_p(260)), b"16-byte aligned"),
                     (dict(kvo=ctypes.c_void_p((1 << 21) + 8)), b"16-byte aligned"),
                     (dict(qo=p), b"overlap"), (dict(kvo=ctypes.c_void_p(256 + 2 * 9 * 11 * 64 * 2 - 16)), b"overlap"),
                     (dict(x=ctypes.c_void_p((1 << 20) + 2 * 9 * 11 * 64 * 2 - 16)), b"overlap")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_header_declares_the_new_entry_point():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    assert "int b200vit_conv_proj_dw(" in h and "b200vit_conv_proj_dw" in _lib.SYMBOLS


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


@pytest.mark.parametrize("ln_mode,host_loop", CS.RUNS)
def test_conv_projection_launches(lib, ln_mode, host_loop):
    calls = CS.record(ln_mode, host_loop)
    names = [c["call"] for c in calls]
    assert names[:3] == ["conv_im2col_nchw", "gemm", "embed_tokens"]
    assert names[-3:] == ["mean_pool", "cast_f32_bf16", "gemm"]
    attn = ["layernorm", "conv_proj_dw", "gemm", "gemm", "attention_kv", "gemm"]
    starts = [i for i, n in enumerate(names) if n == "conv_proj_dw"]
    assert len(starts) == 4 and all(names[i - 1:i + 5] == attn for i in starts)
    cp = [c for c in calls if c["call"] == "conv_proj_dw"]
    assert [(c["h"], c["w"], c["k"], c["s"]) for c in cp] == [(6, 5, 3, 2), (3, 3, 5, 1), (3, 3, 5, 1), (2, 2, 1, 2)]
    kv = [c for c in calls if c["call"] == "attention_kv"]
    assert [(c["Nq"], c["Nk"]) for c in kv] == [(30, 9), (9, 9), (9, 9), (4, 1)]
    # stages 2 and 3 read the previous stage's bf16 stream copy
    assert names.count("conv_im2col_nhwc") == 2


def test_other_families_schedule_fixtures_are_unchanged(lib):
    """Every other family's pinned launch sequence, regenerated, is byte-identical to its fixture."""
    for mod in ("make_engine_schedule", "make_cct_schedule", "make_pit_schedule", "make_levit_schedule",
                "make_twins_svt_schedule", "make_max_vit_schedule"):
        g = importlib.import_module(mod)
        with open(g.FIXTURE) as f:
            assert S.dumps(g.generate()) == f.read(), mod
