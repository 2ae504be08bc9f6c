"""PiT (vit_pytorch_b200.pit) without a GPU: the attribute surface, the prepared pool weights, the fallback rules
including the reference's int(sqrt(n)) grid rule, the argument checks of the unfold and pool entry points, and the
launch sequence of the whole fused forward (tests/golden/pit_schedule.json, made by make_pit_schedule.py).  The
reference-parity tests are in test_family_parity.py."""
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR, ROOT, import_reference, reference_available
from vit_pytorch_b200 import _lib, build, pit as pit_mod
from vit_pytorch_b200.pit import PiT, Pool, Transformer, pool_grid, pool_weights

sys.path.insert(0, GOLDEN_DIR)
from pit_spec import INIT_KWARGS  # noqa: E402
import make_pit_schedule as PS  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def test_attribute_surface():
    m = PiT(**INIT_KWARGS)
    assert isinstance(m.to_patch_embedding[0], torch.nn.Unfold) and isinstance(m.to_patch_embedding[2], torch.nn.Linear)
    assert m.to_patch_embedding[2].in_features == 3 * 8 * 8
    assert m.pos_embedding.shape == (1, 50, 32) and m.cls_token.shape == (1, 1, 32)
    kinds = [type(t).__name__ for t in m.layers]
    assert kinds == ["Transformer", "Pool", "Transformer", "Pool", "Transformer"]
    assert [t.layers[0][0].heads for t in m.stages()] == [2, 2, 4]
    assert not hasattr(m.layers[0], "norm")
    pool = m.layers[1]
    assert pool.downsample.net[0].weight.shape == (64, 1, 3, 3) and pool.downsample.net[0].groups == 32
    assert pool.downsample.net[1].weight.shape == (64, 64, 1, 1) and pool.cls_ff.weight.shape == (64, 32)
    assert m.mlp_head[0].normalized_shape == (128,) and m.mlp_head[1].in_features == 128
    keys = list(m.state_dict())
    assert keys[:4] == ["pos_embedding", "cls_token", "to_patch_embedding.2.weight", "to_patch_embedding.2.bias"] or \
        keys[:4] == ["to_patch_embedding.2.weight", "to_patch_embedding.2.bias", "pos_embedding", "cls_token"]
    assert "layers.1.downsample.net.0.weight" in keys and "layers.1.cls_ff.bias" in keys
    assert keys[-4:] == ["mlp_head.0.weight", "mlp_head.0.bias", "mlp_head.1.weight", "mlp_head.1.bias"]


def test_pool_grid_follows_the_reference_rule():
    assert pool_grid(961) == (31, 31) and pool_grid(64) == (8, 8) and pool_grid(1) == (1, 1)
    assert pool_grid(15) == (3, 5) and pool_grid(6) == (2, 3)
    assert pool_grid(7) is None and pool_grid(10) is None              # einops cannot split 7 / 10 tokens by 2 / 3
    m = PiT(**{**INIT_KWARGS, "image_size": 36, "patch_size": 4})
    assert m.stage_grids(10, 34) == [(8, 8), (4, 4)]                    # a 4 x 16 unfold grid is read as 8 x 8
    assert m.stage_grids(6, 12) is None                                 # 2 x 5: 10 tokens, int(sqrt(10)) = 3


@pytest.fixture
def eligible(monkeypatch):
    """fused_reason with the device / dtype / autograd part passed, so its shape rules can be checked on CPU."""
    monkeypatch.setattr(pit_mod, "common_reason", lambda *a, **k: None)


def test_fused_reason_rules(eligible):
    m = PiT(**{**INIT_KWARGS, "image_size": 36, "patch_size": 4}).eval()
    img = lambda c, h, w: torch.zeros(2, c, h, w)                       # noqa: E731
    assert m.fused_reason(img(3, 36, 36)) is None
    assert m.fused_reason(img(3, 10, 34)) is None                       # the isqrt re-read is fused
    assert "not (B, C, H, W)" in m.fused_reason(torch.zeros(3, 36, 36))
    assert "channel count" in m.fused_reason(img(1, 36, 36))
    assert "smaller than one" in m.fused_reason(img(3, 3, 36))
    assert "positional table" in m.fused_reason(img(3, 40, 40))
    assert "int(sqrt(n))" in m.fused_reason(img(3, 6, 12))
    assert "dim_head=48" in PiT(**{**INIT_KWARGS, "dim_head": 48}).fused_reason(img(3, 32, 32))
    assert "multiples of 8" in PiT(**{**INIT_KWARGS, "mlp_dim": 60}).fused_reason(img(3, 32, 32))
    assert "multiples of 8" in PiT(**{**INIT_KWARGS, "dim": 20}).fused_reason(img(3, 32, 32))


def test_fused_reason_on_cpu_input():
    m = PiT(**INIT_KWARGS).eval()
    assert "CUDA" in m.fused_reason(torch.zeros(2, 3, 32, 32))


def test_isqrt_refusal_raises_like_the_reference():
    """A stage whose token count the reference's Pool cannot reshape raises in the eager graph, as the reference's
    einops call does (EinopsError is a RuntimeError)."""
    kw = {**INIT_KWARGS, "image_size": 36, "patch_size": 4}
    x = torch.randn(2, 3, 6, 12)
    torch.manual_seed(0)
    m = PiT(**kw).eval()
    with torch.inference_mode(), pytest.raises(RuntimeError):
        m(x)
    if reference_available():
        import_reference()
        torch.manual_seed(0)
        r = importlib.import_module("vit_pytorch.pit").PiT(**kw).eval()
        with torch.inference_mode(), pytest.raises(RuntimeError):
            r(x)


@pytest.mark.parametrize("hw", [(1, 1), (2, 2), (3, 5), (7, 7), (8, 8)])
def test_pool_weights_reproduce_the_module(hw):
    """pool_weights applied as the depthwise stride-2 convolution (tap-major weights), the 1 x 1 GEMM and cls_ff in
    fp32 torch gives Pool(x) for bf16-representable parameters."""
    torch.manual_seed(hw[0] * 10 + hw[1])
    D = 16
    pool = Pool(D).eval()
    with torch.no_grad():
        for p in pool.parameters():
            p.copy_(p.bfloat16().float())
    h, w = hw
    x = torch.randn(2, 1 + h * w, D)
    t = pool_weights(pool)
    assert t["w9"].shape == (9, 2 * D) and t["w1"].shape == (2 * D, 2 * D) and t["wc"].shape == (2 * D, D)
    with torch.no_grad():
        grid = x[:, 1:].reshape(2, h, w, D).permute(0, 3, 1, 2)
        a = F.conv2d(grid, t["w9"].t().reshape(2 * D, 1, 3, 3), t["b9"], stride=2, padding=1, groups=D)
        a = a.flatten(2).transpose(1, 2)
        tokens = a @ t["w1"].float().t() + t["b1"]
        cls = x[:, :1] @ t["wc"].float().t() + t["bc"]
        got = torch.cat((cls, tokens), 1)
        want = pool(x)
    assert got.shape == (2, 1 + ((h + 1) // 2) * ((w + 1) // 2), 2 * D)
    assert torch.allclose(got, want, atol=1e-5, rtol=1e-5), (got - want).abs().max()


def test_direct_transformer_call_on_cpu():
    torch.manual_seed(5)
    t = Transformer(32, 2, 2, 32, 64).eval()
    x = torch.randn(2, 17, 32)
    with torch.inference_mode():
        out = t(x)
        want = x
        for a, ff in t.layers:
            want = a(want) + want
            want = ff(want) + want
    assert torch.equal(out, want)


def test_eager_graph_keeps_hooks_observable():
    m = PiT(**INIT_KWARGS).eval()
    seen = []
    m.layers[1].downsample.net[0].register_forward_hook(lambda mod, i, o: seen.append(tuple(o.shape)))
    with torch.inference_mode():
        m(torch.randn(2, 3, 32, 32))
    assert seen == [(2, 64, 4, 4)]                         # a 7 x 7 grid pooled to 4 x 4


def test_unfold_patches_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    def call(*, img=p, out=p, ldo=640, B=2, C=3, H=224, W=224, k=14, s=7):
        rc = lib.b200vit_unfold_patches(img, out, ldo, B, C, H, W, k, s, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(img=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw in (dict(k=1, s=1), dict(s=0), dict(H=13), dict(W=13), dict(B=0), dict(C=0)):
        rc, msg = call(**kw)
        assert rc == -1 and b"bad shape" in msg, kw
    rc, msg = call(ldo=584)
    assert rc == -1 and b"ldo=584" in msg
    rc, msg = call(ldo=596)
    assert rc == -1 and b"multiple of 8" in msg
    rc, msg = call(out=ctypes.c_void_p(264))
    assert rc == -1 and b"16-byte aligned" in msg
    rc, msg = call(k=200, s=100, H=400, W=400, ldo=120000)
    assert rc == -1 and b"shared memory" in msg


def test_pit_pool_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    def call(*, x=p, M=2 * 962, B=2, h=31, w=31, D=256, w9=p, bias=p, a=p, lda=512, cls=p, ldc=256):
        rc = lib.b200vit_pit_pool(x, M, B, h, w, D, w9, bias, a, lda, cls, ldc, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(x=None), dict(w9=None), dict(bias=None), dict(a=None), dict(cls=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw in (dict(h=0), dict(w=0), dict(B=0), dict(D=0)):
        rc, msg = call(**kw)
        assert rc == -1 and b"bad shape" in msg, kw
    rc, msg = call(M=2 * 961)
    assert rc == -1 and b"1922 rows" in msg and b"1924 expected" in msg
    rc, msg = call(D=260, lda=520, ldc=264)
    assert rc == -1 and b"multiple of 8" in msg
    rc, msg = call(lda=504)
    assert rc == -1 and b"lda=504" in msg
    rc, msg = call(ldc=248)
    assert rc == -1 and b"ldc=248" in msg
    for kw in (dict(x=ctypes.c_void_p(264)), dict(a=ctypes.c_void_p(264)), dict(cls=ctypes.c_void_p(264)),
               dict(w9=ctypes.c_void_p(264))):
        rc, msg = call(**kw)
        assert rc == -1 and b"16-byte aligned" in msg, kw
    rc, msg = call(h=3, w=20000, M=2 * 60001, D=8, lda=16, ldc=8)
    assert rc == -1 and b"shared memory" in msg


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in ("b200vit_unfold_patches", "b200vit_pit_pool"):
        assert f"int {name}(" in h and name in _lib.SYMBOLS


# ------------------------------------------------------------------------------------------------ launch sequence
@pytest.fixture(scope="module")
def schedule():
    with open(PS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [PS.run_name(m, h) for m, h in PS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", PS.RUNS)
def test_fused_forward_schedule_matches_fixture(lib, schedule, ln_mode, host_loop):
    name = PS.run_name(ln_mode, host_loop)
    got, want = PS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
def test_stage_transition_sequence(lib, ln_mode):
    """Between two stages: pit_pool, the 1 x 1 GEMM over every row of the next stream, cls_ff over its cls rows, and
    in fold mode the rowstats_cast that primes the next stage; the head normalises the last stage's cls rows."""
    calls = PS.record(ln_mode, "python")
    names = [c["call"] for c in calls]
    assert names[:3] == ["unfold_patches", "gemm", "embed_tokens"] and names[-2:] == ["layernorm", "gemm"]
    starts = [i for i, n in enumerate(names) if n == "pit_pool"]
    assert len(starts) == 2
    for k, i in enumerate(starts):
        pool, conv, cls = calls[i:i + 3]
        assert conv["call"] == cls["call"] == "gemm"
        assert pool["a_bf16"] == conv["a"] and pool["cls_bf16"] == cls["a"]
        assert conv["w"]["key"] == f"pool{k}.w1" and cls["w"]["key"] == f"pool{k}.wc"
        x2 = conv["out_f32"]
        assert cls["out_f32"]["role"] == x2["role"] and cls["out_f32"]["stride"] == [x2["shape"][0] // 2 * x2["shape"][1], 1]
        nxt = calls[i + 3]
        if ln_mode == "fold":
            assert nxt["call"] == "rowstats_cast" and nxt["x"] == x2 and nxt["xb"]["role"] == f"stage{k + 1}.ws.xn"
        else:
            assert nxt["call"] == "layernorm" and nxt["x"] == x2
    assert calls[-2]["row_index"] is not None and calls[-2]["x"]["role"] == calls[starts[-1] + 1]["out_f32"]["role"]
