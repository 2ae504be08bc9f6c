"""SepViT (vit_pytorch_b200.sep_vit) without a GPU: the module surface and that the eager graph raises where the
reference does, a pure-torch fp64 emulation of the fused dataflow (the kernels' address maps, the interleaved window
q | k columns, the constant window-token q | k | v) against the reference's DSSA, the fallback rules, the engine
description of the README config, the argument checks of the new entry points, and the launch sequence of the whole
fused forward (tests/golden/sep_vit_schedule.json, made by make_sep_vit_schedule.py).  The reference-parity tests are
in test_sep_vit_parity.py."""
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build, sep_vit as sv
from vit_pytorch_b200.engine import attention_kernel
from vit_pytorch_b200.sep_vit import DSSA, SepViT, Transformer

sys.path.insert(0, GOLDEN_DIR)
import make_engine_schedule as S  # noqa: E402
import make_sep_vit_schedule as SS  # noqa: E402

README = dict(num_classes=1000, dim=32, dim_head=32, heads=(1, 2, 4, 8), depth=(1, 2, 6, 2), window_size=7)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def small(**kw):
    torch.manual_seed(0)
    return SepViT(**dict(dict(num_classes=5, dim=32, heads=(1, 2), depth=(1, 1)), **kw)).eval()


# ------------------------------------------------------------------------------------------------ surface
def test_module_surface():
    assert set(sv.__all__) >= {"ChanLayerNorm", "DSSA", "FeedForward", "OverlappingPatchEmbed", "PEG", "SepViT",
                               "Transformer"}
    import vit_pytorch_b200
    assert vit_pytorch_b200.SepViT is SepViT
    m = small()
    assert [n for n, _ in m.layers[0][2].layers[0][0].named_parameters()] == [
        "window_tokens", "norm.g", "norm.b", "to_qkv.weight", "window_tokens_to_qk.0.weight",
        "window_tokens_to_qk.0.bias", "window_tokens_to_qk.3.weight", "window_tokens_to_qk.3.bias", "to_out.0.weight",
        "to_out.0.bias"]
    assert isinstance(m.layers[1][2].norm, torch.nn.Identity)


def test_eager_graph_raises_where_the_reference_does():
    m = small()
    with torch.no_grad():
        assert m(torch.randn(1, 3, 112, 56)).shape == (1, 5)
        with pytest.raises(AssertionError, match="divisible by window size"):
            m(torch.randn(1, 3, 96, 96))
    with pytest.raises(AssertionError, match="tuple"):
        SepViT(num_classes=5, dim=32, heads=(1, 2), depth=2)
    with pytest.raises(AssertionError):
        SepViT(num_classes=5, dim=32, heads=(1, 2, 4), depth=(1, 1))


# ------------------------------------------------------------------------------------------------ fp64 dataflow
def fused_dataflow(attn: DSSA, x: torch.Tensor) -> torch.Tensor:
    """DSSA(x) on a (b, c, h, w) map as the fused path computes it, in fp64: channels-last rows (b, y, x), the window
    token's q | k | v projected once, window (b, wy, wx) with row 0 the window token and rows 1 + u*p + v the map rows
    of the kernel's address map, the window-token outputs in row (b*nwy + wy)*nwx + wx, their LayerNorm + GELU and
    the q | k GEMM with per-head interleaved columns, and the attention across windows position by position."""
    b, c, gh, gw = x.shape
    p, H = attn.window_size, attn.heads
    dh = attn.to_qkv.weight.shape[0] // 3 // H
    I = H * dh
    nwy, nwx = gh // p, gw // p
    nw = nwy * nwx
    rows = x.permute(0, 2, 3, 1).reshape(-1, c)
    g, beta = attn.norm.g.reshape(-1), attn.norm.b.reshape(-1)
    xn = (rows - rows.mean(1, keepdim=True)) / (rows.var(1, unbiased=False, keepdim=True) + attn.norm.eps).sqrt()
    xn = xn * g + beta
    W = attn.to_qkv.weight.reshape(3 * I, c)
    qkv = xn @ W.t()
    tok = W @ attn.window_tokens
    o = torch.empty(b * gh * gw, I, dtype=x.dtype)
    tok_out = torch.empty(b * nw, I, dtype=x.dtype)
    for bi in range(b):
        for wy in range(nwy):
            for wx in range(nwx):
                mrows = [(bi * gh + wy * p + u) * gw + wx * p + v for u in range(p) for v in range(p)]
                t = torch.cat((tok[None], qkv[mrows]))                       # [1 + p*p, 3I]
                for h in range(H):
                    q, k, v = (t[:, j * I + h * dh:j * I + (h + 1) * dh] for j in range(3))
                    out = torch.softmax(q @ k.t() * attn.scale, -1) @ v
                    o[mrows, h * dh:(h + 1) * dh] = out[1:]
                    tok_out[(bi * nwy + wy) * nwx + wx, h * dh:(h + 1) * dh] = out[0]
    if nw > 1:
        ln = attn.window_tokens_to_qk[0]
        tv = tok_out.view(-1, H, dh)
        tv = torch.nn.functional.gelu(torch.nn.functional.layer_norm(tv, (dh,), ln.weight, ln.bias, ln.eps))
        conv = attn.window_tokens_to_qk[3]
        wqk = tv.reshape(-1, I) @ conv.weight.reshape(2 * I, I).t() + conv.bias
        mixed = torch.empty_like(o)
        for bi in range(b):
            for h in range(H):
                wq = wqk[bi * nw:(bi + 1) * nw, 2 * h * dh:2 * h * dh + dh]
                wk = wqk[bi * nw:(bi + 1) * nw, 2 * h * dh + dh:2 * (h + 1) * dh]
                P = torch.softmax(wq @ wk.t() * attn.scale, -1)
                for q in range(p * p):
                    u, v = divmod(q, p)
                    mrows = [(bi * gh + (j // nwx) * p + u) * gw + (j % nwx) * p + v for j in range(nw)]
                    mixed[mrows, h * dh:(h + 1) * dh] = P @ o[mrows, h * dh:(h + 1) * dh]
        o = mixed
    y = o @ attn.to_out[0].weight.reshape(c, I).t() + attn.to_out[0].bias
    return y.view(b, gh, gw, c).permute(0, 3, 1, 2)


@pytest.mark.parametrize("p,hw,heads", [(7, (14, 21), 2), (7, (7, 7), 1), (2, (4, 6), 4), (1, (3, 2), 1),
                                        (4, (8, 8), 2)])
def test_fused_dataflow_matches_the_dssa_in_fp64(p, hw, heads):
    torch.manual_seed(p + heads)
    attn = DSSA(16, heads=heads, window_size=p).double().eval()
    with torch.no_grad():
        for prm in attn.parameters():
            prm.add_(0.1 * torch.randn(prm.shape, dtype=torch.float64))
        x = torch.randn(2, 16, *hw, dtype=torch.float64)
        want = attn(x)
        got = fused_dataflow(attn, x)
    assert (got - want).abs().max().item() < 1e-10


# ------------------------------------------------------------------------------------------------ fallback rules
def test_fused_reason_rules(monkeypatch):
    x = torch.zeros(2, 3, 112, 112, dtype=torch.bfloat16)
    m = small().bfloat16()
    assert m.fused_reason(x) == "input is not on a CUDA device"
    monkeypatch.setattr(sv, "common_reason", lambda *a, **k: None)
    assert m.fused_reason(x) is None
    assert "channels" in m.fused_reason(torch.zeros(2, 1, 112, 112))
    assert "not divisible by window_size=7" in m.fused_reason(torch.zeros(2, 3, 96, 96))
    assert "256 windows" in m.fused_reason(torch.zeros(1, 3, 448, 448))
    assert "multiples of 8" in small(dim=36).fused_reason(x)
    big = small()
    for attn, _ in big.layers[0][2].layers:
        attn.window_size = 14
    assert "window_size=14" in big.fused_reason(torch.zeros(1, 3, 224, 224))
    wide = small()
    wide.layers[0][2].layers[0][0].dim_head = 48                       # as a DSSA built with dim_head=48 reports it
    assert "dim_head=48" in wide.fused_reason(x)
    m.train()
    assert "training" in m.fused_reason(x)
    m.eval()
    tr = m.layers[0][2]
    assert "(b, c, h, w)" in tr.fused_reason(torch.zeros(2, 28, 32))
    assert "not divisible" in tr.fused_reason(torch.zeros(2, 32, 27, 28))


def test_fused_reason_names_dtype_device_and_hooks(monkeypatch):
    m = small().bfloat16()
    assert "CUDA" in m.fused_reason(torch.zeros(1, 3, 112, 112, dtype=torch.bfloat16))
    import vit_pytorch_b200.engine as E
    monkeypatch.setattr(E, "why_not_fused", lambda *a, **k: None)
    h = m.layers[0][2].layers[0][0].to_qkv.register_forward_hook(lambda *a: None)
    assert "hooks" in m.fused_reason(torch.zeros(2, 3, 112, 112))
    h.remove()
    monkeypatch.undo()
    m32 = small()
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    assert "dtype" in m32.fused_reason(torch.zeros(1, 3, 112, 112))


# ------------------------------------------------------------------------------------------------ engine description
def test_window_token_records_of_the_readme_config():
    torch.manual_seed(0)
    m = SepViT(**README).eval()
    assert m.stage_maps(224, 224) == [(56, 56), (28, 28), (14, 14), (7, 7)]
    for i, ((_, _, tr), depth, heads, dim) in enumerate(zip(m.layers, (1, 2, 6, 2), (1, 2, 4, 8), (32, 64, 128, 256))):
        layers, norm = tr.encoder_layers()
        assert len(layers) == depth and (norm is None) == (i == 3)
        for L in layers:
            assert (L.heads, L.dim_head, L.scale) == (heads, 32, 32 ** -0.5)
            assert L.qkv_w.shape == (3 * heads * 32, dim) and L.fc1_w.shape == (4 * dim, dim)
            assert L.attention.window == 7 and L.attention.wqk_w.shape == (2 * heads * 32, heads * 32)
            assert attention_kernel(L) == "window_token"
            with pytest.raises(ValueError):
                attention_kernel(L, axial=True)
        eng = tr.engine()
        assert eng.unsupported_reason(56 * 56, grid=(56, 56)) is None
        t = eng.prepared()
        assert t["c_layers"] is None                                   # the per-kernel loop
        L, W = layers[0], layers[0].qkv_w.float()
        assert torch.equal(t["0.tok_qkv"], (W @ L.attention.token.float()).bfloat16())


def test_run_blocks_rejects_grids_before_touching_x(monkeypatch):
    import types
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: types.SimpleNamespace(cuda_stream=0))
    tr = small().layers[0][2]
    eng = tr.engine()
    x = torch.arange(2 * 96 * 32, dtype=torch.float32).view(-1, 32)
    keep = x.clone()
    for grid, what in (((8, 12), "cannot be cut"), (None, "needs `grid`"), ((4, 24), "cannot be cut")):
        with pytest.raises(ValueError, match=what):
            eng.run_blocks(x, 2, 96, grid=grid)
    with pytest.raises(ValueError, match="more than 64"):
        eng.run_blocks(torch.zeros(1 * 63 * 63 * 2, 32), 2, 63 * 63, grid=(63, 63))
    assert torch.equal(x, keep)


# ------------------------------------------------------------------------------------------------ argument checks
def test_attention_window_token_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)

    def call(*, qkv=p, tok=p, out=p, tok_out=None, B=2, gh=14, gw=21, w=7, H=2, dh=32):
        rc = lib.b200vit_attention_window_token(qkv, tok, out, tok_out, B, gh, gw, w, H, dh, 0.17, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(qkv=None), dict(tok=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(dh=48), b"dim_head=48"), (dict(B=0), b"bad shape"), (dict(H=0), b"bad shape"),
                     (dict(w=0), b"bad shape"), (dict(gh=16, gw=16, w=8), b"p=8"), (dict(gh=15), b"not divisible"),
                     (dict(H=65536), b"exceeds the grid"), (dict(tok_out=ctypes.c_void_p(264)), b"16-byte aligned"),
                     (dict(tok=ctypes.c_void_p(260)), b"16-byte aligned")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_window_mix_rejects_bad_arguments(lib):
    p, q = ctypes.c_void_p(256), ctypes.c_void_p(4096)

    def call(*, wqk=p, o=p, out=q, B=2, gh=14, gw=21, w=7, H=2, dh=32):
        rc = lib.b200vit_window_mix(wqk, o, out, B, gh, gw, w, H, dh, 0.17, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(wqk=None), dict(o=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(dh=16), b"dim_head=16"), (dict(B=0), b"bad shape"), (dict(gh=15), b"not divisible"),
                     (dict(gh=7, gw=7), b"1 windows"), (dict(gh=72, gw=72, w=8), b"81 windows"),
                     (dict(out=p), b"must not be o"), (dict(wqk=ctypes.c_void_p(264)), b"16-byte aligned")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_head_layernorm_gelu_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)

    def call(*, buf=p, ld=64, gamma=p, beta=p, T=4, nh=2, dh=32):
        rc = lib.b200vit_head_layernorm_gelu(buf, ld, gamma, beta, T, nh, dh, 1e-5, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(buf=None), dict(gamma=None), dict(beta=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(dh=48), b"dim_head=48"), (dict(T=0), b"bad shape"), (dict(nh=0), b"bad shape"),
                     (dict(ld=32), b"ld=32"), (dict(ld=68), b"ld=68"), (dict(beta=ctypes.c_void_p(260)), b"aligned")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


NEW = ("attention_window_token", "window_mix", "head_layernorm_gelu")


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in NEW:
        assert f"int b200vit_{name}(" in h and f"b200vit_{name}" in _lib.SYMBOLS


def test_library_exports_the_new_entry_points(lib):
    for name in NEW:
        assert hasattr(lib, f"b200vit_{name}")


# ------------------------------------------------------------------------------------------------ launch sequence
@pytest.fixture(scope="module")
def schedule():
    with open(SS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [SS.run_name(m, h) for m, h in SS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", SS.RUNS)
def test_fused_forward_schedule_matches_fixture(lib, schedule, ln_mode, host_loop):
    name = SS.run_name(ln_mode, host_loop)
    got, want = SS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"


@pytest.mark.parametrize("ln_mode,host_loop", SS.RUNS)
def test_window_token_launches(lib, ln_mode, host_loop):
    calls = SS.record(ln_mode, host_loop)
    names = [c["call"] for c in calls]
    assert names[:2] == ["conv_im2col_nchw", "gemm"] and names[-3:] == ["mean_pool", "layernorm", "gemm"]
    att = [c for c in calls if c["call"] == "attention_window_token"]
    assert [(c["gh"], c["gw"], c["p"]) for c in att] == [(28, 14, 7), (14, 7, 7), (14, 7, 7)]
    assert names.count("window_mix") == 3 and names.count("head_layernorm_gelu") == 3
    assert names.count("peg") == 2 and names.count("conv_im2col_nhwc") == 1
    assert "encoder_blocks" not in names


def test_other_families_schedule_fixtures_are_unchanged(lib):
    """Every other family's pinned launch sequence, regenerated, is byte-identical to its fixture."""
    for mod in ("make_engine_schedule", "make_cct_schedule", "make_pit_schedule", "make_levit_schedule",
                "make_twins_svt_schedule", "make_max_vit_schedule", "make_cvt_schedule",
                "make_crossformer_schedule", "make_mobile_vit_schedule"):
        g = importlib.import_module(mod)
        with open(g.FIXTURE) as f:
            assert S.dumps(g.generate()) == f.read(), mod
