"""RegionViT (vit_pytorch_b200.regionvit) without a GPU: the module surface and that the eager graph raises where the
reference does, a pure-torch fp64 emulation of the fused dataflow of one R2L layer (the stream's row layout, the
region rows' attention as pointer offsets, the kernel's window address map and bias index) against R2LTransformer's
PyTorch graph, the fallback rules, the engine description, the argument checks of the new entry point, and the launch
sequence of the whole fused forward (tests/golden/regionvit_schedule.json, made by make_regionvit_schedule.py).  The
reference-parity tests are in test_regionvit_parity.py."""
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build, regionvit as rv
from vit_pytorch_b200.engine import attention_kernel
from vit_pytorch_b200.regionvit import R2LTransformer, RegionViT

sys.path.insert(0, GOLDEN_DIR)
import make_engine_schedule as S  # noqa: E402
import make_regionvit_schedule as RS  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def small(**kw):
    torch.manual_seed(0)
    return RegionViT(**dict(dict(dim=(32, 32, 64, 64), depth=1, num_classes=5), **kw)).eval()


# ------------------------------------------------------------------------------------------------ surface
def test_module_surface():
    assert set(rv.__all__) >= {"Attention", "ChanLayerNorm", "Downsample", "FeedForward", "PEG", "R2LTransformer",
                               "RegionViT"}
    import vit_pytorch_b200
    assert not hasattr(vit_pytorch_b200, "RegionViT")          # the reference package does not export it either
    m = small(tokenize_local_3_conv=True, use_peg=True)
    names = [n for n, _ in m.named_parameters()]
    assert names[:8] == ["local_encoder.0.weight", "local_encoder.0.bias", "local_encoder.1.g", "local_encoder.1.b",
                         "local_encoder.3.weight", "local_encoder.3.bias", "local_encoder.4.g", "local_encoder.4.b"]
    assert "region_encoder.1.weight" in names and "layers.1.1.proj.weight" in names
    tr_names = [n for n, _ in m.layers[1][2].named_parameters()]
    assert tr_names[0] == "layers.0.0.norm.weight" and tr_names[-1] == "local_rel_pos_bias.weight"
    for _, _, tr in m.layers:
        assert tr.layers[0][0].heads == 4 and tr.layers[0][0].to_qkv.weight.shape[0] == 3 * 128


def test_eager_graph_raises_where_the_reference_does():
    m = small()
    with torch.no_grad():
        assert m(torch.randn(1, 3, 112, 56)).shape == (1, 5)
        with pytest.raises(AssertionError, match="region patch size"):
            m(torch.randn(1, 3, 100, 112))
        with pytest.raises(RuntimeError):
            m(torch.randn(1, 3, 84, 84))                     # stage 2: an 11 x 11 local map, a 2 x 2 region map
    with pytest.raises(AssertionError):
        RegionViT(dim=(32, 64, 128))


# ------------------------------------------------------------------------------------------------ fp64 dataflow
def fused_dataflow(tr: R2LTransformer, local: torch.Tensor, region: torch.Tensor):
    """tr(local, region) as the fused path computes it, in fp64: one stream of B*lh*lw local rows (b, y, x) then
    B*rh*rw region rows (b, i, j); per layer the region rows' attention over each image's region tokens and residual,
    then attention_region_local's address map -- window (b, i, j) = region row B*lh*lw + (b*rh + i)*rw + j and the
    local rows ((b*lh + i*wh + u)*lw + j*ww + v) -- with bias table^T[h][(du + W-1) + (dv + W-1)*(2W-1)] between local
    tokens, then the feed-forward over all rows."""
    B, c, lh, lw = local.shape
    rh, rw = region.shape[2:]
    wh, ww, W = lh // rh, lw // rw, tr.window_size
    Ml = B * lh * lw
    x = torch.cat((local.permute(0, 2, 3, 1).reshape(-1, c), region.permute(0, 2, 3, 1).reshape(-1, c)))
    table = tr.local_rel_pos_bias.weight.t()                        # [H, (2W-1)^2]
    ln = torch.nn.functional.layer_norm
    for attn, ff in tr.layers:
        H, dh = attn.heads, attn.dim_head
        I = H * dh
        Wq = attn.to_qkv.weight

        def proj(rows):
            return ln(rows, (c,), attn.norm.weight, attn.norm.bias, attn.norm.eps) @ Wq.t()

        def out(o):
            return o @ attn.to_out[0].weight.t() + attn.to_out[0].bias

        qkv = proj(x[Ml:])
        o = torch.empty(B * rh * rw, I, dtype=x.dtype)
        for b in range(B):
            r = slice(b * rh * rw, (b + 1) * rh * rw)
            for h in range(H):
                q, k, v = (qkv[r, j * I + h * dh:j * I + (h + 1) * dh] for j in range(3))
                o[r, h * dh:(h + 1) * dh] = torch.softmax(q @ k.t() * attn.scale, -1) @ v
        x = x.clone()
        x[Ml:] = x[Ml:] + out(o)
        qkv = proj(x)
        o = torch.empty(x.shape[0], I, dtype=x.dtype)
        for b in range(B):
            for i in range(rh):
                for j in range(rw):
                    rows = [Ml + (b * rh + i) * rw + j] + [(b * lh + i * wh + u) * lw + j * ww + v
                                                           for u in range(wh) for v in range(ww)]
                    n = len(rows)
                    bias = torch.zeros(H, n, n, dtype=x.dtype)
                    for t1 in range(1, n):
                        for t2 in range(1, n):
                            (u1, v1), (u2, v2) = divmod(t1 - 1, ww), divmod(t2 - 1, ww)
                            bias[:, t1, t2] = table[:, (u1 - u2 + W - 1) + (v1 - v2 + W - 1) * (2 * W - 1)]
                    for h in range(H):
                        q, k, v = (qkv[rows, jj * I + h * dh:jj * I + (h + 1) * dh] for jj in range(3))
                        o[rows, h * dh:(h + 1) * dh] = torch.softmax(q @ k.t() * attn.scale + bias[h], -1) @ v
        x = x + out(o)
        f = ff
        hdn = torch.nn.functional.gelu(ln(x, (c,), f[0].weight, f[0].bias, f[0].eps) @ f[1].weight.t() + f[1].bias)
        x = x + hdn @ f[4].weight.t() + f[4].bias
    loc = x[:Ml].view(B, lh, lw, c).permute(0, 3, 1, 2)
    reg = x[Ml:].view(B, rh, rw, c).permute(0, 3, 1, 2)
    return loc, reg


@pytest.mark.parametrize("W,local_hw,region_hw", [(7, (14, 7), (2, 1)),       # square 7 x 7 windows
                                                  (7, (7, 8), (1, 2)),        # non-square 7 x 4 windows
                                                  (14, (14, 14), (1, 1)),     # a 14 x 14 window, 197 tokens
                                                  (7, (4, 6), (2, 3))])       # 2 x 2 windows under a W = 7 table
def test_fused_dataflow_matches_the_r2l_transformer_in_fp64(W, local_hw, region_hw):
    torch.manual_seed(W + local_hw[1])
    tr = R2LTransformer(16, window_size=W, depth=2, heads=2, dim_head=8).double().eval()
    with torch.no_grad():
        for prm in tr.parameters():
            prm.add_(0.1 * torch.randn(prm.shape, dtype=torch.float64))
        local = torch.randn(2, 16, *local_hw, dtype=torch.float64)
        region = torch.randn(2, 16, *region_hw, dtype=torch.float64)
        want = tr.forward_eager(local, region)
        got = fused_dataflow(tr, local, region)
    for g, w in zip(got, want):
        assert (g - w).abs().max().item() < 1e-10


# ------------------------------------------------------------------------------------------------ fallback rules
def test_fused_reason_rules(monkeypatch):
    x = torch.zeros(2, 3, 112, 112, dtype=torch.bfloat16)
    m = small().bfloat16()
    assert m.fused_reason(x) == "input is not on a CUDA device"
    monkeypatch.setattr(rv, "common_reason", lambda *a, **k: None)
    assert m.fused_reason(x) is None
    assert "channels" in m.fused_reason(torch.zeros(2, 1, 112, 112))
    assert "channels=4" in small(channels=4).fused_reason(x)
    assert "not divisible" in m.fused_reason(torch.zeros(2, 3, 100, 112))
    assert "does not split" in m.fused_reason(torch.zeros(1, 3, 84, 84))
    assert "multiples of 8" in small(dim=(36, 32, 64, 64)).fused_reason(x)
    assert "dim[0]=48" in small(dim=(48, 32, 64, 64), tokenize_local_3_conv=True).fused_reason(x)
    assert small(dim=(64, 32, 64, 64), tokenize_local_3_conv=True).fused_reason(x) is None
    big = small(window_size=16)                  # a 16 x 16 window of 256 local tokens in stage 1
    assert "at most 255" in big.fused_reason(torch.zeros(1, 3, 256, 256))
    assert small(window_size=14).fused_reason(torch.zeros(1, 3, 224, 224)) is None
    wide = small()
    wide.layers[0][2].layers[0][0].dim_head = 64                        # as an Attention built with dim_head=64
    assert "dim_head=64" in wide.fused_reason(x)
    m.train()
    assert "training" in m.fused_reason(x)
    m.eval()
    assert small(attn_dropout=0.1, ff_dropout=0.2).fused_reason(x) is None
    tr = m.layers[0][2]
    assert "(b, c, h, w)" in tr.fused_reason(torch.zeros(2, 28, 32), torch.zeros(2, 32, 4, 4))


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
    assert "autograd" in small().bfloat16().requires_grad_(True).fused_reason(
        torch.zeros(1, 3, 112, 112, dtype=torch.bfloat16))


# ------------------------------------------------------------------------------------------------ engine description
def test_region_local_records_of_the_readme_config():
    torch.manual_seed(0)
    m = RegionViT().eval()
    assert m.stage_maps(224, 224) == [(56, 56, 8, 8), (28, 28, 4, 4), (14, 14, 2, 2), (7, 7, 1, 1)]
    assert m.stage_maps(224, 112)[-1] == (7, 4, 1, 1)
    for (_, _, tr), depth, dim in zip(m.layers, (2, 2, 8, 2), (64, 128, 256, 512)):
        layers, norm = tr.encoder_layers()
        assert len(layers) == depth and norm is None
        for L in layers:
            assert (L.heads, L.dim_head, L.scale) == (4, 32, 32 ** -0.5)
            assert L.qkv_w.shape == (3 * 128, dim) and L.fc1_w.shape == (4 * dim, dim)
            assert L.attention.window == 7 and L.attention.bias is tr.local_rel_pos_bias.weight
            assert attention_kernel(L) == "region_local"
            with pytest.raises(ValueError):
                attention_kernel(L, axial=True)
        t = tr.engine().prepared()
        assert t["c_layers"] is None                                   # the per-kernel loop
        assert torch.equal(t["0.r2l"], tr.local_rel_pos_bias.weight.float().t())


def test_run_blocks_rejects_grids_before_touching_x(monkeypatch):
    import types
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: types.SimpleNamespace(cuda_stream=0))
    tr = small().layers[1][2]
    eng = tr.engine()
    x = torch.arange(2 * (14 * 14 + 4) * 32, dtype=torch.float32).view(-1, 32)
    keep = x.clone()
    for kw, what in ((dict(grid=(14, 14)), "needs `grid`"), (dict(regions=(2, 2)), "needs `grid`"),
                     (dict(grid=(14, 14), regions=(3, 3)), "rows")):
        with pytest.raises(ValueError, match=what):
            eng.run_blocks(x, 2, 14 * 14, **kw)
    for grid, regions, what in (((14, 14), (1, 4), "does not split"), ((16, 8), (2, 2), "larger than window_size"),
                                ((28, 14), (2, 1), "larger than window_size")):
        y = torch.zeros(2 * (grid[0] * grid[1] + regions[0] * regions[1]), 32)
        with pytest.raises(ValueError, match=what):
            eng.run_blocks(y, 2, grid[0] * grid[1], grid=grid, regions=regions)
        assert not y.any()
    y = torch.zeros(1 * (16 * 16 + 1), 32)
    tr.window_size = 16                                                # as a table built for window 16
    eng.prep.key = None                                                # the layer description is rebuilt
    with pytest.raises(ValueError, match="at most 255"):
        eng.run_blocks(y, 1, 256, grid=(16, 16), regions=(1, 1))
    assert torch.equal(x, keep)


# ------------------------------------------------------------------------------------------------ argument checks
def test_attention_region_local_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)

    def call(*, qkv=p, out=p, table=p, B=2, lh=14, lw=21, rh=2, rw=3, W=7, H=4, dh=32):
        rc = lib.b200vit_attention_region_local(qkv, out, table, B, lh, lw, rh, rw, W, H, dh, 0.17, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(qkv=None), dict(out=None), dict(table=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(dh=64), b"dim_head=64"), (dict(B=0), b"bad shape"), (dict(H=0), b"bad shape"),
                     (dict(rh=0), b"bad shape"), (dict(W=0), b"bad shape"), (dict(lh=15), b"not divisible"),
                     (dict(lw=20), b"not divisible"), (dict(W=6), b"window_size=6"),
                     (dict(lh=32, lw=32, rh=2, rw=2, W=16), b"256 tokens"), (dict(H=65536), b"exceeds the grid"),
                     (dict(table=ctypes.c_void_p(260)), b"16-byte aligned"),
                     (dict(out=ctypes.c_void_p(264)), b"16-byte aligned")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_header_declares_the_new_entry_point():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    assert "int b200vit_attention_region_local(" in h and "b200vit_attention_region_local" in _lib.SYMBOLS


def test_library_exports_the_new_entry_point(lib):
    assert hasattr(lib, "b200vit_attention_region_local")


# ------------------------------------------------------------------------------------------------ launch sequence
@pytest.fixture(scope="module")
def schedule():
    with open(RS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [RS.run_name(m, h) for m, h in RS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", RS.RUNS)
def test_fused_forward_schedule_matches_fixture(lib, schedule, ln_mode, host_loop):
    name = RS.run_name(ln_mode, host_loop)
    got, want = RS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"


@pytest.mark.parametrize("ln_mode,host_loop", RS.RUNS)
def test_region_local_launches(lib, ln_mode, host_loop):
    calls = RS.record(ln_mode, host_loop)
    names = [c["call"] for c in calls]
    assert names[:3] == ["conv_im2col_nchw", "gemm", "head_layernorm_gelu"]
    assert names[-3:] == ["mean_pool", "layernorm", "gemm"]
    r2l = [c for c in calls if c["call"] == "attention_region_local"]
    assert [(c["lh"], c["lw"], c["rh"], c["rw"]) for c in r2l] == [(28, 14, 4, 2), (14, 7, 2, 1), (14, 7, 2, 1),
                                                                    (7, 4, 1, 1), (4, 2, 1, 1)]
    assert [(c["B"], c["N"]) for c in calls if c["call"] == "attention"] == [(2, 8), (2, 2), (2, 2), (2, 1), (2, 1)]
    assert names.count("patchify_nd") == 1 and names.count("peg") == 3 and names.count("conv_im2col_nhwc") == 2 + 6
    assert names.count("head_layernorm_gelu") == 2 and "encoder_blocks" not in names


def test_other_families_schedule_fixtures_are_unchanged(lib):
    """Every other family's pinned launch sequence, regenerated, is byte-identical to its fixture."""
    for mod in ("make_engine_schedule", "make_cct_schedule", "make_pit_schedule", "make_levit_schedule",
                "make_twins_svt_schedule", "make_max_vit_schedule", "make_cvt_schedule",
                "make_crossformer_schedule", "make_mobile_vit_schedule", "make_sep_vit_schedule"):
        g = importlib.import_module(mod)
        with open(g.FIXTURE) as f:
            assert S.dumps(g.generate()) == f.read(), mod
