"""CrossFormer (vit_pytorch_b200.crossformer) without a GPU: the attribute and state_dict surface, the dynamic position
bias table against the reference's `biases[rel_pos_indices]` in fp64, the stage-1 weight packing and the map geometry,
the engine's description of the layers and the table's refresh, the fallback rules, that the eager graph raises where
the reference does, the argument checks of b200vit_cross_embed_nchw, and the launch sequence of the whole fused forward
(tests/golden/crossformer_schedule.json, made by make_crossformer_schedule.py).  The reference-parity tests are in
test_crossformer_parity.py."""
import copy
import ctypes
import importlib
import json
import os
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from vit_pytorch_b200 import _lib, build, crossformer as cf
from vit_pytorch_b200.crossformer import Attention, CrossEmbedLayer, CrossFormer, dpb_table, embed_weights
from vit_pytorch_b200.engine import attention_kernel

sys.path.insert(0, GOLDEN_DIR)
from crossformer_spec import SMALL  # noqa: E402
import make_crossformer_schedule as CS  # noqa: E402
import make_engine_schedule as S  # noqa: E402

README = dict(dim=(64, 128, 256, 512), depth=(2, 2, 8, 2), global_window_size=(8, 4, 2, 1), local_window_size=7)


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


# ------------------------------------------------------------------------------------------------ module surface
def test_module_surface():
    m = CrossFormer(**SMALL)
    assert set(cf.__all__) >= {"Attention", "CrossEmbedLayer", "CrossFormer", "DynamicPositionBias", "FeedForward",
                               "LayerNorm", "Transformer", "cast_tuple"}
    sd = m.state_dict()
    assert not any("rel_pos_indices" in k for k in sd)
    a = m.layers[0][1].layers[0][0]
    assert "rel_pos_indices" in dict(a.named_buffers())
    assert [n for n, _ in a.named_children()] == ["norm", "dropout", "to_qkv", "to_out", "dpb"]
    assert [k for k in sd if k.startswith("layers.0.1.layers.0.0.dpb.")][:4] == [
        "layers.0.1.layers.0.0.dpb.0.weight", "layers.0.1.layers.0.0.dpb.0.bias",
        "layers.0.1.layers.0.0.dpb.1.weight", "layers.0.1.layers.0.0.dpb.1.bias"]
    assert [c.out_channels for c in m.layers[0][0].convs] == [32, 16, 8, 8]
    assert [c.kernel_size[0] for c in m.layers[0][0].convs] == [4, 8, 16, 32]
    assert isinstance(m.to_logits[1], torch.nn.Linear)
    assert cf.cast_tuple(3, 4) == (3, 3, 3, 3) and cf.cast_tuple((1, 2), 4) == (1, 2)


# ------------------------------------------------------------------------------------------------ position bias table
@pytest.mark.parametrize("w", range(1, 9))
def test_dpb_table_is_the_references_first_outputs(w):
    """The table b200vit_attention_window_relpos reads, looked up the kernel's way ((du + w - 1)(2w - 1) + dv + w - 1
    for the signed offset (du, dv) of query and key), equals biases[rel_pos_indices] of the reference's graph in
    fp64: the first (2w - 1)^2 of the (2w + 1)^2 outputs, for every head."""
    torch.manual_seed(w)
    a = Attention(96, 'short', w).eval()
    with torch.no_grad():
        for p in a.dpb.parameters():
            p.add_(torch.randn_like(p) * 0.3)
    a = a.to(torch.bfloat16)                         # the table is built in fp32 from the bf16 parameters
    table = dpb_table(a)
    assert table.dtype == torch.float32 and table.shape == ((2 * w - 1) ** 2, a.heads) == ((2 * w - 1) ** 2, 3)
    a64 = copy.deepcopy(a).double()
    with torch.no_grad():
        biases = a64.dpb(cf._rel_offsets(w, "cpu").double())
    assert biases.shape == ((2 * w + 1) ** 2,)
    ref = biases[a64.rel_pos_indices]                # [w^2, w^2]
    r = torch.arange(w * w)
    u, v = r // w, r % w
    idx = (u[:, None] - u[None, :] + w - 1) * (2 * w - 1) + (v[:, None] - v[None, :] + w - 1)
    for h in range(a.heads):
        got = table[:, h].double()[idx]
        assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5), (w, h, (got - ref).abs().max())
    assert torch.equal(table[:, 0], table[:, 2])


def test_dpb_update_rebuilds_the_prepared_table():
    m = CrossFormer(**SMALL).eval()
    eng = m.layers[1][1].engine()
    t0 = eng.prepared()["1.relpos"].clone()
    assert t0.shape == (2, 49)                       # stage 2: 2 heads of 32, global window 4
    with torch.no_grad():
        m.layers[1][1].layers[0][2].dpb[0].weight.mul_(2.0)
    t1 = eng.prepared()["1.relpos"]
    assert not torch.equal(t0, t1)
    assert torch.equal(t1, dpb_table(m.layers[1][1].layers[0][2]).t())


# ------------------------------------------------------------------------------------------------ weights and maps
def test_stage1_weight_packing():
    cel = CrossEmbedLayer(3, 64, (4, 8, 16, 32), stride=4)
    t = embed_weights(cel, True)
    w = t["w"]
    off = 0
    for c in cel.convs:
        n, K = c.out_channels, c.weight[0].numel()
        kp = (K + 63) // 64 * 64
        blk = w[off:off + n * kp].reshape(n, kp)
        assert torch.equal(blk[:, :K], c.weight.detach().reshape(n, K).bfloat16())
        assert not blk[:, K:].any()
        off += n * kp
    assert off == w.numel() and torch.equal(t["b"], torch.cat([c.bias.detach() for c in cel.convs]))
    # C = 1, k = 2: K = 4 padded to 64
    one = _lib.cross_embed_pack([torch.ones(8, 1, 2, 2)])
    assert one.shape == (8 * 64,) and one.reshape(8, 64)[:, :4].all() and not one.reshape(8, 64)[:, 4:].any()
    # a later stage: columns (tap row, tap column, channel) of conv_im2col_nhwc
    cel2 = CrossEmbedLayer(64, 128, (2, 4), stride=2)
    t2 = embed_weights(cel2, False)
    c = cel2.convs[1]
    assert torch.equal(t2["w1"], c.weight.detach().permute(0, 2, 3, 1).reshape(64, -1).bfloat16())


def test_stage_maps_match_the_convolutions():
    m = CrossFormer(**README)
    maps = m.stage_maps(224, 224)
    assert [ms[0] for ms in maps] == [(56, 56), (28, 28), (14, 14), (7, 7)] and all(len(set(ms)) == 1 for ms in maps)
    x = torch.zeros(1, 3, 64, 128)
    s = CrossFormer(**dict(SMALL, global_window_size=(8, 4, 2, 1)))
    for (cel, _), ms in zip(s.layers, s.stage_maps(64, 128)):
        shapes = {tuple(conv(x).shape[2:]) for conv in cel.convs}
        assert shapes == set(ms)
        x = torch.zeros(1, cel.convs[0].out_channels * 0 + sum(c.out_channels for c in cel.convs), *ms[0])
    odd = CrossFormer(**dict(SMALL, cross_embed_kernel_sizes=((4, 8), (2, 3), (2, 4), (2, 4))))
    assert len(set(odd.stage_maps(64, 64)[1])) == 2 and len(odd.stage_maps(64, 64)) == 2


# ------------------------------------------------------------------------------------------------ engine description
def test_window_records_of_the_readme_config():
    m = CrossFormer(**README)
    layers = [L for _, t in m.layers for L in t.encoder_layers()[0]]
    assert len(layers) == 28
    assert [L.attention.dilated for L in layers] == [False, True] * 14
    wins = [(L.attention.size, L.attention.dilated) for _, t in m.layers for L in t.encoder_layers()[0][:2]]
    assert wins == [(7, False), (8, True), (7, False), (4, True), (7, False), (2, True), (7, False), (1, True)]
    assert {attention_kernel(L) for L in layers} == {"window_relpos"}
    assert [(L.heads, L.dim_head) for L in layers[::4]][:4] == [(2, 32), (4, 32), (8, 32), (8, 32)]
    L = layers[0]
    assert L.attention.rel_pos_bias.shape == (13 * 13, 2) and L.qkv_w.shape == (192, 64) and L.out_w.shape == (64, 64)
    assert L.fc1_w.shape == (256, 64) and L.fc2_w.shape == (64, 256) and L.ln1.eps == 1e-5


def test_inner_width_below_dim():
    m = CrossFormer(**dict(SMALL, dim=(64, 80, 112, 144)))
    L = m.layers[1][1].encoder_layers()[0][0]
    assert (L.heads, L.dim_head) == (2, 32) and L.qkv_w.shape == (192, 80) and L.out_w.shape == (80, 64)
    assert [c.out_channels for c in m.layers[1][0].convs] == [40, 40]


# ------------------------------------------------------------------------------------------------ fallback rules
@pytest.fixture
def eligible(monkeypatch):
    """fused_reason with the device / dtype / autograd part passed, so its shape rules can be checked on CPU."""
    monkeypatch.setattr(cf, "common_reason", lambda *a, **k: None)


def test_fused_reason_rules_with_the_engine_window_limit(eligible):
    img = lambda h, w, c=3: torch.zeros(2, c, h, w)                        # noqa: E731
    mk = lambda **kw: CrossFormer(**dict(SMALL, **kw)).eval()               # noqa: E731
    m = mk()
    assert m.fused_reason(img(64, 64)) is None and m.fused_reason(img(64, 128)) is None
    assert CrossFormer(**README).eval().fused_reason(img(224, 224)) is None
    assert "not (B, 3, H, W)" in m.fused_reason(torch.zeros(3, 64, 64))
    assert "not (B, 3, H, W)" in m.fused_reason(img(64, 64, c=1))
    assert mk(channels=1).fused_reason(img(64, 64, c=1)) is None
    assert "window_size=9: a window of 81 tokens" in mk(local_window_size=9).fused_reason(img(576, 576))
    assert "window_size=9: a window of 81 tokens" in mk(global_window_size=(9, 1, 1, 1)).fused_reason(img(576, 576))
    assert "not divisible" in m.fused_reason(img(48, 48))
    assert "not divisible" in mk(global_window_size=(3, 1, 1, 1)).fused_reason(img(64, 64))
    assert "torch.cat raises" in mk(cross_embed_kernel_sizes=((4, 8), (2, 3), (2, 4), (2, 4))).fused_reason(
        img(64, 64))
    assert "stage 1" in mk(cross_embed_kernel_sizes=((4, 36), (2, 4), (2, 4), (2, 4))).fused_reason(img(64, 64))
    assert "stage 1" in mk(cross_embed_kernel_sizes=((2, 4, 8, 16, 32), (2, 4), (2, 4), (2, 4))).fused_reason(
        img(64, 64))
    assert "stage 1" in mk(channels=5).fused_reason(img(64, 64, c=5))
    assert "stage 1" in mk(dim=(256, 64, 96, 128), cross_embed_kernel_sizes=((4, 8), (2, 4), (2, 4), (2, 4))
                           ).fused_reason(img(64, 64))                  # a stem scale of width 128
    assert "at most 16" in mk(cross_embed_kernel_sizes=((4, 8), (2, 18), (2, 4), (2, 4))).fused_reason(img(64, 64))
    assert "multiples of 8" in mk(dim=(64, 68, 96, 128)).fused_reason(img(64, 64))
    assert "multiples of 8" in mk(dim=(96, 64, 96, 128)).fused_reason(img(64, 64))   # stem 48 / 24 / 12 / 12
    assert "no attention heads" in mk(dim=(64, 16, 96, 128)).fused_reason(img(64, 64))
    assert "empty" in mk(local_window_size=1, global_window_size=1).fused_reason(img(8, 8))
    assert "> 16384" in mk(local_window_size=1, global_window_size=1).fused_reason(img(520, 520))
    assert mk(attn_dropout=0.1, ff_dropout=0.1).fused_reason(img(64, 64)) is None


def test_fused_reason_common_rules():
    m = CrossFormer(**SMALL).eval()
    assert "CUDA" in m.fused_reason(torch.zeros(2, 3, 64, 64))
    assert "depth == 0" in CrossFormer(**dict(SMALL, depth=(1, 0, 1, 1))).eval().fused_reason(
        torch.zeros(2, 3, 64, 64))


# ------------------------------------------------------------------------------------------------ raise parity
def test_eager_graph_raises_where_the_reference_does():
    torch.manual_seed(0)
    m = CrossFormer(**SMALL).eval()
    with torch.inference_mode():
        with pytest.raises(RuntimeError, match="same dtype"):
            copy.deepcopy(m).bfloat16()(torch.randn(1, 3, 64, 64).bfloat16())
        with pytest.raises(RuntimeError, match="not divisible"):
            m(torch.randn(1, 3, 48, 48))
        odd = CrossFormer(**dict(SMALL, cross_embed_kernel_sizes=((4, 8), (2, 3), (2, 4), (2, 4)))).eval()
        with pytest.raises(RuntimeError, match="Sizes of tensors must match"):
            odd(torch.randn(1, 3, 64, 64))


# ------------------------------------------------------------------------------------------------ argument checks
def test_cross_embed_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(1 << 20)

    def call(*, img=p, w=p, bias=p, out=p, ldo=64, B=2, C=3, H=64, W=64, ks=(4, 8, 16, 32), ns=(32, 16, 8, 8), s=4):
        S_ = len(ks)
        rc = lib.b200vit_cross_embed_nchw(img, w, bias, out, ldo, B, C, H, W, S_, (ctypes.c_int * S_)(*ks),
                                          (ctypes.c_int * S_)(*ns), s, None)
        return rc, lib.b200vit_last_error()
    for kw in (dict(img=None), dict(w=None), dict(bias=None), dict(out=None)):
        rc, msg = call(**kw)
        assert rc == -1 and b"null" in msg, kw
    for kw, what in ((dict(B=0), b"bad shape"), (dict(C=5), b"bad shape"), (dict(C=0), b"bad shape"),
                     (dict(ks=(2, 4, 8, 16, 32), ns=(8,) * 5), b"5 scales"), (dict(s=9), b"stride 9"),
                     (dict(s=0), b"stride 0"), (dict(ks=(4, 36), ns=(32, 32)), b"kernel 36"),
                     (dict(ks=(2, 8), ns=(32, 32)), b"kernel 2"), (dict(ns=(32, 16, 8, 4)), b"width 4"),
                     (dict(ks=(4, 64), ns=(32, 32)), b"kernel 64"), (dict(ks=(4,), ns=(72,), ldo=72), b"width 72"),
                     (dict(ks=(4, 7), ns=(32, 32)), b"maps to"), (dict(H=2), b"exceeds"),
                     (dict(ldo=60), b"ldo=60"), (dict(ldo=65), b"ldo=65"),
                     (dict(w=ctypes.c_void_p((1 << 20) + 8)), b"aligned"),
                     (dict(out=ctypes.c_void_p((1 << 20) + 4)), b"aligned")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_header_declares_the_new_entry_point():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    assert "int b200vit_cross_embed_nchw(" in h and "b200vit_cross_embed_nchw" in _lib.SYMBOLS
    for name, v in (("SCALES", _lib.CROSS_EMBED_MAX_SCALES), ("KERNEL", _lib.CROSS_EMBED_MAX_KERNEL),
                    ("CHANNELS", _lib.CROSS_EMBED_MAX_CHANNELS), ("STRIDE", _lib.CROSS_EMBED_MAX_STRIDE),
                    ("WIDTH", _lib.CROSS_EMBED_MAX_WIDTH)):
        assert f"#define B200VIT_CROSS_EMBED_MAX_{name} {v} " in h


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
def test_cross_embedding_and_window_launches(lib, ln_mode, host_loop):
    calls = CS.record(ln_mode, host_loop)
    names = [c["call"] for c in calls]
    assert names[0] == "cross_embed_nchw" and names.count("cross_embed_nchw") == 1
    assert names[-3:] == ["mean_pool", "cast_f32_bf16", "gemm"]
    # stages 2 to 4: per scale, im2col of the previous stream copy and a GEMM into the scale's column slice
    im = [i for i, n in enumerate(names) if n == "conv_im2col_nhwc"]
    assert len(im) == 6 and all(names[i + 1] == "gemm" for i in im)
    slices = [(calls[i + 1]["out_f32"]["offset"], calls[i + 1]["out_f32"]["shape"], calls[i + 1]["out_f32"]["stride"])
              for i in im]
    assert slices == [(0, [128, 16], [32, 1]), (16 * 4, [128, 16], [32, 1]), (0, [32, 24], [48, 1]),
                      (24 * 4, [32, 24], [48, 1]), (0, [8, 32], [64, 1]), (32 * 4, [8, 32], [64, 1])]
    rel = [c for c in calls if c["call"] == "attention_window_relpos"]
    assert [(c["gh"], c["w"], c["grid"]) for c in rel] == [(16, 2, False), (16, 2, True), (8, 2, False),
                                                         (8, 2, True), (4, 2, False), (4, 1, True), (2, 2, False),
                                                         (2, 2, True)]
    assert names.count("embed_tokens") == 0


def test_other_families_schedule_fixtures_are_unchanged(lib):
    """Every other family's pinned launch sequence, regenerated, is byte-identical to its fixture."""
    for mod in ("make_engine_schedule", "make_cct_schedule", "make_pit_schedule", "make_levit_schedule",
                "make_twins_svt_schedule", "make_max_vit_schedule", "make_cvt_schedule"):
        g = importlib.import_module(mod)
        with open(g.FIXTURE) as f:
            assert S.dumps(g.generate()) == f.read(), mod
