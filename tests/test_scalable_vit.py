"""ScalableViT without a GPU: the reference's errors in the eager graph, how the encoder describes its layers to the
engine (padded key heads, the FeedForward-first second half, the records), an fp64 emulation of the fused dataflow
against the reference's logits on every golden case, the engine's reasons for the kernels' limits, the argument checks
of b200vit_attention_kv_ex and b200vit_attention_iwsa, and the pinned launch sequence
(tests/golden/scalable_vit_schedule.json, made by make_scalable_vit_schedule.py)."""
import ctypes
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_DIR, load_golden
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.engine import InteractiveWindows, StridedKV
from vit_pytorch_b200.scalable_vit import ScalableViT, Transformer, padded_key_width

sys.path.insert(0, GOLDEN_DIR)
import make_scalable_vit_schedule as SS  # noqa: E402
from scalable_vit_spec import FAMILY, SCALABLE_VIT_CASES  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


def test_eager_raises_the_reference_window_assertion():
    m = ScalableViT(num_classes=3, dim=32, heads=1, depth=(1,), reduction_factor=2, window_size=5).eval()
    with torch.no_grad(), pytest.raises(AssertionError, match=r"height \(16\) or width \(16\) of feature map is not "
                                                              r"divisible by the window size \(5, 5\)"):
        m(torch.randn(1, 3, 64, 64))


def test_eager_raises_where_the_key_convolution_is_larger_than_the_map():
    m = ScalableViT(num_classes=3, dim=32, heads=1, depth=(1,), reduction_factor=8).eval()
    with torch.no_grad(), pytest.raises(RuntimeError):
        m(torch.randn(1, 3, 16, 16))


def test_key_widths_run_padded_to_multiples_of_16():
    assert [padded_key_width(d) for d in (8, 16, 24, 32, 40, 48, 56, 64)] == [16, 16, 32, 32, 48, 48, 64, 64]


def test_encoder_layers_pad_key_heads_and_put_the_feed_forward_first():
    t = Transformer(dim=64, depth=2, heads=2, ssa_dim_key=40, ssa_dim_value=32, ssa_reduction_factor=4,
                    iwsa_dim_key=24, iwsa_dim_value=64, iwsa_window_size=8)
    layers, norm = t.encoder_layers()
    assert len(layers) == 4 and norm is not None
    for i, L in enumerate(layers):
        if i % 2 == 0:
            A = L.attention
            assert isinstance(A, StridedKV) and A.stride == 4 and A.dim_value == 32 and not L.ff_first
            assert L.dim_head == 48 and L.qkv_w.shape == (96, 64) and A.kv_w.shape == (96 + 64, 64, 4, 4)
            assert L.scale == 40 ** -0.5
            w = t.layers[i // 2][0].to_q.weight.reshape(2, 40, 64)
            q = L.qkv_w.reshape(2, 48, 64)
            assert torch.equal(q[:, :40], w) and not q[:, 40:].any()
        else:
            A = L.attention
            assert isinstance(A, InteractiveWindows) and A.size == 8 and L.ff_first
            assert L.dim_head == 32 and L.qkv_w.shape == (2 * 64 + 128, 64) and A.value_width(L) == 64
            assert L.out_w.shape == (64, 128) and L.scale == 24 ** -0.5


def test_engine_reasons_name_the_kernel_limits():
    t = Transformer(dim=32, depth=1, heads=1, ssa_dim_value=48)
    assert "dim_value=48" in t.engine().unsupported_reason(64, grid=(8, 8))
    t = Transformer(dim=32, depth=1, heads=1, iwsa_dim_key=72)
    assert "dim_key=80" in t.engine().unsupported_reason(64, grid=(8, 8))
    t = Transformer(dim=32, depth=1, heads=1, iwsa_window_size=5)
    assert "not divisible by the window size (5, 5)" in t.engine().unsupported_reason(64, grid=(8, 8))
    t = Transformer(dim=32, depth=1, heads=1, iwsa_window_size=None, ssa_reduction_factor=1)
    assert "16384" in t.engine().unsupported_reason(256 * 128, grid=(256, 128))
    assert t.engine().unsupported_reason(128 * 128, grid=(128, 128)) is None
    t = Transformer(dim=32, depth=1, heads=1, ssa_reduction_factor=4)
    assert "key patches" in t.engine().unsupported_reason(9, grid=(3, 3))


def test_attention_kv_ex_rejects_bad_arguments(lib):
    p, pkv, pout = ctypes.c_void_p(256), ctypes.c_void_p(1 << 30), ctypes.c_void_p(1 << 31)

    def call(*, q=p, ldq=96, kv=pkv, ldkv=160, out=pout, B=2, Nq=4096, Nk=64, H=2, dk=48, dv=32):
        rc = lib.b200vit_attention_kv_ex(q, ldq, kv, ldkv, out, B, Nq, Nk, H, dk, dv, 0.15, None)
        return rc, lib.b200vit_last_error()
    for kw, what in ((dict(q=None), b"null"), (dict(B=0), b"bad shape"), (dict(dk=40), b"dk=40"),
                     (dict(dv=48), b"dv=48"), (dict(Nk=16385), b"Nk=16385"), (dict(ldq=88), b"ldq=88"),
                     (dict(ldkv=152), b"ldkv=152"), (dict(out=ctypes.c_void_p(264)), b"16-byte aligned"),
                     (dict(out=ctypes.c_void_p(256 + 4096 * 2)), b"overlaps"),
                     (dict(out=ctypes.c_void_p((1 << 30) - 16)), b"overlaps")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_attention_iwsa_rejects_bad_arguments(lib):
    def call(*, qkv=ctypes.c_void_p(256), ld=192, lim=ctypes.c_void_p(1 << 30), out=ctypes.c_void_p(1 << 31), B=2,
             gh=64, gw=64, wh=64, ww=64, H=2, dk=32, dv=32):
        rc = lib.b200vit_attention_iwsa(qkv, ld, lim, out, B, gh, gw, wh, ww, H, dk, dv, 0.17, None)
        return rc, lib.b200vit_last_error()
    for kw, what in ((dict(lim=None), b"null"), (dict(wh=0), b"bad shape"), (dict(dk=40), b"dk=40"),
                     (dict(dv=16), b"dv=16"), (dict(wh=5, ww=5), b"not divisible"),
                     (dict(gh=256, gw=128, wh=256, ww=128), b"more than 16384"), (dict(ld=184), b"ld=184"),
                     (dict(ld=196), b"ld=196"), (dict(out=ctypes.c_void_p((1 << 31) + 8)), b"16-byte aligned"),
                     (dict(out=ctypes.c_void_p(256 + 64)), b"overlaps"),
                     (dict(lim=ctypes.c_void_p((1 << 31) + 1024)), b"overlaps")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)


def test_header_declares_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "b200vit.h")) as f:
        h = f.read()
    for name in ("b200vit_attention_kv_ex", "b200vit_attention_iwsa"):
        assert f"int {name}(" in h and name in _lib.SYMBOLS


# ------------------------------------------------------------------------------------------------ fp64 dataflow
def _ln(x, norm):
    return (x - x.mean(1, keepdim=True)) / (x.var(1, unbiased=False, keepdim=True) + norm.eps).sqrt() * norm.gamma + \
        norm.beta


def im2col_nhwc(x, B, H, W, k, s, p):
    """b200vit_conv_im2col_nhwc: channels-last x [B*H*W, C] -> rows (b, oy, ox), column (i*k + j)*C + c."""
    C = x.shape[1]
    m = F.pad(x.reshape(B, H, W, C), (0, 0, p, p, p, p))
    oh, ow = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    taps = [m[:, i:i + s * (oh - 1) + 1:s, j:j + s * (ow - 1) + 1:s] for i in range(k) for j in range(k)]
    return torch.cat(taps, dim=-1).reshape(B * oh * ow, k * k * C)


def conv_rows(w):
    """A Conv2d weight in im2col_nhwc's column order."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


def attend(q, k, v, H, scale):
    """softmax(scale q k^T) v per head of G sequences: q [G, n, H*dk], k [G, m, H*dk], v [G, m, H*dv]."""
    G, n, m = q.shape[0], q.shape[1], k.shape[1]
    qh, kh, vh = (t.reshape(G, t.shape[1], H, -1).transpose(1, 2) for t in (q, k, v))
    o = torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1) @ vh
    return o.transpose(1, 2).reshape(G, n, -1)


def encoder(layers, x, B, h, w):
    """TransformerEngine.run_blocks over the EncoderLayers as they describe themselves (padded q / k rows, ff_first,
    the records) on the channels-last map x [B*h*w, D]."""
    D = x.shape[1]

    def ff(L, x):
        return x + F.gelu(_ln(x, L.ln2) @ L.fc1_w.t() + L.fc1_b) @ L.fc2_w.t() + L.fc2_b

    for L in layers:
        A, H, dk = L.attention, L.heads, L.dim_head
        if L.ff_first:
            x = ff(L, x)
        xn = _ln(x, L.ln1)
        if isinstance(A, StridedKV):
            r = A.stride
            kv = im2col_nhwc(xn, B, h, w, r, r, 0) @ conv_rows(A.kv_w).t()
            Nk = (h // r) * (w // r)
            q = (xn @ L.qkv_w.t()).view(B, h * w, H * dk)
            kv = kv.view(B, Nk, -1)
            o = attend(q, kv[..., :H * dk], kv[..., H * dk:], H, L.scale).reshape(B * h * w, -1)
        else:
            qkv = xn @ L.qkv_w.t()
            v = qkv[:, 2 * H * dk:]
            lim = im2col_nhwc(v, B, h, w, 3, 1, 1) @ conv_rows(A.lim_w).t() + A.lim_b
            wh, ww = A.window((h, w))
            b, wy, wx, u, t = torch.meshgrid(torch.arange(B), torch.arange(h // wh), torch.arange(w // ww),
                                             torch.arange(wh), torch.arange(ww), indexing="ij")
            rows = ((b * h + wy * wh + u) * w + wx * ww + t).reshape(-1, wh * ww)     # map-order windows
            g = qkv[rows.reshape(-1)].view(rows.shape[0], wh * ww, -1)
            oa = attend(g[..., :H * dk], g[..., H * dk:2 * H * dk], g[..., 2 * H * dk:], H, L.scale)
            o = torch.empty_like(lim)
            o[rows.reshape(-1)] = oa.reshape(-1, o.shape[1])
            o = o + lim                                   # the LIM added before the one rounding
        x = x + o @ L.out_w.t() + L.out_b
        if not L.ff_first:
            x = ff(L, x)
    return x


def fused_dataflow(m, img):
    """ScalableViT.forward_fused's dataflow in the dtype of m and img."""
    B = img.shape[0]
    maps = m.stage_maps(img.shape[2], img.shape[3])
    h, w = maps[0]
    a = F.unfold(img, 7, padding=3, stride=4).transpose(1, 2).reshape(B * h * w, -1)   # (c, ky, kx) columns
    x = a @ m.to_patches.weight.reshape(m.to_patches.out_channels, -1).t() + m.to_patches.bias
    for i, ((tr, down), (h, w)) in enumerate(zip(m.layers, maps)):
        layers, norm = tr.encoder_layers()
        x = encoder(layers[:1], x, B, h, w)
        peg = tr.layers[0][2].proj
        xm = x.view(B, h, w, -1).permute(0, 3, 1, 2)
        x = (F.conv2d(xm, peg.weight, peg.bias, padding=1, groups=xm.shape[1]) + xm).permute(0, 2, 3, 1).reshape(
            B * h * w, -1)
        x = encoder(layers[1:], x, B, h, w)
        if down is not None:
            oh, ow = maps[i + 1]
            x = im2col_nhwc(_ln(x, norm), B, h, w, 3, 2, 1) @ conv_rows(down.conv.weight).t() + down.conv.bias
    pooled = x.view(B, h * w, -1).mean(1)
    hl = m.mlp_head[1]
    pooled = F.layer_norm(pooled, pooled.shape[-1:], hl.weight, hl.bias, hl.eps)
    return pooled @ m.mlp_head[2].weight.t() + m.mlp_head[2].bias


@pytest.mark.parametrize("name", sorted(SCALABLE_VIT_CASES))
def test_fused_dataflow_matches_the_reference_in_fp64(name):
    """q / k heads padded to multiples of 16 with zero rows, the LIM added to the attention output before the
    out-projection, windows gathered in map order, the FeedForward before the IWSA: the reference's logits."""
    spec = FAMILY.cases[name]
    m = FAMILY.build(spec).double()
    with torch.no_grad():
        got = fused_dataflow(m, FAMILY.input(spec).double())
    want = load_golden("scalable_vit")["cases"][name]["logits_fp32"]
    torch.testing.assert_close(got.float(), want, rtol=1e-4, atol=1e-4)


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
def test_stage_one_runs_the_readme_attention_shapes(schedule, ln_mode, host_loop):
    """Stage 1: SSA on attention_kv_ex with dk 48 (dim_key 40 padded), dv 32 over 8 x 8 keys; IWSA on attention_iwsa
    over one 64 x 64 window; each run once per layer, the SSA first."""
    calls = schedule[SS.run_name(ln_mode, host_loop)]
    kv = [c for c in calls if c["call"] == "attention_kv_ex"]
    iw = [c for c in calls if c["call"] == "attention_iwsa"]
    assert len(kv) == len(iw) == 3
    assert {k: kv[0][k] for k in ("Nq", "Nk", "H", "dk", "dv")} == dict(Nq=4096, Nk=64, H=2, dk=48, dv=32)
    assert kv[0]["scale"] == pytest.approx(40 ** -0.5)
    assert {k: iw[0][k] for k in ("gh", "gw", "wh", "ww", "H", "dk", "dv")} == dict(gh=64, gw=64, wh=64, ww=64, H=2,
                                                                                    dk=32, dv=32)
    assert calls.index(kv[0]) < calls.index(iw[0])
