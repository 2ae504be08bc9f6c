"""-m gpu: CvT on the H100.  b200vit_conv_proj_dw against an fp64 reference with per-element bounds (every kernel size,
strides 1 to 3, odd and one-token maps), what it writes, that repeated calls give the same bits and that each image's
outputs come from its own rows only; then the model: every case of tests/golden/cvt_spec.py through the comparison of
test_gpu_family_parity.py in both LayerNorm modes, CUDA-graph replay, weight refresh and the eager fall-backs."""
import sys

import pytest
import torch

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR
from oracle.bounds import check
from oracle.grid_attention_bounds import conv_reference
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from cvt_spec import CVT_CASES, FAMILY  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")


# ================================================================================================ conv_proj_dw
def make_inputs(B, h, w, C, k, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B * h * w, C, device=DEV, generator=g).bfloat16()
    wq, wkv = (torch.randn(k * k, C, device=DEV, generator=g) / k for _ in range(2))
    bq, bkv = (torch.randn(C, device=DEV, generator=g) for _ in range(2))
    return x, wq, bq, wkv, bkv


def run_conv_proj(x, wq, bq, wkv, bkv, B, h, w, k, s, pad_rows=3):
    """(q, kv) written into the heads of NaN-filled buffers with `pad_rows` rows past them, and those buffers."""
    C = x.shape[1]
    oh, ow = (h - 1) // s + 1, (w - 1) // s + 1
    bq_buf = torch.full((B * h * w + pad_rows, C), NAN, device=DEV, dtype=torch.bfloat16)
    bkv_buf = torch.full((B * oh * ow + pad_rows, C), NAN, device=DEV, dtype=torch.bfloat16)
    q, kv = bq_buf[:B * h * w], bkv_buf[:B * oh * ow]
    _lib.conv_proj_dw(x, wq, bq, wkv, bkv, q, kv, B, h, w, k, s)
    torch.cuda.synchronize()
    return q, kv, bq_buf, bkv_buf


@pytest.mark.parametrize("B,h,w,C,k,s", [(2, 56, 56, 64, 3, 2), (3, 25, 19, 64, 3, 2), (2, 7, 5, 384, 3, 2),
                                         (1, 13, 10, 192, 5, 3), (2, 8, 8, 40, 7, 1), (2, 4, 4, 64, 1, 2),
                                         (2, 1, 1, 64, 3, 2), (2, 9, 14, 96, 7, 3), (1, 3, 2, 8, 5, 4)])
def test_conv_proj_dw_against_fp64_and_repeatable(B, h, w, C, k, s):
    x, wq, bq, wkv, bkv = make_inputs(B, h, w, C, k, seed=B * h * w + C + k * 10 + s)
    q, kv, qbuf, kvbuf = run_conv_proj(x, wq, bq, wkv, bkv, B, h, w, k, s)
    assert torch.isnan(qbuf[B * h * w:]).all() and torch.isnan(kvbuf[kv.shape[0]:]).all()   # nothing past the maps
    ref, bound = conv_reference(x, wq, bq, B, h, w, k, 1)
    check(q, ref, bound, f"q {B}x{h}x{w}x{C} k={k}")
    ref, bound = conv_reference(x, wkv, bkv, B, h, w, k, s)
    assert ref.shape == kv.shape
    check(kv, ref, bound, f"kv {B}x{h}x{w}x{C} k={k} s={s}")
    q2, kv2, _, _ = run_conv_proj(x, wq, bq, wkv, bkv, B, h, w, k, s)
    assert torch.equal(q2, q) and torch.equal(kv2, kv)


@pytest.mark.parametrize("k,s", [(3, 2), (7, 3)])
def test_conv_proj_dw_keeps_each_image_to_itself(k, s):
    """A NaN in every row of one image leaves every other image's outputs bit-identical; rows past the input are
    never read (the input is the head of a NaN-poisoned buffer)."""
    B, h, w, C = 3, 11, 9, 64
    x, wq, bq, wkv, bkv = make_inputs(B, h, w, C, k, seed=31 + k)
    M = B * h * w
    big = torch.full((M + 5, C), NAN, device=DEV, dtype=torch.bfloat16)
    big[:M] = x
    q, kv, _, _ = run_conv_proj(big[:M], wq, bq, wkv, bkv, B, h, w, k, s)
    assert not torch.isnan(q).any() and not torch.isnan(kv).any()
    bad = big[:M].clone()
    bad[h * w:2 * h * w] = NAN                                       # image 1
    q2, kv2, _, _ = run_conv_proj(bad, wq, bq, wkv, bkv, B, h, w, k, s)
    nq, nkv = h * w, kv.shape[0] // B
    for b in (0, 2):
        assert torch.equal(q2[b * nq:(b + 1) * nq], q[b * nq:(b + 1) * nq])
        assert torch.equal(kv2[b * nkv:(b + 1) * nkv], kv[b * nkv:(b + 1) * nkv])
    assert torch.isnan(q2[nq:2 * nq]).all() and torch.isnan(kv2[nkv:2 * nkv]).all()


# ============================================================================================================ model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(CVT_CASES))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec against the reference's stored logits and the module's own bf16 graph with the shared
    comparison (fused_reason is None, launches counted, tol 3e-2), in both LayerNorm modes."""
    monkeypatch.setitem(P.FAMILIES, "cvt", FAMILY)
    monkeypatch.setitem(P.GPU, "cvt", dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens("cvt", name, ln_mode, monkeypatch)


def small_model(seed=0, name="odd_nonsquare_c1"):
    spec = dict(CVT_CASES[name], seed=seed)
    return FAMILY.build(spec).to(DEV, torch.bfloat16), FAMILY.input(spec).to(DEV)


def test_cuda_graph_replay_matches_eager_launches():
    m, x = small_model()
    with torch.inference_mode():
        want = m(x).clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                m(x)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m(x)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, want)


def test_graphed_forward():
    m, x = small_model()
    with torch.inference_mode():
        want = m(x).clone()
    fwd = GraphedForward(m, x)
    got = fwd(x)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_weight_refresh_tracks_the_eager_graph():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
    # load_state_dict: another seed's weights
    other, _ = small_model(seed=9)
    m.load_state_dict(other.state_dict())
    with torch.inference_mode():
        got, want = m(x), m.forward_eager(x)
    assert not torch.equal(want, before)
    assert (got.float() - want.float()).abs().max().item() < 5e-2
    # an in-place update of a projection BatchNorm's running variance: picked up by the version counter
    bn = m.layers[1][2].layers[0][0].to_kv.net[1]
    with torch.no_grad():
        bn.running_var.mul_(3.0)
    with torch.inference_mode():
        got2, want2 = m(x), m.forward_eager(x)
    assert not torch.equal(want2, want)
    assert (got2.float() - want2.float()).abs().max().item() < 5e-2


def test_eager_fallbacks(monkeypatch):
    m, x = small_model()
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        with monkeypatch.context() as mp:
            mp.setenv("B200VIT_DISABLE_FUSED", "1")
            assert "B200VIT_DISABLE_FUSED" in m.fused_reason(x)
            _lib.reset_launch_count()
            want = m(x).clone()
            assert _lib.launch_count() == 0
        seen = []
        h = m.layers[0][2].layers[0][0].to_kv.register_forward_hook(lambda mod, i, o: seen.append(tuple(o.shape)))
        assert "hooks" in m.fused_reason(x)
        _lib.reset_launch_count()
        got = m(x)
        assert _lib.launch_count() == 0 and seen == [(2, 256, 13, 10)] and torch.equal(got, want)
        h.remove()
        assert m.fused_reason(x) is None
    m.train()
    with torch.inference_mode():
        assert "BatchNorm2d is in training mode" in m.fused_reason(x)
    m.eval()
    with torch.inference_mode():
        bad = x[:, :, :, :1].contiguous().repeat(1, 2, 1, 1)       # two channels into a one-channel model
        assert "not (B, 1, H, W)" in m.fused_reason(bad)
