"""-m gpu: RegionViT on the H100.  b200vit_attention_region_local against an fp64 reference with per-element bounds
(windows 7 x 7, 14 x 14, 7 x 4, 2 x 2 and 1 x 1, one and four heads, several images), with poisoned rows around the
stream it reads and writes, repeatability, and NaN / Inf kept inside their window; then the model: every case of
tests/golden/regionvit_spec.py through the comparison of test_gpu_family_parity.py in both LayerNorm modes,
CUDA-graph replay, weight refresh (a `.data` write with refresh_fused_weights(), an in-place update of the bias
table), the direct R2LTransformer call and the eager fall-backs."""
import sys

import pytest
import torch

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR
from oracle.bounds import check
from oracle.grid_attention_bounds import region_local_reference, region_window_rows
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from regionvit_spec import FAMILY, REGIONVIT_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = dict(device=DEV, dtype=torch.bfloat16)
NAN = float("nan")
PAD = 5          # poisoned rows before and after the addressed ones
DH = 32


# ======================================================================================= region-to-local attention
def run_region_local(qkv, table, B, lh, lw, rh, rw, W, H):
    """The kernel between NaN rows of qkv, writing between NaN rows of out; asserts the padding kept."""
    M = qkv.shape[0]
    big = torch.full((M + 2 * PAD, qkv.shape[1]), NAN, **BF)
    big[PAD:PAD + M] = qkv
    obig = torch.full((M + 2 * PAD, H * DH), NAN, **BF)
    _lib.attention_region_local(big[PAD:PAD + M], obig[PAD:PAD + M], table, B, lh, lw, rh, rw, W, H, DH, DH ** -0.5)
    torch.cuda.synchronize()
    assert torch.isnan(obig[:PAD]).all() and torch.isnan(obig[PAD + M:]).all()
    return obig[PAD:PAD + M].clone()


def make_inputs(B, lh, lw, rh, rw, W, H, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    M = B * (lh * lw + rh * rw)
    qkv = (torch.randn(M, 3 * H * DH, device=DEV, generator=g) * 1.5).bfloat16()
    table = 2.0 * torch.randn(H, (2 * W - 1) ** 2, device=DEV, generator=g)
    return qkv, table


R2L_SHAPES = [  # B, lh, lw, rh, rw, W: the window
    (2, 56, 56, 8, 8, 7),      # 7 x 7, the README's stage 1
    (2, 14, 7, 2, 1, 7),       # 7 x 7
    (2, 28, 28, 2, 2, 14),     # 14 x 14: 197 tokens, four key blocks
    (3, 14, 14, 1, 1, 14),     # 14 x 14, one window per image
    (2, 7, 4, 1, 1, 7),        # 7 x 4, the non-square last stage
    (2, 4, 4, 2, 2, 7),        # 2 x 2 under a W = 7 table
    (2, 3, 5, 3, 5, 7),        # 1 x 1: a local token and its region token
    (2, 21, 30, 3, 2, 15),     # 7 x 15: 106 tokens, two key blocks
]


@pytest.mark.parametrize("H", [1, 4])
@pytest.mark.parametrize("B,lh,lw,rh,rw,W", R2L_SHAPES)
def test_attention_region_local_within_bounds_and_repeatable(B, lh, lw, rh, rw, W, H):
    qkv, table = make_inputs(B, lh, lw, rh, rw, W, H, seed=B * lh * lw + rh * rw + W + H)
    out = run_region_local(qkv, table, B, lh, lw, rh, rw, W, H)
    assert torch.isfinite(out).all()
    ref, bnd = region_local_reference(qkv, table, B, lh, lw, rh, rw, W, H, DH ** -0.5)
    check(out, ref, bnd, f"region_local B={B} {lh}x{lw} / {rh}x{rw} W={W} H={H}")
    assert torch.equal(run_region_local(qkv, table, B, lh, lw, rh, rw, W, H), out)


@pytest.mark.parametrize("bad", ["nan_q_local", "inf_v_region", "nan_k_local"])
def test_attention_region_local_keeps_nan_and_inf_inside_the_window(bad):
    B, lh, lw, rh, rw, W, H = 2, 28, 28, 2, 2, 14, 2
    qkv, table = make_inputs(B, lh, lw, rh, rw, W, H, seed=3)
    clean = run_region_local(qkv, table, B, lh, lw, rh, rw, W, H)
    rows = region_window_rows(B, lh, lw, rh, rw, DEV)
    win = 1 * 4 + 1 * 2 + 0                               # window (b=1, i=1, j=0)
    dirty = qkv.clone()
    I = H * DH
    if bad == "nan_q_local":
        dirty[rows[win, 150], 3] = NAN                    # head 0's query of a local token in the third key block
    elif bad == "inf_v_region":
        dirty[rows[win, 0], 2 * I + DH + 1] = float("inf")   # head 1's value of the region token
    else:
        dirty[rows[win, 70], I + 5] = NAN                 # head 0's key of a local token in the second key block
    out = run_region_local(dirty, table, B, lh, lw, rh, rw, W, H)
    inside = torch.zeros(qkv.shape[0], dtype=torch.bool, device=DEV)
    inside[rows[win]] = True
    same = lambda a, b: (a == b) | (torch.isnan(a) & torch.isnan(b))  # noqa: E731
    assert same(out, clean)[~inside].all()
    assert not torch.isfinite(out[inside]).all()


# ============================================================================================================ model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(REGIONVIT_CASES))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec against the reference's stored logits and the module's own bf16 graph with the shared
    comparison (fused_reason is None, launches counted, tol 3e-2), in both LayerNorm modes."""
    monkeypatch.setitem(P.FAMILIES, "regionvit", FAMILY)
    monkeypatch.setitem(P.GPU, "regionvit", dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens("regionvit", name, ln_mode, monkeypatch)


def small_model(seed=0, name="three_conv_peg_112"):
    spec = dict(REGIONVIT_CASES[name], seed=seed)
    return FAMILY.build(spec).to(DEV, torch.bfloat16), FAMILY.input(spec).to(DEV)


def test_graphed_forward_replays_the_eager_launches_bit_for_bit():
    m, x = small_model()
    with torch.inference_mode():
        want = m(x).clone()
    fwd = GraphedForward(m, x)
    got = fwd(x)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_data_write_and_refresh_change_the_output():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
        w = m.layers[1][2].layers[0][0].to_qkv.weight
        w.data.mul_(-1.5)                                 # through .data: the version counter does not move
        m.refresh_fused_weights()
        after = m(x).clone()
        want = m.forward_eager(x)
    assert not torch.equal(after, before)
    assert (after.float() - want.float()).abs().max().item() < 3e-2


def test_in_place_bias_update_rebuilds_the_table():
    m, x = small_model()
    tr = m.layers[0][2]
    with torch.inference_mode():
        before = m(x).clone()
        t0 = tr.engine().prepared()["0.r2l"].clone()
    with torch.no_grad():
        tr.local_rel_pos_bias.weight.mul_(-3.0)           # in place: the version counter moves
    with torch.inference_mode():
        after = m(x).clone()
        want = m.forward_eager(x)
        t1 = tr.engine().prepared()["0.r2l"]
    assert torch.equal(t1, tr.local_rel_pos_bias.weight.float().t()) and not torch.equal(t1, t0)
    assert not torch.equal(after, before)
    assert (after.float() - want.float()).abs().max().item() < 3e-2


@pytest.mark.parametrize("local_hw,region_hw", [((14, 21), (2, 3)), ((7, 8), (1, 2)), ((4, 4), (2, 2))])
def test_direct_r2l_transformer_call_against_its_pytorch_graph(local_hw, region_hw):
    m, _ = small_model()
    tr = m.layers[1][2]
    c = tr.layers[0][0].to_qkv.weight.shape[1]
    g = torch.Generator(device=DEV).manual_seed(local_hw[0] + region_hw[1])
    local = torch.randn(2, c, *local_hw, device=DEV, generator=g).bfloat16()
    region = torch.randn(2, c, *region_hw, device=DEV, generator=g).bfloat16()
    with torch.inference_mode():
        assert tr.fused_reason(local, region) is None
        _lib.reset_launch_count()
        got = tr(local, region)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = tr.forward_eager(local, region)
    for gt, wt, src in zip(got, want, (local, region)):
        assert gt.shape == src.shape and gt.dtype == torch.bfloat16
        assert (gt.float() - wt.float()).abs().max().item() < 6e-2


def test_eager_fallbacks(monkeypatch):
    m, x = small_model()
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        with monkeypatch.context() as mp:
            mp.setenv("B200VIT_DISABLE_FUSED", "1")
            assert "B200VIT_DISABLE_FUSED" in m.fused_reason(x)
            _lib.reset_launch_count()
            m(x)
            assert _lib.launch_count() == 0
        seen = []
        h = m.layers[0][2].layers[0][0].to_qkv.register_forward_hook(lambda mod, i, o: seen.append(tuple(o.shape)))
        assert "hooks" in m.fused_reason(x)
        got = m(x)
        assert seen == [(3, 16, 384), (3 * 16, 50, 384)]  # the region tokens, then 16 windows of 49 + 1 tokens
        assert (got.float() - m.forward_eager(x).float()).abs().max().item() < 5e-2
        h.remove()
        assert m.fused_reason(x) is None
        m.train()
        assert "training" in m.fused_reason(x)
        m.eval()
        assert m.fused_reason(x.float()) is not None
        assert "does not split" in m.fused_reason(torch.zeros(1, 3, 84, 84, **BF))
        with pytest.raises(RuntimeError):
            m(torch.zeros(1, 3, 84, 84, **BF))            # the graph runs and raises at stage 2
