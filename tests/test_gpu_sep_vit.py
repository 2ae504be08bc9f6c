"""-m gpu: SepViT on the H100.  b200vit_attention_window_token and b200vit_window_mix against an fp64 reference with
the per-element bounds of oracle/attention_bounds.py (windows 1 to 7 wide, every head width, one and four heads,
non-square window grids), their isolation (NaN and Inf stay in their window, resp. image and head; no read or write
outside the addressed rows) and repeatability; b200vit_head_layernorm_gelu against fp64 with the head-norm bounds of
oracle/row_bounds.py; then the model: every case of tests/golden/sep_vit_spec.py through the comparison of
test_gpu_family_parity.py in both LayerNorm modes, CUDA-graph replay, weight refresh, the direct transformer call at
other window sizes and the eager fall-backs."""
import sys

import pytest
import torch

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR
from oracle.bounds import check
from oracle.grid_attention_bounds import (head_layernorm_gelu_reference, mix_reference, window_rows,
                                          window_token_reference)
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from sep_vit_spec import FAMILY, SEP_VIT_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = dict(device=DEV, dtype=torch.bfloat16)
NAN = float("nan")
PAD = 5          # poisoned rows before and after the addressed ones


def poisoned(t, rows=PAD):
    big = torch.full((t.shape[0] + 2 * rows, t.shape[1]), NAN, device=DEV, dtype=t.dtype)
    big[rows:rows + t.shape[0]] = t
    return big


# ========================================================================================= window-token attention
def run_window_token(qkv, tok, B, gh, gw, p, H, dh, with_tok=True):
    """The kernel between NaN rows of qkv, writing between NaN rows of out and tok_out; asserts the padding kept."""
    M, I, nw = B * gh * gw, H * dh, (gh // p) * (gw // p)
    big, obig = poisoned(qkv), torch.full((M + 2 * PAD, I), NAN, **BF)
    tbig = torch.full((B * nw + 2 * PAD, I), NAN, **BF)
    _lib.attention_window_token(big[PAD:PAD + M], tok, obig[PAD:PAD + M], tbig[PAD:PAD + B * nw] if with_tok else None,
                                B, gh, gw, p, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    assert torch.isnan(obig[:PAD]).all() and torch.isnan(obig[PAD + M:]).all()
    assert torch.isnan(tbig[:PAD]).all() and torch.isnan(tbig[PAD + B * nw:]).all()
    if not with_tok:
        assert torch.isnan(tbig).all()
    return obig[PAD:PAD + M].clone(), tbig[PAD:PAD + B * nw].clone()


WT_SHAPES = [  # B, gh, gw, p
    (2, 7, 7, 7),          # one window
    (1, 56, 56, 7),        # the README's stage 1: 64 windows
    (2, 28, 14, 7),        # non-square window grid
    (3, 8, 12, 4),
    (2, 6, 4, 2),
    (2, 3, 5, 1),          # one token and its window token
]


@pytest.mark.parametrize("H", [1, 4])
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("B,gh,gw,p", WT_SHAPES)
def test_attention_window_token_within_bounds_and_repeatable(B, gh, gw, p, dh, H):
    g = torch.Generator(device=DEV).manual_seed(B * gh * gw + 7 * p + dh + H)
    qkv = (torch.randn(B * gh * gw, 3 * H * dh, device=DEV, generator=g) * 1.5).bfloat16()
    tok = (torch.randn(3 * H * dh, device=DEV, generator=g) * 1.5).bfloat16()
    out, tout = run_window_token(qkv, tok, B, gh, gw, p, H, dh)
    assert torch.isfinite(out).all() and torch.isfinite(tout).all()
    ref, bnd, tref, tbnd = window_token_reference(qkv, tok, B, gh, gw, p, H, dh)
    check(out, ref, bnd, f"window_token {B}x{gh}x{gw} p={p} dh={dh} H={H}")
    check(tout, tref, tbnd, f"window_token {B}x{gh}x{gw} p={p} dh={dh} H={H}: window tokens")
    out2, tout2 = run_window_token(qkv, tok, B, gh, gw, p, H, dh)
    assert torch.equal(out2, out) and torch.equal(tout2, tout)
    out3, _ = run_window_token(qkv, tok, B, gh, gw, p, H, dh, with_tok=False)
    assert torch.equal(out3, out)


@pytest.mark.parametrize("bad", ["nan_q", "inf_v"])
def test_attention_window_token_keeps_nan_and_inf_inside_the_window(bad):
    B, gh, gw, p, H, dh = 2, 14, 21, 7, 2, 32
    g = torch.Generator(device=DEV).manual_seed(5)
    qkv = torch.randn(B * gh * gw, 3 * H * dh, device=DEV, generator=g).bfloat16()
    tok = torch.randn(3 * H * dh, device=DEV, generator=g).bfloat16()
    clean, tclean = run_window_token(qkv, tok, B, gh, gw, p, H, dh)
    rows = window_rows(B, gh, gw, p, p, DEV)
    win = 1 * 6 + 1 * 3 + 2                               # window (b=1, wy=1, wx=2)
    dirty = qkv.clone()
    r = rows[win, 10]
    if bad == "nan_q":
        dirty[r, 3] = NAN                                 # head 0's query
    else:
        dirty[r, 2 * H * dh + dh + 1] = float("inf")      # head 1's value
    out, tout = run_window_token(dirty, tok, B, gh, gw, p, H, dh)
    inside = torch.zeros(B * gh * gw, dtype=torch.bool, device=DEV)
    inside[rows[win]] = True
    same = lambda a, b: (a == b) | (torch.isnan(a) & torch.isnan(b))  # noqa: E731
    assert same(out, clean)[~inside].all()
    keep = torch.ones(tout.shape[0], dtype=torch.bool, device=DEV)
    keep[win] = False
    assert same(tout, tclean)[keep].all()
    assert not torch.isfinite(out[inside]).all()


# ================================================================================================ window mix
def run_mix(wqk, o, B, gh, gw, p, H, dh):
    M, I = B * gh * gw, H * dh
    nw = (gh // p) * (gw // p)
    wbig, obig = poisoned(wqk), poisoned(o)
    out = torch.full((M + 2 * PAD, I), NAN, **BF)
    _lib.window_mix(wbig[PAD:PAD + B * nw], obig[PAD:PAD + M], out[PAD:PAD + M], B, gh, gw, p, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    assert torch.isnan(out[:PAD]).all() and torch.isnan(out[PAD + M:]).all()
    return out[PAD:PAD + M].clone()


MIX_SHAPES = [  # B, gh, gw, p: nw
    (3, 14, 7, 7),         # 2, non-square grid
    (2, 4, 4, 2),          # 4
    (2, 28, 28, 7),        # 16
    (1, 7, 7, 1),          # 49
    (2, 56, 56, 7),        # 64
    (2, 16, 64, 4),        # 64, non-square grid
    (2, 24, 9, 3),         # 24
]


@pytest.mark.parametrize("H", [1, 4])
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("B,gh,gw,p", MIX_SHAPES)
def test_window_mix_within_bounds_and_repeatable(B, gh, gw, p, dh, H):
    g = torch.Generator(device=DEV).manual_seed(B * gh * gw + 11 * p + dh + H)
    nw = (gh // p) * (gw // p)
    wqk = (torch.randn(B * nw, 2 * H * dh, device=DEV, generator=g) * 1.5).bfloat16()
    o = torch.randn(B * gh * gw, H * dh, device=DEV, generator=g).bfloat16()
    out = run_mix(wqk, o, B, gh, gw, p, H, dh)
    assert torch.isfinite(out).all()
    ref, bnd = mix_reference(wqk, o, B, gh, gw, p, H, dh)
    check(out, ref, bnd, f"window_mix {B}x{gh}x{gw} p={p} dh={dh} H={H}")
    assert torch.equal(run_mix(wqk, o, B, gh, gw, p, H, dh), out)


@pytest.mark.parametrize("bad", ["nan_wq", "inf_o"])
def test_window_mix_keeps_nan_and_inf_inside_the_image_and_head(bad):
    B, gh, gw, p, H, dh = 3, 14, 14, 7, 4, 32
    g = torch.Generator(device=DEV).manual_seed(9)
    nw = 4
    wqk = torch.randn(B * nw, 2 * H * dh, device=DEV, generator=g).bfloat16()
    o = torch.randn(B * gh * gw, H * dh, device=DEV, generator=g).bfloat16()
    clean = run_mix(wqk, o, B, gh, gw, p, H, dh)
    b, h = 1, 2
    w2, o2 = wqk.clone(), o.clone()
    if bad == "nan_wq":
        w2[b * nw + 3, 2 * h * dh + 5] = NAN
    else:
        o2[(b * gh + 9) * gw + 3, h * dh + 7] = float("inf")
    out = run_mix(w2, o2, B, gh, gw, p, H, dh)
    inside = torch.zeros_like(out, dtype=torch.bool)
    inside[b * gh * gw:(b + 1) * gh * gw, h * dh:(h + 1) * dh] = True
    same = (out == clean) | (torch.isnan(out) & torch.isnan(clean))
    assert same[~inside].all()
    assert not torch.isfinite(out[inside]).all()


# ================================================================================================ head LayerNorm + GELU
@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("T,H", [(128, 1), (130, 2), (64, 8), (37, 5)])
def test_head_layernorm_gelu_against_fp64(T, H, dh):
    g = torch.Generator(device=DEV).manual_seed(T + H + dh)
    x = (torch.randn(T, H * dh, device=DEV, generator=g) * 2 + 0.5).bfloat16()
    gamma = 1 + 0.3 * torch.randn(dh, device=DEV, generator=g)
    beta = 0.3 * torch.randn(dh, device=DEV, generator=g)
    ld = H * dh + 8
    buf = torch.full((T + 2, ld), NAN, **BF)
    buf[:T, :H * dh] = x
    _lib.head_layernorm_gelu(buf[:T], gamma, beta, H, dh)
    torch.cuda.synchronize()
    assert torch.isnan(buf[T:]).all() and torch.isnan(buf[:T, H * dh:]).all()
    ref, bound = head_layernorm_gelu_reference(x, gamma, beta, H, dh)
    check(buf[:T, :H * dh].view(T, H, dh), ref, bound, f"head_layernorm_gelu {T}x{H}x{dh}")


# ============================================================================================================ model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(SEP_VIT_CASES))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec against the reference's stored logits and the module's own bf16 graph with the shared
    comparison (fused_reason is None, launches counted, tol 3e-2), in both LayerNorm modes."""
    monkeypatch.setitem(P.FAMILIES, "sep_vit", FAMILY)
    monkeypatch.setitem(P.GPU, "sep_vit", dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens("sep_vit", name, ln_mode, monkeypatch)


def small_model(seed=0, name="two_stage_batch3"):
    spec = dict(SEP_VIT_CASES[name], seed=seed)
    return FAMILY.build(spec).to(DEV, torch.bfloat16), FAMILY.input(spec).to(DEV)


def test_graphed_forward_replays_the_eager_launches_bit_for_bit():
    m, x = small_model()
    with torch.inference_mode():
        want = m(x).clone()
    fwd = GraphedForward(m, x)
    got = fwd(x)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_window_token_data_write_and_refresh_change_the_output():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
        tok = m.layers[0][2].layers[0][0].window_tokens
        tok.data.mul_(-1.5)                               # through .data: the version counter does not move
        m.refresh_fused_weights()
        after = m(x).clone()
        want = m.forward_eager(x)
    assert not torch.equal(after, before)
    assert (after.float() - want.float()).abs().max().item() < 3e-2


@pytest.mark.parametrize("p,hw", [(7, (14, 21)), (4, (8, 16)), (2, (6, 4)), (1, (3, 5))])
def test_direct_transformer_call_against_its_pytorch_graph(p, hw):
    """A stage's Transformer called on a channels-first map runs fused; its DSSAs' window_size set to p."""
    m, _ = small_model()
    tr = m.layers[0][2]
    for attn, _ in tr.layers:
        attn.window_size = p
    g = torch.Generator(device=DEV).manual_seed(11 + p)
    fmap = torch.randn(2, tr.layers[0][0].to_qkv.weight.shape[1], *hw, device=DEV, generator=g).bfloat16()
    with torch.inference_mode():
        assert tr.fused_reason(fmap) is None
        _lib.reset_launch_count()
        got = tr(fmap)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = tr.forward_eager(fmap)
    assert got.shape == fmap.shape and got.dtype == torch.bfloat16
    assert (got.float() - want.float()).abs().max().item() < 6e-2


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
        assert seen == [(3 * 16, 3 * 64, 50)]             # 28 x 28 map: 16 windows of 49 tokens + the window token
        assert (got.float() - m.forward_eager(x).float()).abs().max().item() < 5e-2
        h.remove()
        assert m.fused_reason(x) is None
        m.train()
        assert "training" in m.fused_reason(x)
        assert "training" in m.layers[0][2].fused_reason(torch.zeros(2, 64, 28, 28, **BF))
        m.eval()
        assert m.fused_reason(x.float()) is not None
        big = torch.zeros(1, 3, 448, 448, **BF)           # 112 x 112: 256 windows in stage 1
        assert "windows" in m.fused_reason(big)
