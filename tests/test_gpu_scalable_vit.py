"""-m gpu: ScalableViT on the H100.  b200vit_attention_iwsa and b200vit_attention_kv_ex against an fp64 reference with
the per-element bounds of oracle/attention_bounds.py, extended here for the LIM operand that attention_iwsa adds before
its one rounding: windows of 1 to 4096 tokens, non-square whole-map windows, every built (dk, dv) pair, key counts
around the 64-key block and both the resident and the ring path of the key / value kernel.  Then their isolation
(poisoned rows around every buffer, NaN / Inf kept inside a window, resp. an image), bit-identical repeats, and the
model: every case of tests/golden/scalable_vit_spec.py through the comparison of test_gpu_family_parity.py in both
LayerNorm modes, CUDA-graph replay, weight refresh, the direct Transformer call and the eager fall-backs."""
import math
import sys

import pytest
import torch

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR, load_golden
from oracle.bounds import check
from oracle.grid_attention_bounds import iwsa_reference, kv_ex_reference, window_rows
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from scalable_vit_spec import FAMILY, SCALABLE_VIT_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = dict(device=DEV, dtype=torch.bfloat16)
NAN = float("nan")
PAD = 5          # poisoned rows before and after the addressed ones
PAIRS = [(dk, dv) for dk in (16, 32, 48, 64) for dv in (32, 64)]
FALLBACK = {"fallback_value48"}


def seeded(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(**BF)


def iwsa_inputs(B, gh, gw, H, dk, dv, seed):
    M = B * gh * gw
    qkv = seeded((M, H * (2 * dk + dv)), seed)
    lim = seeded((M, H * dv), seed + 1, 0.5)
    return qkv, lim


# (B, gh, gw, wh, ww, H, dk, dv): windows of 1, 49, 64, 256, 1024 and 4096 tokens, non-square whole maps
IWSA_SHAPES = [
    (2, 4, 6, 1, 1, 2, 32, 32),
    (2, 14, 14, 7, 7, 2, 32, 32),
    (1, 16, 16, 8, 8, 2, 48, 32),
    (2, 32, 32, 16, 16, 1, 32, 64),
    (1, 32, 32, 32, 32, 2, 32, 32),
    (1, 64, 64, 64, 64, 2, 32, 32),
    (2, 24, 40, 24, 40, 1, 64, 64),
    (1, 9, 13, 9, 13, 3, 16, 32),
]


@pytest.mark.parametrize("B,gh,gw,wh,ww,H,dk,dv", IWSA_SHAPES)
def test_iwsa_against_fp64(B, gh, gw, wh, ww, H, dk, dv):
    qkv, lim = iwsa_inputs(B, gh, gw, H, dk, dv, seed=gh * 31 + ww)
    out = torch.empty(B * gh * gw, H * dv, **BF)
    scale = dk ** -0.5
    _lib.attention_iwsa(qkv, lim, out, B, gh, gw, wh, ww, H, dk, dv, scale)
    ref, bound = iwsa_reference(qkv, lim, B, gh, gw, wh, ww, H, dk, dv, scale)
    print(f"iwsa {B}x{gh}x{gw} win {wh}x{ww} H{H} dk{dk} dv{dv}: worst |got - ref| / bound "
          f"{check(out, ref, bound, 'attention_iwsa'):.3f}")


@pytest.mark.parametrize("dk,dv", PAIRS)
def test_iwsa_every_width_pair(dk, dv):
    B, gh, gw, wh, ww, H = 2, 16, 12, 8, 6, 2
    qkv, lim = iwsa_inputs(B, gh, gw, H, dk, dv, seed=dk + dv)
    out = torch.empty(B * gh * gw, H * dv, **BF)
    _lib.attention_iwsa(qkv, lim, out, B, gh, gw, wh, ww, H, dk, dv, 0.2)
    ref, bound = iwsa_reference(qkv, lim, B, gh, gw, wh, ww, H, dk, dv, 0.2)
    check(out, ref, bound, f"attention_iwsa dk{dk} dv{dv}")


# (B, Nq, Nk, H): key counts 1, 63, 64, 65, and 2000 keys (more than any resident set: the ring path)
KV_SHAPES = [(2, 100, 1, 2), (2, 130, 63, 2), (1, 200, 64, 3), (2, 70, 65, 2), (1, 129, 2000, 1)]


@pytest.mark.parametrize("B,Nq,Nk,H", KV_SHAPES)
@pytest.mark.parametrize("dk,dv", [(48, 32), (16, 64), (64, 32)])
def test_kv_ex_against_fp64(B, Nq, Nk, H, dk, dv):
    q = seeded((B * Nq, H * dk), Nq + dk)
    kv = seeded((B * Nk, H * (dk + dv)), Nk + dv)
    out = torch.empty(B * Nq, H * dv, **BF)
    scale = 40 ** -0.5
    _lib.attention_kv_ex(q, kv, out, B, Nq, Nk, H, dk, dv, scale)
    ref, bound = kv_ex_reference(q, kv, B, Nq, Nk, H, dk, dv, scale)
    check(out, ref, bound, f"attention_kv_ex B{B} Nq{Nq} Nk{Nk} dk{dk} dv{dv}")


@pytest.mark.parametrize("dk,dv", PAIRS)
def test_kv_ex_every_width_pair(dk, dv):
    B, Nq, Nk, H = 2, 96, 80, 2
    q = seeded((B * Nq, H * dk), dk)
    kv = seeded((B * Nk, H * (dk + dv)), dv)
    out = torch.empty(B * Nq, H * dv, **BF)
    _lib.attention_kv_ex(q, kv, out, B, Nq, Nk, H, dk, dv, 0.15)
    ref, bound = kv_ex_reference(q, kv, B, Nq, Nk, H, dk, dv, 0.15)
    check(out, ref, bound, f"attention_kv_ex dk{dk} dv{dv}")


def test_kv_ex_with_equal_widths_is_attention_kv_bit_for_bit():
    B, Nq, Nk, H, d = 2, 300, 49, 2, 64
    q, kv = seeded((B * Nq, H * d), 1), seeded((B * Nk, 2 * H * d), 2)
    a, b = torch.empty(B * Nq, H * d, **BF), torch.empty(B * Nq, H * d, **BF)
    _lib.attention_kv(q, kv, a, B, Nq, Nk, H, d, 0.125)
    _lib.attention_kv_ex(q, kv, b, B, Nq, Nk, H, d, d, 0.125)
    assert torch.equal(a, b)


# ============================================================================================================ isolation
def poisoned(t, rows=PAD):
    big = torch.full((t.shape[0] + 2 * rows, t.shape[1]), NAN, device=DEV, dtype=t.dtype)
    big[rows:rows + t.shape[0]] = t
    return big


def test_iwsa_reads_and_writes_only_its_rows_and_repeats_bit_for_bit():
    B, gh, gw, wh, ww, H, dk, dv = 2, 16, 16, 8, 8, 2, 48, 32
    qkv, lim = iwsa_inputs(B, gh, gw, H, dk, dv, 7)
    M = qkv.shape[0]
    want = torch.empty(M, H * dv, **BF)
    _lib.attention_iwsa(qkv, lim, want, B, gh, gw, wh, ww, H, dk, dv, 0.2)
    # NaN rows around qkv and lim, sentinel rows around out
    pq, pl = poisoned(qkv), poisoned(lim)
    po = torch.full((M + 2 * PAD, H * dv), 7.0, **BF)
    _lib.attention_iwsa(pq[PAD:PAD + M], pl[PAD:PAD + M], po[PAD:PAD + M], B, gh, gw, wh, ww, H, dk, dv, 0.2)
    assert torch.equal(po[PAD:PAD + M], want)
    assert (po[:PAD] == 7).all() and (po[PAD + M:] == 7).all()
    again = torch.empty_like(want)
    _lib.attention_iwsa(qkv, lim, again, B, gh, gw, wh, ww, H, dk, dv, 0.2)
    assert torch.equal(again, want)


@pytest.mark.parametrize("bad", [NAN, float("inf")])
@pytest.mark.parametrize("win", [8, 16])
def test_iwsa_keeps_nan_and_inf_in_their_window(bad, win):
    B, gh, gw, H, dk, dv = 2, 16, 16, 2, 32, 32
    qkv, lim = iwsa_inputs(B, gh, gw, H, dk, dv, 11)
    M = qkv.shape[0]
    want = torch.empty(M, H * dv, **BF)
    _lib.attention_iwsa(qkv, lim, want, B, gh, gw, win, win, H, dk, dv, 0.2)
    rows = window_rows(B, gh, gw, win, win, DEV)
    hit = rows[1, 3].item()                   # a key / value row of the second window
    qkv2 = qkv.clone()
    qkv2[hit, H * dk:] = bad
    got = torch.empty_like(want)
    _lib.attention_iwsa(qkv2, lim, got, B, gh, gw, win, win, H, dk, dv, 0.2)
    inside = torch.zeros(M, dtype=torch.bool, device=DEV)
    inside[rows[1]] = True
    assert torch.equal(got[~inside], want[~inside])


@pytest.mark.parametrize("bad", [NAN, float("inf")])
def test_kv_ex_keeps_nan_and_inf_in_their_image(bad):
    B, Nq, Nk, H, dk, dv = 3, 150, 70, 2, 48, 32
    q, kv = seeded((B * Nq, H * dk), 3), seeded((B * Nk, H * (dk + dv)), 4)
    want = torch.empty(B * Nq, H * dv, **BF)
    _lib.attention_kv_ex(q, kv, want, B, Nq, Nk, H, dk, dv, 0.2)
    kv2 = kv.clone()
    kv2[Nk + 5] = bad                         # image 1
    got = torch.empty_like(want)
    _lib.attention_kv_ex(q, kv2, got, B, Nq, Nk, H, dk, dv, 0.2)
    assert torch.equal(got[:Nq], want[:Nq]) and torch.equal(got[2 * Nq:], want[2 * Nq:])
    # poisoned rows around q and kv, sentinels around out
    pq, pkv = poisoned(q), poisoned(kv)
    po = torch.full((B * Nq + 2 * PAD, H * dv), 7.0, **BF)
    _lib.attention_kv_ex(pq[PAD:PAD + B * Nq], pkv[PAD:PAD + B * Nk], po[PAD:PAD + B * Nq], B, Nq, Nk, H, dk, dv, 0.2)
    assert torch.equal(po[PAD:PAD + B * Nq], want)
    assert (po[:PAD] == 7).all() and (po[PAD + B * Nq:] == 7).all()


@pytest.mark.parametrize("Nk", [64, 2000])
def test_kv_ex_repeats_bit_for_bit(Nk):
    """The resident (64 keys) and the ring (2000 keys) path give the same bits on every call."""
    B, Nq, H, dk, dv = 2, 300, 2, 48, 32
    q, kv = seeded((B * Nq, H * dk), 5), seeded((B * Nk, H * (dk + dv)), 6)
    a, b = torch.empty(B * Nq, H * dv, **BF), torch.empty(B * Nq, H * dv, **BF)
    _lib.attention_kv_ex(q, kv, a, B, Nq, Nk, H, dk, dv, 0.2)
    _lib.attention_kv_ex(q, kv, b, B, Nq, Nk, H, dk, dv, 0.2)
    assert torch.equal(a, b)


# ============================================================================================================ model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(set(SCALABLE_VIT_CASES) - FALLBACK))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec that runs fused against the reference's stored logits and the module's own bf16 graph
    with the shared comparison (fused_reason is None, launches counted, tol 3e-2), in both LayerNorm modes."""
    monkeypatch.setitem(P.FAMILIES, "scalable_vit", FAMILY)
    monkeypatch.setitem(P.GPU, "scalable_vit", dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens("scalable_vit", name, ln_mode, monkeypatch)


def test_fallback_case_runs_the_pytorch_graph():
    name = "fallback_value48"
    spec = SCALABLE_VIT_CASES[name]
    m = FAMILY.build(spec).to(DEV, torch.bfloat16)
    x = FAMILY.input(spec).to(DEV)
    with torch.inference_mode():
        assert "dim_value=48" in m.fused_reason(x)
        _lib.reset_launch_count()
        out = m(x)
    torch.cuda.synchronize()
    assert _lib.launch_count() == 0
    stored = load_golden("scalable_vit")["cases"][name]["logits_fp32"]
    assert (out.float().cpu() - stored).abs().max().item() < 3e-2


def small_model(seed=0, name="batch3"):
    spec = dict(SCALABLE_VIT_CASES[name], seed=seed)
    return FAMILY.build(spec).to(DEV, torch.bfloat16), FAMILY.input(spec).to(DEV)


def test_graphed_forward_replays_the_eager_launches_bit_for_bit():
    m, x = small_model()
    with torch.inference_mode():
        want = m(x).clone()
    fwd = GraphedForward(m, x)
    got = fwd(x)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_weight_refresh_after_in_place_update():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
        iwsa = m.layers[0][0].layers[0][4]
        iwsa.local_interactive_module.bias.add_(0.5)
        after = m(x)
        with pytest.MonkeyPatch.context() as mp:
            mp.setenv("B200VIT_DISABLE_FUSED", "1")
            eager = m(x)
    assert not torch.equal(before, after)
    assert (after.float() - eager.float()).abs().max().item() < 3e-2


def test_other_fallbacks():
    m, x = small_model()
    with torch.inference_mode():
        assert m.fused_reason(x.float()) is not None
        assert "CUDA" in m.fused_reason(x.cpu())
        h = m.layers[0][0].layers[0][0].register_forward_hook(lambda *a: None)
        assert "hooks" in m.fused_reason(x)
        h.remove()
        assert m.fused_reason(x) is None
    m.train()
    assert m.fused_reason(x) is not None       # autograd is recording: the parameters require grad
    spec = dict(SCALABLE_VIT_CASES["batch3"], seed=0, dropout=0.1)
    md = FAMILY.build(spec).to(DEV, torch.bfloat16).train()
    with torch.inference_mode():
        assert md.fused_reason(x) == "dropout is active"
        md.eval()
        assert md.fused_reason(x) is None


@pytest.mark.parametrize("window,hw", [(None, (16, 12)), (8, (16, 16)), (4, (8, 12))])
def test_direct_transformer_call_against_its_pytorch_graph(window, hw):
    """A stage's Transformer called on a channels-first map runs fused, its windows set to `window`."""
    m, _ = small_model()
    for tr in (m.layers[0][0], m.layers[1][0]):       # with its ChanLayerNorm, and the last stage's without one
        for layer in tr.layers:
            layer[4].window_size = window
        g = torch.Generator(device=DEV).manual_seed(17)
        fmap = torch.randn(2, tr.layers[0][0].to_q.in_channels, *hw, device=DEV, generator=g).bfloat16()
        with torch.inference_mode():
            assert tr.fused_reason(fmap) is None
            _lib.reset_launch_count()
            got = tr(fmap)
            torch.cuda.synchronize()
            assert _lib.launch_count() > 0
            want = tr.forward_eager(fmap)
        assert got.shape == fmap.shape and got.dtype == torch.bfloat16
        # the last stage's stream is not normalised (values up to about 6 here, where one bf16 step is 1/32), and the
        # eager graph rounds to bf16 after every op: at most 4 bf16 steps of the largest value apart
        d, top = (got.float() - want.float()).abs().max().item(), want.float().abs().max().item()
        print(f"direct {window} {hw}: max |fused - eager| {d:.4f}, max |eager| {top:.2f}")
        assert d <= 4 * 2.0 ** (math.floor(math.log2(max(top, 1.0))) - 7)
