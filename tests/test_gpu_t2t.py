"""-m gpu: T2T-ViT on the H100.  The soft-split unfold kernels bit-exact against torch.nn.functional.unfold, the
dh 160 instance of b200vit_attention_varlen against oracle/attention_bounds.py, b200vit_attention_wide against the fp64
reference of oracle/wide_attention_bounds.py, their isolation (poisoned rows around every buffer, NaN / Inf kept inside
an image) and bit-identical repeats; then the model: every case of tests/golden/t2t_spec.py through the comparison of
test_gpu_family_parity.py in both LayerNorm modes, CUDA-graph replay, weight refresh, the direct Transformer call and
the eager fall-backs."""
import sys

import pytest
import torch
import torch.nn.functional as F

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR, load_golden
from oracle.attention_bounds import qkv_attention_reference, qkv_inputs
from oracle.bounds import check
from oracle.wide_attention_bounds import qkv_wide_reference, wide_inputs
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward
from vit_pytorch_b200.pit import pool_grid
from vit_pytorch_b200.t2t import T2TViT

sys.path.insert(0, GOLDEN_DIR)
from t2t_spec import FAMILY, T2T_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = dict(device=DEV, dtype=torch.bfloat16)
NAN = float("nan")
PAD = 5          # poisoned rows before and after the addressed ones
FALLBACK = {"past_wide_cap"}


def seeded(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(**BF)


def unfold_ref(img, k, s, p):
    return F.unfold(img.float(), k, padding=p, stride=s).transpose(1, 2).reshape(-1, img.shape[1] * k * k)


# ---------------------------------------------------------------------------------------------------- unfold
@pytest.mark.parametrize("B,C,H,W,k,s", [(2, 3, 224, 224, 7, 4), (2, 3, 32, 32, 7, 4), (3, 1, 16, 64, 7, 4),
                                         (2, 3, 17, 23, 3, 2), (1, 4, 9, 9, 3, 1), (2, 2, 5, 5, 5, 3)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_unfold_image_bit_exact(B, C, H, W, k, s, dtype):
    img = seeded((B, C, H, W), 11 + H)
    p = s // 2
    ref = unfold_ref(img, k, s, p)
    K = C * k * k
    ldo = (K + 7) // 8 * 8 + 8
    rows = ref.shape[0]
    buf = torch.full((rows + 2 * PAD, ldo), NAN, device=DEV, dtype=dtype)
    out = buf[PAD:PAD + rows]
    _lib.t2t_unfold_image(img, out, k, s, p)
    torch.cuda.synchronize()
    assert torch.equal(out[:, :K].float().cpu(), ref.cpu())
    assert (out[:, K:] == 0).all()
    assert buf[:PAD].isnan().all() and buf[PAD + rows:].isnan().all()


@pytest.mark.parametrize("B,n,C,k,s", [(2, 3136, 147, 3, 2), (2, 64, 147, 3, 2), (3, 64, 27, 3, 2), (2, 20, 5, 3, 2),
                                       (2, 1089, 27, 3, 2), (1, 49, 8, 5, 1)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_unfold_tokens_bit_exact(B, n, C, k, s, dtype):
    """Token rows with a row stride past C (the LayerNorm output's padding poisoned), read as int(sqrt(n)) rows."""
    ld = (C + 7) // 8 * 8 + 8
    xbuf = torch.full((B * n + 2 * PAD, ld), NAN, **BF)
    x = xbuf[PAD:PAD + B * n]
    x[:, :C] = seeded((B * n, C), 7 + n)
    h, w = pool_grid(n)
    p = s // 2
    img = x[:, :C].reshape(B, h, w, C).permute(0, 3, 1, 2)
    ref = unfold_ref(img, k, s, p)
    K = C * k * k
    ldo = (K + 7) // 8 * 8
    rows = ref.shape[0]
    buf = torch.full((rows + 2 * PAD, ldo), NAN, device=DEV, dtype=dtype)
    out = buf[PAD:PAD + rows]
    _lib.t2t_unfold_tokens(x[:, :C], (h, w), out, k, s, p)
    torch.cuda.synchronize()
    assert torch.equal(out[:, :K].float().cpu(), ref.cpu())
    assert (out[:, K:] == 0).all()
    assert buf[:PAD].isnan().all() and buf[PAD + rows:].isnan().all()


def test_unfold_tokens_keeps_nan_inside_its_image():
    B, n, C = 3, 64, 27
    x = seeded((B * n, C), 5)
    x[n + 10, 3] = NAN
    x[n + 20, 4] = float("inf")
    out = torch.empty(B * 16, 248, **BF)
    _lib.t2t_unfold_tokens(x, (8, 8), out, 3, 2, 1)
    torch.cuda.synchronize()
    assert out[:16].isfinite().all() and out[32:].isfinite().all() and not out[16:32].isfinite().all()


# ---------------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("lengths", [[3136, 3136], [64, 64, 64], [1, 65, 200], [784]])
@pytest.mark.parametrize("kind", ["normal", "peaked", "late_max", "vmean"])
def test_varlen_160_against_fp64(lengths, kind):
    """The one head of a soft split up to 160 wide (147 padded with zero columns, as the projection writes it)."""
    qkv = qkv_inputs(kind, lengths, 1, 160, seed=sum(lengths), device=DEV)
    qkv.view(-1, 3, 160)[:, :, 147:] = 0
    cu, tp, tiles = _lib.varlen_index(lengths, DEV)
    out = torch.empty(qkv.shape[0], 160, **BF)
    scale = 147 ** -0.5
    _lib.attention_varlen(qkv, out, cu, tp, tiles, 1, 160, scale)
    torch.cuda.synchronize()
    ref, bound = qkv_attention_reference(qkv, lengths, 1, 160, scale)
    check(out, ref, bound, f"varlen dh 160 {lengths} {kind}")
    assert (out[:, 147:] == 0).all()


@pytest.mark.parametrize("B,n,w,dp", [(2, 784, 1323, 1344), (3, 16, 1323, 1344), (2, 64, 243, 256), (1, 1, 441, 448),
                                      (2, 1024, 300, 320), (5, 130, 441, 448)])
@pytest.mark.parametrize("qk_std", [1.0, 0.3])
def test_wide_against_fp64(B, n, w, dp, qk_std):
    qkv = wide_inputs(B, n, w, dp, seed=n + w, qk_std=qk_std, device=DEV)
    out = torch.empty(B * n, dp, **BF)
    scale = w ** -0.5
    # a workspace of two images: the batch runs in chunks
    ws = torch.empty(_lib.attention_wide_workspace(n, dp, 2), device=DEV, dtype=torch.uint8)
    _lib.attention_wide(qkv, B, n, dp, scale, ws, out=out)
    torch.cuda.synchronize()
    ref, bound = qkv_wide_reference(qkv, B, n, dp, scale)
    check(out, ref, bound, f"wide B={B} n={n} w={w}")
    assert (out[:, w:] == 0).all()


def test_wide_residual_epilogue_adds_the_rounded_output():
    B, n, w, dp = 3, 100, 441, 448
    qkv = wide_inputs(B, n, w, dp, seed=3, device=DEV)
    ws = torch.empty(_lib.attention_wide_workspace(n, dp, B), device=DEV, dtype=torch.uint8)
    out = torch.empty(B * n, dp, **BF)
    _lib.attention_wide(qkv, B, n, dp, 0.05, ws, out=out)
    x = torch.randn(B * n, 448, device=DEV)
    x[:, w:] = NAN                                   # past n_resid: never touched
    x0 = x.clone()
    _lib.attention_wide(qkv, B, n, dp, 0.05, ws, x=x, n_resid=w)
    torch.cuda.synchronize()
    assert torch.equal(x[:, :w], x0[:, :w] + out[:, :w].float())
    assert x[:, w:].isnan().all()


def test_wide_isolation_and_repeats():
    """Poisoned rows around qkv and out, a NaN and an Inf inside image 1: images 0 and 2 bit-identical to a clean run,
    the rows around out untouched; two runs give the same bits."""
    B, n, w, dp = 3, 200, 243, 256
    clean = wide_inputs(B, n, w, dp, seed=9, device=DEV)
    qbuf = torch.full((B * n + 2 * PAD, 3 * dp), NAN, **BF)
    qkv = qbuf[PAD:PAD + B * n]
    qkv.copy_(clean)
    ws = torch.full((_lib.attention_wide_workspace(n, dp, 1),), 255, device=DEV, dtype=torch.uint8)
    obuf = torch.full((B * n + 2 * PAD, dp), NAN, **BF)
    out = obuf[PAD:PAD + B * n]
    _lib.attention_wide(qkv, B, n, dp, w ** -0.5, ws, out=out)
    first = out.clone()
    _lib.attention_wide(qkv, B, n, dp, w ** -0.5, ws, out=out)
    torch.cuda.synchronize()
    assert torch.equal(first, out) and first.isfinite().all()
    assert obuf[:PAD].isnan().all() and obuf[PAD + B * n:].isnan().all()
    qkv[n + 7, 3] = NAN
    qkv[n + 50, dp + 5] = float("inf")
    qkv[n + 60, 2 * dp + 1] = NAN
    _lib.attention_wide(qkv, B, n, dp, w ** -0.5, ws, out=out)
    torch.cuda.synchronize()
    assert torch.equal(out[:n], first[:n]) and torch.equal(out[2 * n:], first[2 * n:])
    assert not out[n:2 * n].isfinite().all()


def test_varlen_160_isolation():
    lengths = [300, 300, 300]
    qkv = qkv_inputs("normal", lengths, 1, 160, seed=4, device=DEV)
    cu, tp, tiles = _lib.varlen_index(lengths, DEV)
    out = torch.empty(900, 160, **BF)
    _lib.attention_varlen(qkv, out, cu, tp, tiles, 1, 160, 0.08)
    first = out.clone()
    qkv[310, 2 * 160 + 3] = NAN
    qkv[350, 160 + 3] = float("inf")
    _lib.attention_varlen(qkv, out, cu, tp, tiles, 1, 160, 0.08)
    torch.cuda.synchronize()
    assert torch.equal(out[:300], first[:300]) and torch.equal(out[600:], first[600:])


# ---------------------------------------------------------------------------------------------------- model
@pytest.mark.parametrize("name", sorted(set(T2T_CASES) - FALLBACK))
@pytest.mark.parametrize("ln_mode", P.BOTH)
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    monkeypatch.setitem(P.FAMILIES, FAMILY.name, FAMILY)
    monkeypatch.setitem(P.GPU, FAMILY.name, dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens(FAMILY.name, name, ln_mode, monkeypatch)


def _model(name):
    spec = T2T_CASES[name]
    return FAMILY.build(spec).to(DEV, torch.bfloat16), FAMILY.input(spec).to(DEV)


@pytest.mark.parametrize("name", sorted(FALLBACK))
def test_fallback_cases_take_the_pytorch_graph(name, monkeypatch):
    """No soft-split kernel runs (the main encoder, called by the PyTorch graph as a module, may run its own)."""
    m, x = _model(name)
    called = []
    for fn in ("t2t_unfold_image", "t2t_unfold_tokens", "attention_wide", "attention_varlen"):
        real = getattr(_lib, fn)
        monkeypatch.setattr(_lib, fn, lambda *a, _f=fn, _r=real, **k: (called.append(_f), _r(*a, **k))[1])
    with torch.inference_mode():
        r = m.fused_reason(x)
        assert r is not None and "1024" in r
        out = m(x)
    assert called == []
    stored = load_golden(FAMILY.name)["cases"][name]["logits_fp32"]
    assert (out.float().cpu() - stored).abs().max().item() < 3e-2


def test_graph_replay_matches_eager_call():
    m, x = _model("k3_small")
    with torch.inference_mode():
        want = m(x)
    g = GraphedForward(m, x)
    got = g(x)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_weight_refresh_after_in_place_update():
    m, x = _model("pool_mean")
    with torch.inference_mode():
        before = m(x)
        with torch.no_grad():
            m.to_patch_embedding[3].layers[0][1].net[1].weight.mul_(1.5)   # the first soft split's fc1
            m.to_patch_embedding[7].layers[0][0].to_qkv.weight.mul_(0.5)   # the second's projection
        after = m(x)
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("B200VIT_DISABLE_FUSED", "1")
        with torch.inference_mode():
            eager = m(x)
    assert not torch.equal(before, after)
    assert (after.float() - eager.float()).abs().max().item() < 3e-2


def test_direct_transformer_call_and_soft_split_modules():
    m, x = _model("pool_mean")
    tokens = seeded((2, 17, 64), 3)
    with torch.inference_mode():
        assert m.transformer.fused_reason(tokens) is None
        got = m.transformer(tokens)
        split = m.to_patch_embedding[3]
        assert split.fused_reason(seeded((2, 64, 147), 4)) is not None     # 147 wide: the PyTorch graph
        s_out = split(seeded((2, 64, 147), 4))
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("B200VIT_DISABLE_FUSED", "1")
        with torch.inference_mode():
            want = m.transformer(tokens)
    assert (got.float() - want.float()).abs().max().item() < 5e-2
    assert s_out.shape == (2, 64, 147)


def test_fallbacks():
    m, x = _model("pool_mean")
    with torch.inference_mode():
        assert m.fused_reason(x.float()).startswith("input dtype")
        h = m.to_patch_embedding[3].register_forward_hook(lambda *a: None)
        assert "hooks" in m.fused_reason(x)
        out = m(x)
        h.remove()
        assert m.fused_reason(x) is None
        fused = m(x)
    assert (out.float() - fused.float()).abs().max().item() < 3e-2
    other = T2TViT(image_size=32, num_classes=7, dim=64, transformer=torch.nn.Identity()).to(**BF).eval()
    with torch.inference_mode():
        assert "transformer=" in other.fused_reason(x)
        assert other(x).shape == (2, 7)
