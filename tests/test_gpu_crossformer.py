"""-m gpu: CrossFormer on the H100.  b200vit_cross_embed_nchw against an fp64 reference with per-element GEMM bounds
(the README stem, k = 32, one channel, odd image sizes, several CTAs per image), its determinism, per-image isolation
and what it writes; the later stages' per-scale GEMMs into column slices of the stream; then the model: every case of
tests/golden/crossformer_spec.py through the comparison of test_gpu_family_parity.py (the second expectation is the
module's own fp32 graph: its bf16 graph raises, as the reference's does), CUDA-graph replay, weight refresh, an
in-place update of the dynamic position bias and the eager fall-backs."""
import sys

import pytest
import torch
import torch.nn.functional as F

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR
from oracle.bounds import C_ACC, U, check
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from crossformer_spec import CROSSFORMER_CASES, FAMILY  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")


# ====================================================================================== cross-scale embedding kernel
def embed_inputs(B, C, H, W, ks, widths, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    img = torch.randn(B, C, H, W, device=DEV, generator=g).bfloat16()
    ws = [(torch.randn(n, C, k, k, device=DEV, generator=g) * (C * k * k) ** -0.5).bfloat16()
          for k, n in zip(ks, widths)]
    bias = torch.randn(sum(widths), device=DEV, generator=g)
    return img, ws, bias


def embed_reference(img, ws, bias, s):
    """fp64 (ref, bound): the concatenated convolutions channels-last, and per element the fp32 accumulation bound
    (C_ACC * K + 2) u sum |w x| plus the bias add's rounding."""
    outs, mags, off = [], [], 0
    for w in ws:
        n, k = w.shape[0], w.shape[2]
        b = bias[off:off + n].double()
        outs.append(F.conv2d(img.double(), w.double(), b, stride=s, padding=(k - s) // 2))
        K = w[0].numel()
        mag = F.conv2d(img.double().abs(), w.double().abs(), None, stride=s, padding=(k - s) // 2)
        mags.append((C_ACC * K + 2) * U * mag)
        off += n
    ref = torch.cat(outs, 1)
    e = torch.cat(mags, 1) + 2 * U * ref.abs() + 1e-30
    to_rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])     # noqa: E731
    return to_rows(ref), to_rows(e)


def run_embed(img, ws, bias, s, ldo_pad=8, pad_rows=3):
    """out as the head [M, dim] of a NaN buffer [M + pad_rows, dim + ldo_pad]; returns (buffer, out)."""
    B, _, H, W = img.shape
    ks, widths = [w.shape[2] for w in ws], [w.shape[0] for w in ws]
    p = (ks[0] - s) // 2
    M = B * _lib.conv_out_size(H, ks[0], s, p) * _lib.conv_out_size(W, ks[0], s, p)
    D = sum(widths)
    big = torch.full((M + pad_rows, D + ldo_pad), NAN, device=DEV)
    out = big[:M, :D]
    _lib.cross_embed_nchw(img, _lib.cross_embed_pack(ws), bias, out, ks, widths, s)
    torch.cuda.synchronize()
    return big, out


EMBED_CASES = {
    # the README stem: 56 x 56 tokens per image, 28 CTAs each
    "readme_stem": dict(B=2, C=3, H=224, W=224, ks=(4, 8, 16, 32), widths=(32, 16, 8, 8), s=4),
    # k = 32 at stride 8, one channel, odd image sizes, widths up to 64
    "k32_c1_odd": dict(B=3, C=1, H=203, W=117, ks=(8, 16, 32), widths=(64, 8, 24), s=8),
    # three scales at stride 2 on an odd, non-square image (K = 4 * 3: one partial k-step)
    "three_scale_odd": dict(B=2, C=3, H=37, W=53, ks=(2, 4, 8), widths=(32, 16, 16), s=2),
    # one scale, four channels, stride 1
    "single_c4_s1": dict(B=2, C=4, H=19, W=40, ks=(3,), widths=(40,), s=1),
    # C = 1, k = 2: K = 4, zero-padded to one 16-wide k-step
    "c1_k2": dict(B=2, C=1, H=30, W=18, ks=(2, 4), widths=(8, 16), s=2),
}


@pytest.mark.parametrize("name", sorted(EMBED_CASES))
def test_cross_embed_within_bounds_and_repeatable(name):
    c = EMBED_CASES[name]
    img, ws, bias = embed_inputs(c["B"], c["C"], c["H"], c["W"], c["ks"], c["widths"], seed=len(name))
    big, out = run_embed(img, ws, bias, c["s"])
    M, D = out.shape
    assert torch.isnan(big[M:]).all() and torch.isnan(big[:M, D:]).all()     # nothing outside [M, dim) is written
    assert not torch.isnan(out).any()
    ref, bound = embed_reference(img, ws, bias, c["s"])
    check(out, ref, bound, f"cross_embed {name}")
    _, again = run_embed(img, ws, bias, c["s"])
    assert torch.equal(again, out)


def test_cross_embed_keeps_a_nan_in_its_image():
    c = EMBED_CASES["three_scale_odd"]
    img, ws, bias = embed_inputs(c["B"], c["C"], c["H"], c["W"], c["ks"], c["widths"], seed=3)
    _, clean = run_embed(img, ws, bias, c["s"])
    img2 = img.clone()
    img2[1, 2, 20, 30] = NAN
    _, out = run_embed(img2, ws, bias, c["s"])
    per = clean.shape[0] // c["B"]
    assert torch.equal(out[:per], clean[:per])
    assert torch.isnan(out[per:]).any()
    # only the tokens whose windows cover the pixel change
    changed = ~((out == clean) | (torch.isnan(out) & torch.isnan(clean))).all(1)
    assert 0 < changed.sum().item() < per


def test_cross_embed_rejects_what_it_is_not_built_for():
    img, ws, bias = embed_inputs(1, 3, 32, 32, (4, 3), (16, 16), seed=1)
    out = torch.empty(16 * 16, 32, device=DEV)
    with pytest.raises(_lib.B200VitError, match="maps to"):            # k - s odd for one scale: another map size
        _lib.cross_embed_nchw(img, _lib.cross_embed_pack(ws), bias, out, [4, 3], [16, 16], 2)
    img, ws, bias = embed_inputs(1, 3, 32, 32, (4, 8), (12, 20), seed=1)
    with pytest.raises(_lib.B200VitError, match="width"):
        _lib.cross_embed_nchw(img, _lib.cross_embed_pack(ws), bias, out, [4, 8], [12, 20], 2)


@pytest.mark.parametrize("k,s,C,widths", [(2, 2, 64, (64, 64)), (4, 2, 64, (64, 64)), (4, 2, 80, (40, 40))])
def test_later_stage_gemms_write_only_their_column_slices(k, s, C, widths):
    """conv_im2col_nhwc + the bias GEMM per scale into out_f32 = stream[:, off:off + n] with ldo > dim: every other
    column and the rows past the map stay untouched, and each slice is within the GEMM bound."""
    B, H, W = 2, 14, 10
    g = torch.Generator(device=DEV).manual_seed(k * 100 + C)
    x = torch.randn(B * H * W, C, device=DEV, generator=g).bfloat16()
    p = (k - s) // 2
    oh, ow = _lib.conv_out_size(H, k, s, p), _lib.conv_out_size(W, k, s, p)
    M, D = B * oh * ow, sum(widths)
    big = torch.full((M + 2, D + 16), NAN, device=DEV)
    a = torch.empty(M, k * k * C, device=DEV, dtype=torch.bfloat16)
    _lib.conv_im2col_nhwc(x, a, B, H, W, k, s, p)
    off = 0
    for n in widths:
        w = (torch.randn(n, k * k * C, device=DEV, generator=g) * (k * k * C) ** -0.5).bfloat16()
        b = torch.randn(n, device=DEV, generator=g)
        before = big.clone()
        _lib.gemm(a, w, out_f32=big[:M, off:off + n], bias=b)
        torch.cuda.synchronize()
        outside = torch.ones_like(big, dtype=torch.bool)
        outside[:M, off:off + n] = False
        assert torch.equal(big[outside].isnan(), before[outside].isnan())
        ref = a.double() @ w.double().t() + b.double()
        e = (C_ACC * k * k * C + 2) * U * (a.double().abs() @ w.double().abs().t()) + 2 * U * ref.abs() + 1e-30
        check(big[:M, off:off + n], ref, e, f"stage GEMM k={k} C={C} slice {off}")
        off += n
    assert torch.isnan(big[M:]).all() and torch.isnan(big[:, D:]).all()


# ============================================================================================================ model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(CROSSFORMER_CASES))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec against the reference's stored logits and the module's own fp32 graph with the shared
    comparison (fused_reason is None, launches counted, tol 3e-2), in both LayerNorm modes."""
    monkeypatch.setitem(P.FAMILIES, "crossformer", FAMILY)
    monkeypatch.setitem(P.GPU, "crossformer", dict(tol=3e-2, ln_modes=P.BOTH, second="own fp32"))
    P.test_fused_against_reference_goldens("crossformer", name, ln_mode, monkeypatch)


SPEC = dict(CROSSFORMER_CASES["small_64"], seed=0)


def small_model():
    return FAMILY.build(SPEC).to(DEV, torch.bfloat16), FAMILY.input(SPEC).to(DEV)


def own_fp32(m, x):
    """The module's own PyTorch graph in fp32 on the CPU, on m's current weights."""
    ref = FAMILY.build(SPEC)
    ref.load_state_dict({k: v.float().cpu() for k, v in m.state_dict().items()})
    with torch.no_grad():
        return ref.forward_eager(x.float().cpu())


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
    fwd = GraphedForward(m, x)
    got = fwd(x)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_weight_refresh_and_dpb_update_change_the_next_output():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
        m.to_logits[1].bias.data.add_(1.0)                  # through .data: the version counter does not move
        m.refresh_fused_weights()
        after = m(x).clone()
    assert torch.allclose(after.float(), before.float() + 1.0, atol=5e-2)
    # the stage-1 cross-scale embedding's weights through .data, then refresh
    with torch.inference_mode():
        m.layers[0][0].convs[3].weight.data.mul_(-1.0)
        m.refresh_fused_weights()
        got = m(x).clone()
    want = own_fp32(m, x)
    assert (got.float().cpu() - want).abs().max().item() < 5e-2
    # an in-place update of a dynamic position bias MLP: its version moves, the table is rebuilt
    dpb = m.layers[1][1].layers[0][2].dpb                   # stage 2's long-distance attention
    with torch.no_grad():
        dpb[0].weight.mul_(3.0)
        dpb[9].weight.mul_(4.0)
    with torch.inference_mode():
        got2 = m(x).clone()
    want2 = own_fp32(m, x)
    assert not torch.equal(got2, got)
    assert (got2.float().cpu() - want2).abs().max().item() < 5e-2


def test_eager_fallbacks(monkeypatch):
    m, x = small_model()
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        with monkeypatch.context() as mp:
            mp.setenv("B200VIT_DISABLE_FUSED", "1")
            assert "B200VIT_DISABLE_FUSED" in m.fused_reason(x)
        # a bf16 eager graph raises, as the reference's does
        with monkeypatch.context() as mp:
            mp.setenv("B200VIT_DISABLE_FUSED", "1")
            with pytest.raises(RuntimeError, match="same dtype"):
                m(x)
        seen = []
        h = m.layers[0][1].layers[0][0].to_qkv.register_forward_hook(lambda mod, i, o: seen.append(o.shape))
        assert "hooks" in m.fused_reason(x)
        h.remove()
        assert m.fused_reason(x) is None
        assert "dtype" in m.fused_reason(x.float())
        assert "not (B, 3, H, W)" in m.fused_reason(x[:, :2])
        # a 48 x 48 image: stage 2's 6 x 6 map is not divisible into 4 x 4 global windows
        assert "not divisible" in m.fused_reason(x[:, :, :48, :48])
        m.train()
        assert m.fused_reason(x) is None                    # no dropout
    with torch.enable_grad():
        assert "autograd" in m.fused_reason(x)
