"""-m gpu: LeViT on the H100.  b200vit_attention_posbias against its fp64 reference with per-element bounds
(oracle/grid_attention_bounds.py: bias and GELU included), what it writes and which rows it reads; the Hardswish GEMM
epilogue against fp64 (oracle/bounds.py gemm_reference); then the model:
every case of tests/golden/levit_spec.py through the comparison of test_gpu_family_parity.py, the distill-head case,
CUDA-graph replay, weight refresh and the eager fall-backs."""
import sys

import pytest
import torch

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR, load_golden
from oracle.bounds import bf16_ulp, check, gemm_reference
from oracle.grid_attention_bounds import posbias_reference
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from levit_spec import DISTILL, FAMILY, LEVIT_CASES  # noqa: E402
from parity import weights_digest  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
PAIRS = [(dk, dv) for dk in (16, 32, 64) for dv in (32, 64, 128)]


# ================================================================================================ attention_posbias
def make_qkv(B, F, H, dk, dv, seed, pad_cols=8, pad_rows=3):
    """A bf16 [B*F*F, H*(2 dk + dv)] view with row stride H*(2 dk + dv) + pad_cols of a buffer whose rows past B*F*F
    are NaN (never to be read), and an fp32 bias table [H, F*F]."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    W = H * (2 * dk + dv)
    big = torch.full((B * F * F + pad_rows, W + pad_cols), NAN, device=DEV, dtype=torch.bfloat16)
    big[:B * F * F, :W] = torch.randn(B * F * F, W, device=DEV, generator=g).bfloat16()
    table = 2.0 * torch.randn(H, F * F, device=DEV, generator=g)
    return big[:B * F * F, :W], table


def run_posbias(qkv, table, B, F, s, H, dk, dv, gelu=True, pad_rows=3):
    Fq = -(-F // s)
    big = torch.full((B * Fq * Fq + pad_rows, H * dv), NAN, device=DEV, dtype=torch.bfloat16)
    out = big[:B * Fq * Fq]
    _lib.attention_posbias(qkv, out, table, B, F, s, H, dk, dv, dk ** -0.5, gelu_out=gelu)
    torch.cuda.synchronize()
    return big, out


@pytest.mark.parametrize("F", [1, 2, 4, 7, 14, 24, 32])
@pytest.mark.parametrize("s", [1, 2])
@pytest.mark.parametrize("dk,dv", PAIRS)
def test_posbias_within_bounds(dk, dv, s, F):
    B, H = 2, 3
    qkv, table = make_qkv(B, F, H, dk, dv, seed=dk * 1000 + dv * 10 + F + s)
    big, out = run_posbias(qkv, table, B, F, s, H, dk, dv)
    Fq = -(-F // s)
    assert torch.isnan(big[B * Fq * Fq:]).all()
    assert not torch.isnan(out).any()
    ref, bound = posbias_reference(qkv, table, B, F, s, H, dk, dv, dk ** -0.5)
    check(out, ref, bound, f"posbias dk={dk} dv={dv} s={s} F={F}")


def test_posbias_without_gelu_and_at_the_key_limit():
    F = 64                                                          # 4096 keys: B200VIT_ATTN_POSBIAS_MAX_KEYS
    assert F * F == _lib.ATTN_POSBIAS_MAX_KEYS
    for s, gelu in ((2, True), (1, False)):
        qkv, table = make_qkv(1, F, 1, 32, 64, seed=7 + s)
        big, out = run_posbias(qkv, table, 1, F, s, 1, 32, 64, gelu=gelu)
        assert torch.isnan(big[out.shape[0]:]).all()
        ref, bound = posbias_reference(qkv, table, 1, F, s, 1, 32, 64, 32 ** -0.5, gelu=gelu)
        check(out, ref, bound, f"posbias F=64 s={s} gelu={gelu}")


@pytest.mark.parametrize("F,s", [(7, 1), (14, 2), (24, 1), (9, 2)])
def test_posbias_keeps_each_image_to_itself(F, s):
    """NaN and Inf in image 1's rows leave every other image's output bit-identical."""
    B, H, dk, dv = 3, 2, 32, 64
    qkv, table = make_qkv(B, F, H, dk, dv, seed=F * 10 + s)
    _, clean = run_posbias(qkv, table, B, F, s, H, dk, dv)
    for bad in (NAN, float("inf")):
        q2 = qkv.clone()
        q2[F * F:2 * F * F:3] = bad
        _, out = run_posbias(q2, table, B, F, s, H, dk, dv)
        Fq = -(-F // s)
        img = torch.arange(B * Fq * Fq, device=DEV) // (Fq * Fq)
        same = ((out == clean) | (torch.isnan(out) & torch.isnan(clean))).all(1)
        assert same[img != 1].all()


# ================================================================================================ Hardswish GEMM
@pytest.mark.parametrize("M,N,K", [(300, 200, 96), (64, 128, 40), (1000, 384, 256)])
def test_hardswish_epilogue_against_fp64(M, N, K):
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) * K ** -0.5 * 3).bfloat16()
    b = torch.randn(N, device=DEV, generator=g)
    big = torch.full((M + 2, N), NAN, device=DEV, dtype=torch.bfloat16)
    _lib.gemm_hardswish(a, w, out_bf16=big[:M], bias=b)
    torch.cuda.synchronize()
    assert torch.isnan(big[M:]).all()
    ref, e = gemm_reference(a, w, bias=b, hardswish=True)
    check(big[:M], ref, e + bf16_ulp(ref.abs() + e) / 2, f"hardswish gemm {M}x{N}x{K}")


def test_gelu_and_hardswish_together_are_rejected():
    a = torch.zeros(64, 64, device=DEV, dtype=torch.bfloat16)
    out = torch.empty(64, 64, device=DEV, dtype=torch.bfloat16)
    rc = _lib.lib().b200vit_gemm_bf16(a.data_ptr(), 64, a.data_ptr(), 64, out.data_ptr(), None, 64, None, None, None,
                                      0, 1e-5, None, None, 64, 64, 64, _lib.EPI_GELU | _lib.EPI_HARDSWISH, None)
    assert rc == -1 and b"exclusive" in _lib.lib().b200vit_last_error()


# ============================================================================================================ model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(LEVIT_CASES))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec against the reference's stored logits and the module's own bf16 graph with the shared
    comparison (fused_reason is None, launches counted, tol 3e-2); both LayerNorm settings, which change nothing."""
    monkeypatch.setitem(P.FAMILIES, "levit", FAMILY)
    monkeypatch.setitem(P.GPU, "levit", dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens("levit", name, ln_mode, monkeypatch)


def distill_model():
    return FAMILY.build(DISTILL).to(DEV, torch.bfloat16), FAMILY.input(DISTILL).to(DEV)


def test_distill_head_against_reference(monkeypatch):
    case = load_golden("levit")["distill"]
    assert weights_digest(FAMILY.build(DISTILL)) == case["weights"]
    m, x = distill_model()
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        _lib.reset_launch_count()
        out, distill = m(x)
        assert _lib.launch_count() > 0
        monkeypatch.setenv("B200VIT_DISABLE_FUSED", "1")
        eo, ed = m(x)
    for got, want in ((out, case["out_fp32"]), (distill, case["distill_fp32"]), (out, eo), (distill, ed)):
        assert got.shape == want.shape
        mx, frac = P.stats(got, want)
        print(f"levit distill: max {mx:.5f} within {frac:.4f}")
        assert mx < 3e-2


def small_model(seed=0, name="dk16_dv32_112"):
    spec = dict(LEVIT_CASES[name], seed=seed)
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


@pytest.mark.parametrize("distill", [False, True])
def test_graphed_forward(distill):
    m, x = distill_model() if distill else small_model()
    with torch.inference_mode():
        want = m(x)
        want = tuple(t.clone() for t in want) if distill else want.clone()
    fwd = GraphedForward(m, x)
    got = fwd(x)
    torch.cuda.synchronize()
    if distill:
        assert isinstance(got, tuple) and all(torch.equal(g, w) for g, w in zip(got, want))
    else:
        assert torch.equal(got, want)


def test_weight_update_needs_refresh_and_running_stats_do_not():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
        m.mlp_head.bias.data.add_(1.0)                    # through .data: the version counter does not move
        m.refresh_fused_weights()
        after = m(x)
    assert torch.allclose(after.float(), before.float() + 1.0, atol=5e-2)
    bn = m.backbone[0].layers[0][0].to_out[2]
    with torch.inference_mode():
        ref = m.forward_eager(x).clone()
    with torch.no_grad():
        bn.running_mean.add_(3.0)                         # in place: picked up by the version counter
    with torch.inference_mode():
        got = m(x)
        want = m.forward_eager(x)
    assert not torch.equal(want, ref)
    assert (got.float() - want.float()).abs().max().item() < 5e-2


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
        h = m.backbone[1].layers[0][0].to_q.register_forward_hook(lambda mod, i, o: seen.append(tuple(o.shape)))
        assert "hooks" in m.fused_reason(x)
        _lib.reset_launch_count()
        m(x)
        assert _lib.launch_count() == 0 and seen == [(2, 16 * 4, 4, 4)]         # 4 heads of 16, stride 2 on 7 x 7
        h.remove()
        assert m.fused_reason(x) is None
