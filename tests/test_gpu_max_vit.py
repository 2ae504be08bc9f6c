"""-m gpu: MaxViT on the H100.  b200vit_attention_window_relpos against an fp64 reference with per-element bounds (block
and grid windows, every window size and head width, non-square maps), what it writes and which rows it reads;
b200vit_mbconv_dwconv, the squeeze-excitation kernels and the SiLU / sigmoid GEMM epilogues against fp64; then the
model: every case of tests/golden/max_vit_spec.py through the comparison of test_gpu_family_parity.py, CUDA-graph
replay, weight refresh and the eager fall-backs."""
import sys

import pytest
import torch

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR
from oracle.bounds import C_ACC, U, bf16_ulp, check
from oracle.grid_attention_bounds import relpos_reference, window_rows
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from max_vit_spec import FAMILY, MAX_VIT_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
WIDTHS = (32, 64, 80, 128)


# ================================================================================================ window attention
def make_inputs(B, gh, gw, w, H, dh, seed, pad_rows=3):
    """qkv bf16 [B*gh*gw, 3 H dh] as the head of a buffer whose rows past it are NaN (never to be read), and a bias
    table [H, (2w-1)^2]."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    M = B * gh * gw
    big = torch.full((M + pad_rows, 3 * H * dh), NAN, device=DEV, dtype=torch.bfloat16)
    big[:M] = torch.randn(M, 3 * H * dh, device=DEV, generator=g).bfloat16()
    table = 2.0 * torch.randn(H, (2 * w - 1) ** 2, device=DEV, generator=g)
    return big[:M], table


def run_relpos(qkv, table, B, gh, gw, w, grid, H, dh, pad_rows=3):
    big = torch.full((B * gh * gw + pad_rows, H * dh), NAN, device=DEV, dtype=torch.bfloat16)
    out = big[:B * gh * gw]
    _lib.attention_window_relpos(qkv, out, table, B, gh, gw, w, grid, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    return big, out


@pytest.mark.parametrize("dh", WIDTHS)
@pytest.mark.parametrize("w,gh,gw", [(2, 4, 6), (3, 9, 6), (4, 8, 16), (5, 10, 5), (6, 12, 6), (7, 14, 28), (8, 16, 8)])
@pytest.mark.parametrize("grid", [False, True])
def test_relpos_within_bounds(grid, w, gh, gw, dh):
    B, H = 2, 2
    qkv, table = make_inputs(B, gh, gw, w, H, dh, seed=dh * 100 + w * 10 + grid)
    big, out = run_relpos(qkv, table, B, gh, gw, w, grid, H, dh)
    assert torch.isnan(big[B * gh * gw:]).all()                  # nothing past the map is written
    assert not torch.isnan(out).any()                            # ... and every row of it is
    ref, bound = relpos_reference(qkv, table, B, gh, gw, w, grid, H, dh, dh ** -0.5)
    check(out, ref, bound, f"relpos grid={grid} w={w} {gh}x{gw} dh={dh}")


@pytest.mark.parametrize("grid", [False, True])
def test_relpos_keeps_a_nan_inside_its_window(grid):
    """NaN and Inf in one token's q, k and v leave every row outside that token's window bit-identical."""
    B, gh, gw, w, H, dh = 2, 14, 21, 7, 2, 32
    qkv, table = make_inputs(B, gh, gw, w, H, dh, seed=11)
    _, clean = run_relpos(qkv, table, B, gh, gw, w, grid, H, dh)
    rows = window_rows(B, gh, gw, w, w, DEV, dilated=grid)
    tok = int(rows[5, 10])
    inside = torch.zeros(B * gh * gw, dtype=torch.bool, device=DEV)
    inside[rows[5]] = True
    for bad in (NAN, float("inf")):
        q2 = qkv.clone()
        q2[tok] = bad
        _, out = run_relpos(q2, table, B, gh, gw, w, grid, H, dh)
        same = ((out == clean) | (torch.isnan(out) & torch.isnan(clean))).all(1)
        assert same[~inside].all()
        assert not same[inside].all()


# ================================================================================================ MBConv kernels
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("B,h,w,C", [(2, 9, 13, 64), (1, 27, 27, 136), (3, 7, 5, 8), (2, 56, 56, 256)])
def test_mbconv_dwconv_against_fp64_and_repeatable(B, h, w, C, stride):
    g = torch.Generator(device=DEV).manual_seed(B * h * w + C + stride)
    x = torch.randn(B * h * w, C, device=DEV, generator=g).bfloat16()
    w9 = torch.randn(9, C, device=DEV, generator=g) / 3
    bias = torch.randn(C, device=DEV, generator=g)
    oh, ow = -(-h // stride), -(-w // stride)
    big = torch.full((B * oh * ow + 2, C), NAN, device=DEV, dtype=torch.bfloat16)
    y = big[:B * oh * ow]
    part = torch.full((B, _lib.mbconv_parts(oh, ow), C), NAN, device=DEV)
    _lib.mbconv_dwconv(x, w9, bias, y, part, B, h, w, stride)
    torch.cuda.synchronize()
    assert torch.isnan(big[B * oh * ow:]).all()
    xi = x.double().reshape(B, h, w, C).permute(0, 3, 1, 2)
    conv = torch.nn.functional.conv2d(xi, w9.double().t().reshape(C, 1, 3, 3), bias.double(), stride=stride,
                                      padding=1, groups=C)
    ref = torch.nn.functional.gelu(conv).permute(0, 2, 3, 1).reshape(-1, C)
    mag = torch.nn.functional.conv2d(xi.abs(), w9.double().abs().t().reshape(C, 1, 3, 3), bias.double().abs(),
                                     stride=stride, padding=1, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    e = 1.13 * 12 * U * mag + 8 * U * ref.abs() + 1.5e-5      # fp32 taps (slope of GELU <= 1.13), its fit within 1.2e-5
    check(y, ref, e + bf16_ulp(ref.abs() + e) / 2, f"dwconv {B}x{h}x{w}x{C} s={stride}")
    # the partial sums: exactly the fp32 sums of the rounded outputs, each slot written
    assert not torch.isnan(part).any()
    tot = part.double().sum(1)
    want = y.double().reshape(B, oh * ow, C).sum(1)
    assert torch.allclose(tot, want, rtol=1e-5, atol=1e-3)
    y2, part2 = torch.empty_like(y), torch.empty_like(part)
    _lib.mbconv_dwconv(x, w9, bias, y2, part2, B, h, w, stride)
    torch.cuda.synchronize()
    assert torch.equal(y2, y) and torch.equal(part2, part)


def test_se_pool_and_scale():
    B, P, C, n = 3, 5, 72, 300
    g = torch.Generator(device=DEV).manual_seed(5)
    part = torch.randn(B, P, C, device=DEV, generator=g) * 10
    pooled = torch.empty(B, C, device=DEV, dtype=torch.bfloat16)
    _lib.se_pool(part, pooled, n)
    want = part.double().sum(1) / n
    check(pooled, want, 8 * U * part.double().abs().sum(1) / n + bf16_ulp(want.abs()) / 2, "se_pool")
    h = torch.randn(B * n, C, device=DEV, generator=g).bfloat16()
    gate = torch.rand(B, C, device=DEV, generator=g).bfloat16()
    h0 = h.clone()
    _lib.se_scale(h, gate, B, n)
    torch.cuda.synchronize()
    want = (h0.float().reshape(B, n, C) * gate.float()[:, None]).reshape(B * n, C).bfloat16()
    assert torch.equal(h, want)


@pytest.mark.parametrize("act", ["silu", "sigmoid"])
@pytest.mark.parametrize("M,N,K", [(1, 64, 256), (64, 768, 3072), (300, 200, 96), (256, 3072, 768)])
def test_silu_and_sigmoid_epilogues_against_fp64(act, M, N, K):
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) * K ** -0.5 * 3).bfloat16()
    big = torch.full((M + 2, N), NAN, device=DEV, dtype=torch.bfloat16)
    (_lib.gemm_silu if act == "silu" else _lib.gemm_sigmoid)(a, w, out_bf16=big[:M])
    torch.cuda.synchronize()
    assert torch.isnan(big[M:]).all()
    y = a.double() @ w.double().t()
    ref = y * torch.sigmoid(y) if act == "silu" else torch.sigmoid(y)
    e_y = (C_ACC * K + 2) * U * (a.double().abs() @ w.double().abs().t())
    slope = 1.1 if act == "silu" else 0.25
    e = slope * e_y + 8 * U * ref.abs() + 4 * U * (y.abs() * (act == "silu")) + 1e-30
    check(big[:M], ref, e + bf16_ulp(ref.abs() + e) / 2, f"{act} gemm {M}x{N}x{K}")


# ============================================================================================================ model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(MAX_VIT_CASES))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec against the reference's stored logits and the module's own bf16 graph with the shared
    comparison (fused_reason is None, launches counted, tol 3e-2), in both LayerNorm modes."""
    monkeypatch.setitem(P.FAMILIES, "max_vit", FAMILY)
    monkeypatch.setitem(P.GPU, "max_vit", dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens("max_vit", name, ln_mode, monkeypatch)


def small_model(seed=0, name="odd_nonsquare_c1"):
    spec = dict(MAX_VIT_CASES[name], seed=seed)
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


def test_weight_update_needs_refresh_and_running_stats_do_not():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
        m.mlp_head[2].bias.data.add_(1.0)                 # through .data: the version counter does not move
        m.refresh_fused_weights()
        after = m(x)
    assert torch.allclose(after.float(), before.float() + 1.0, atol=5e-2)
    bn = m.layers[2][0].fn[8]                             # the residual MBConv's last BatchNorm (stage 2)
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
        h = m.layers[0][6].fn.to_qkv.register_forward_hook(lambda mod, i, o: seen.append(tuple(o.shape)))
        assert "hooks" in m.fused_reason(x)
        _lib.reset_launch_count()
        m(x)
        assert _lib.launch_count() == 0 and seen == [(2 * 2 * 4, 49, 96)]     # 2 x 4 grid windows of 7 x 7, dim 32
        h.remove()
        assert m.fused_reason(x) is None
        m.train()
        assert "dropout is active" in m.fused_reason(x)            # the case keeps the default dropout 0.1
