"""-m gpu: MobileViT on the H100.  b200vit_attention_groups against an fp64 reference with the per-element bounds of
oracle/attention_bounds.py (group lengths 1 to 4096, one and four heads, non-square maps, rectangular patches), its
isolation (NaN and Inf stay in their group, no read or write outside the addressed rows) and repeatability; the SiLU
depthwise kernel against fp64 and its GELU instance against b200vit_mbconv_dwconv bit for bit; the SiLU GEMM epilogue
with an LN fold and with fp32 outputs at full M; then the model: every case of tests/golden/mobile_vit_spec.py
through the comparison of test_gpu_family_parity.py in both LayerNorm modes, CUDA-graph replay, weight refresh, the
direct transformer call and the eager fall-backs."""
import sys

import pytest
import torch

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR
from oracle.bounds import U, bf16_bound, bf16_ulp, check, gemm_inputs, gemm_reference, stats_reference
from oracle.grid_attention_bounds import group_rows, groups_reference, silu_bound
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from mobile_vit_spec import FAMILY, MOBILE_VIT_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = dict(device=DEV, dtype=torch.bfloat16)
NAN = float("nan")
DH = 8
SCALE = DH ** -0.5


# ================================================================================================ group attention
PAD = 5          # poisoned rows before and after the addressed ones


def run_groups(qkv, B, gh, gw, ph, pw, H):
    """The kernel on qkv placed between NaN rows, writing between NaN rows: returns out; asserts the padding kept."""
    M = B * gh * gw
    big = torch.full((M + 2 * PAD, 3 * H * DH), NAN, device=DEV, dtype=torch.bfloat16)
    big[PAD:PAD + M] = qkv
    obig = torch.full((M + 2 * PAD, H * DH), NAN, device=DEV, dtype=torch.bfloat16)
    _lib.attention_groups(big[PAD:PAD + M], obig[PAD:PAD + M], B, gh, gw, ph, pw, H, DH, SCALE)
    torch.cuda.synchronize()
    assert torch.isnan(obig[:PAD]).all() and torch.isnan(obig[PAD + M:]).all()
    return obig[PAD:PAD + M].clone()


SHAPES = [  # B, gh, gw, ph, pw: group length
    (3, 2, 2, 2, 2),       # 1
    (2, 4, 3, 1, 1),       # 12
    (4, 8, 8, 2, 2),       # 16
    (2, 16, 32, 2, 4),     # 64, rectangular patch, non-square map
    (2, 13, 9, 1, 1),      # 117
    (2, 32, 32, 2, 2),     # 256
    (1, 64, 32, 2, 1),     # 1024
    (1, 64, 64, 1, 1),     # 4096
]


@pytest.mark.parametrize("H", [1, 4])
@pytest.mark.parametrize("B,gh,gw,ph,pw", SHAPES)
def test_attention_groups_within_bounds_and_repeatable(B, gh, gw, ph, pw, H):
    g = torch.Generator(device=DEV).manual_seed(B * gh * gw + ph * 10 + pw + H)
    qkv = (torch.randn(B * gh * gw, 3 * H * DH, device=DEV, generator=g) * 1.5).bfloat16()
    out = run_groups(qkv, B, gh, gw, ph, pw, H)
    assert torch.isfinite(out).all()
    ref, bnd = groups_reference(qkv, B, gh, gw, ph, pw, H, DH, SCALE)
    check(out, ref, bnd, f"groups {B}x{gh}x{gw} patch {ph}x{pw} H={H}")
    assert torch.equal(run_groups(qkv, B, gh, gw, ph, pw, H), out)


@pytest.mark.parametrize("bad", ["nan_q", "inf_k"])
def test_attention_groups_keeps_nan_and_inf_inside_the_group(bad):
    B, gh, gw, ph, pw, H = 2, 8, 12, 2, 2, 4
    g = torch.Generator(device=DEV).manual_seed(7)
    qkv = torch.randn(B * gh * gw, 3 * H * DH, device=DEV, generator=g).bfloat16()
    clean = run_groups(qkv, B, gh, gw, ph, pw, H)
    y, x = 5, 7                                           # group (b=1, i=1, j=1)
    row = (1 * gh + y) * gw + x
    dirty = qkv.clone()
    if bad == "nan_q":
        dirty[row, 3] = NAN                               # head 0's query
    else:
        dirty[row, H * DH + 2 * DH + 1] = float("inf")    # head 2's key
    out = run_groups(dirty, B, gh, gw, ph, pw, H)
    rows = group_rows(B, gh, gw, ph, pw, DEV)
    inside = torch.zeros(B * gh * gw, dtype=torch.bool, device=DEV)
    inside[rows[(1 * ph + 1) * pw + 1]] = True
    same = (out == clean) | (torch.isnan(out) & torch.isnan(clean))
    assert same[~inside].all()
    assert not torch.isfinite(out[inside]).all()


# ================================================================================================ depthwise SiLU
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("B,h,w,C", [(2, 9, 13, 64), (1, 27, 27, 136), (3, 7, 5, 8), (2, 32, 32, 256)])
def test_dwconv_silu_against_fp64(B, h, w, C, stride):
    g = torch.Generator(device=DEV).manual_seed(B * h * w + C + stride)
    x = torch.randn(B * h * w, C, device=DEV, generator=g).bfloat16()
    w9 = torch.randn(9, C, device=DEV, generator=g) / 3
    bias = torch.randn(C, device=DEV, generator=g)
    oh, ow = -(-h // stride), -(-w // stride)
    big = torch.full((B * oh * ow + 2, C), NAN, device=DEV, dtype=torch.bfloat16)
    y = big[:B * oh * ow]
    _lib.mbconv_dwconv_ex(x, w9, bias, y, None, B, h, w, stride, act="silu")
    torch.cuda.synchronize()
    assert torch.isnan(big[B * oh * ow:]).all()
    xi = x.double().reshape(B, h, w, C).permute(0, 3, 1, 2)
    conv = torch.nn.functional.conv2d(xi, w9.double().t().reshape(C, 1, 3, 3), bias.double(), stride=stride,
                                      padding=1, groups=C)
    ref = torch.nn.functional.silu(conv).permute(0, 2, 3, 1).reshape(-1, C)
    mag = torch.nn.functional.conv2d(xi.abs(), w9.double().abs().t().reshape(C, 1, 3, 3), bias.double().abs(),
                                     stride=stride, padding=1, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    pre = conv.permute(0, 2, 3, 1).reshape(-1, C)
    # fp32 taps (slope of SiLU <= 1.1), ex2 / rcp approximations and the products' roundings
    e = 1.1 * 12 * U * mag + 16 * U * (ref.abs() + pre.abs()) + 1e-30
    check(y, ref, e + bf16_ulp(ref.abs() + e) / 2, f"dwconv silu {B}x{h}x{w}x{C} s={stride}")
    y2 = torch.empty_like(y)
    _lib.mbconv_dwconv_ex(x, w9, bias, y2, None, B, h, w, stride, act="silu")
    torch.cuda.synchronize()
    assert torch.equal(y2, y)


@pytest.mark.parametrize("stride", [1, 2])
def test_dwconv_ex_gelu_gives_the_bits_of_mbconv_dwconv(stride):
    B, h, w, C = 2, 15, 11, 72
    g = torch.Generator(device=DEV).manual_seed(3 + stride)
    x = torch.randn(B * h * w, C, device=DEV, generator=g).bfloat16()
    w9 = torch.randn(9, C, device=DEV, generator=g) / 3
    bias = torch.randn(C, device=DEV, generator=g)
    oh, ow = -(-h // stride), -(-w // stride)
    y0, y1 = (torch.empty(B * oh * ow, C, device=DEV, dtype=torch.bfloat16) for _ in range(2))
    p0, p1 = (torch.empty(B, _lib.mbconv_parts(oh, ow), C, device=DEV) for _ in range(2))
    _lib.mbconv_dwconv(x, w9, bias, y0, p0, B, h, w, stride)
    _lib.mbconv_dwconv_ex(x, w9, bias, y1, p1, B, h, w, stride, act="gelu")
    torch.cuda.synchronize()
    assert torch.equal(y0, y1) and torch.equal(p0, p1)


# ================================================================================================ SiLU GEMM epilogue
@pytest.mark.parametrize("M,N,K", [(4096, 192, 96), (3000, 480, 120), (8192, 576, 144)])
def test_silu_with_ln_fold_against_bounds(M, N, K):
    d = gemm_inputs(M, N, K, parts=2, seed=M + N, device=DEV)
    out = torch.full((M + 2, N), NAN, device=DEV, dtype=torch.bfloat16)
    _lib.gemm_act(d["a"], d["w"], act="silu", out_bf16=out[:M], bias=d["bias"], ln_sums=d["ln_sums"],
                  col_s=d["col_s"])
    torch.cuda.synchronize()
    assert torch.isnan(out[M:]).all()
    y, e_y = gemm_reference(d["a"], d["w"], bias=d["bias"], ln_sums=d["ln_sums"], col_s=d["col_s"])
    ref, e = silu_bound(y, e_y)
    check(out[:M], ref, bf16_bound(ref, e), f"silu lnfold {M}x{N}x{K}")


@pytest.mark.parametrize("M,N,K", [(4096, 96, 576), (2048, 384, 96)])
def test_silu_with_fp32_and_bf16_outputs_against_bounds(M, N, K):
    d = gemm_inputs(M, N, K, seed=M + K, device=DEV)
    o32 = torch.full((M, N), NAN, device=DEV)
    o16 = torch.full((M, N), NAN, device=DEV, dtype=torch.bfloat16)
    _lib.gemm_act(d["a"], d["w"], act="silu", out_f32=o32, out_bf16=o16, bias=d["bias"])
    torch.cuda.synchronize()
    y, e_y = gemm_reference(d["a"], d["w"], bias=d["bias"])
    ref, e = silu_bound(y, e_y)
    check(o32, ref, e, f"silu fp32 {M}x{N}x{K}")
    assert torch.equal(o16, o32.bfloat16())


@pytest.mark.parametrize("M,N,K", [(4096, 96, 576), (3000, 384, 96), (8192, 576, 144)])
def test_silu_with_row_statistics_against_bounds(M, N, K):
    """EPI_SILU with EPI_STATS (and the LN fold) at full M: the bf16 output within its bound, and the statistics those
    exact bf16 values have, part by part."""
    d = gemm_inputs(M, N, K, parts=2, seed=M + 7 * N, device=DEV)
    parts = _lib.stats_parts(N)
    out = torch.full((M, N), NAN, device=DEV, dtype=torch.bfloat16)
    st = torch.full((M, parts, 2), NAN, device=DEV)
    _lib.gemm_act(d["a"], d["w"], act="silu", out_bf16=out, bias=d["bias"], ln_sums=d["ln_sums"], col_s=d["col_s"],
                  stats_out=st)
    torch.cuda.synchronize()
    y, e_y = gemm_reference(d["a"], d["w"], bias=d["bias"], ln_sums=d["ln_sums"], col_s=d["col_s"])
    ref, e = silu_bound(y, e_y)
    check(out, ref, bf16_bound(ref, e), f"silu stats {M}x{N}x{K}")
    sref, sbound = stats_reference(out, parts)
    check(st, sref, sbound, f"silu stats {M}x{N}x{K}: row statistics")


# ================================================================================================ strided im2col
@pytest.mark.parametrize("B,H,W,C", [(2, 16, 16, 64), (3, 7, 5, 40)])
def test_im2col_of_a_column_slice_matches_the_contiguous_map(B, H, W, C):
    """conv_im2col_nhwc on the right half of an [M, 2C] buffer (b200vit_conv_im2col_nhwc_ex) gives the bits of the
    same map stored contiguously, and never reads the left half (NaN there)."""
    g = torch.Generator(device=DEV).manual_seed(B * H * W + C)
    x = torch.randn(B * H * W, C, device=DEV, generator=g).bfloat16()
    cat = torch.full((B * H * W, 2 * C), NAN, device=DEV, dtype=torch.bfloat16)
    cat[:, C:] = x
    want = torch.empty(B * H * W, 9 * C, device=DEV, dtype=torch.bfloat16)
    got = torch.empty_like(want)
    _lib.conv_im2col_nhwc(x, want, B, H, W, 3, 1, 1)
    _lib.conv_im2col_nhwc(cat[:, C:], got, B, H, W, 3, 1, 1)
    torch.cuda.synchronize()
    assert not torch.isnan(got).any() and torch.equal(got, want)


# ============================================================================================================ model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(MOBILE_VIT_CASES))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec against the reference's stored logits and the module's own bf16 graph with the shared
    comparison (fused_reason is None, launches counted, tol 3e-2), in both LayerNorm modes."""
    monkeypatch.setitem(P.FAMILIES, "mobile_vit", FAMILY)
    monkeypatch.setitem(P.GPU, "mobile_vit", dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens("mobile_vit", name, ln_mode, monkeypatch)


def small_model(seed=0, name="xxs_expansion2"):
    spec = dict(MOBILE_VIT_CASES[name], seed=seed)
    return FAMILY.build(spec).to(DEV, torch.bfloat16), FAMILY.input(spec).to(DEV)


def test_graphed_forward_replays_the_eager_launches_bit_for_bit():
    m, x = small_model()
    with torch.inference_mode():
        want = m(x).clone()
    fwd = GraphedForward(m, x)
    got = fwd(x)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_running_stats_and_data_writes_change_the_next_output():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
        m.to_logits[2].weight.data.mul_(2.0)              # through .data: the version counter does not move
        m.refresh_fused_weights()
        after = m(x).clone()
    assert torch.allclose(after.float(), 2 * before.float(), rtol=2e-2, atol=2e-2)
    assert not torch.equal(after, before)
    bn = m.trunk[1][1].conv2[1]
    with torch.no_grad():
        bn.running_mean.add_(0.5)                         # in place: picked up by the version counter
    with torch.inference_mode():
        got = m(x)
        want = m.forward_eager(x)
    assert not torch.equal(got, after)
    assert (got.float() - want.float()).abs().max().item() < 5e-2


def test_direct_transformer_call_against_its_pytorch_graph():
    m, _ = small_model()
    tr = m.trunk[0][1].transformer
    g = torch.Generator(device=DEV).manual_seed(11)
    tok = torch.randn(2, 4, 64, tr.layers[0][0].norm.normalized_shape[0], device=DEV, generator=g).bfloat16()
    with torch.inference_mode():
        assert tr.fused_reason(tok) is None
        _lib.reset_launch_count()
        got = tr(tok)
        torch.cuda.synchronize()
        assert _lib.launch_count() > 0
        want = tr.forward_eager(tok)
    assert got.shape == tok.shape and got.dtype == torch.bfloat16
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
        h = m.trunk[0][1].transformer.layers[0][0].to_qkv.register_forward_hook(
            lambda mod, i, o: seen.append(tuple(o.shape)))
        assert "hooks" in m.fused_reason(x)
        assert "hooks" in m.trunk[0][1].transformer.fused_reason(torch.zeros(2, 4, 64, 64, **BF))
        got = m(x)                  # the PyTorch graph; the transformers without hooks still run fused inside it
        assert seen == [(2, 4, 64, 96)]                   # 16 x 16 map, 2 x 2 patches: 4 groups of 64 tokens
        assert (got.float() - m.forward_eager(x).float()).abs().max().item() < 5e-2
        h.remove()
        assert m.fused_reason(x) is None
        m.trunk[0][0].conv[1].train()
        assert "BatchNorm2d" in m.fused_reason(x)
        m.eval()
        assert m.fused_reason(x.float()) is not None
        assert m.fused_reason(x[:, :, :100].contiguous()) is not None   # 13 x 16 maps: not divisible by 2 x 2
