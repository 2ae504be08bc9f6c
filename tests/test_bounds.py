"""The error bounds of oracle/bounds.py are neither loose nor tight (CPU only, small shapes, the GPU sweep's input
distributions).

Tight: an fp32 emulation of the kernels' arithmetic -- an fp32 matmul and the epilogue formula of gemm.cu in fp32,
the patch LayerNorm in fp32 -- passes the checker.
Loose: each defect a persistent kernel could plausibly have, planted into the fp64 reference, is flagged: a dropped
k step, a tile or half a tile of the CTA's previous tile, a bias or residual read one column or one 64-column slab
off, LayerNorm sums or a statistics part of the wrong row or part, a patch row of the previous patch row."""
import math

import pytest
import torch

from oracle import bounds as Bd
from oracle import vit_oracle as O

BM, BN = 128, 128           # tile of the 128-wide instances
GRID = 3                    # persistent CTAs of the emulated launch (= n tiles, so tile - GRID has the same shape)
M, N, K = 5 * BM - 17, 320, 3 * 64 - 24
MODES = ("bias", "lnfold_bias", "lnfold_bias_gelu", "resid_stats", "resid_stats_bias")


def stats_parts(n):
    bn = 256 if n > 128 else 128
    return 2 * ((n + bn - 1) // bn)


def tile_region(t, n=N, m=M):
    nt = (n + BN - 1) // BN
    mb, nb = divmod(t, nt)
    return slice(mb * BM, min(mb * BM + BM, m)), slice(nb * BN, min(nb * BN + BN, n))


def inputs(parts=3, seed=0):
    return Bd.gemm_inputs(M, N, K, parts=parts, seed=seed)


def kwargs(mode, x):
    """gemm_reference keywords of a mode; the output is bf16 except for the residual stream (fp32 + bf16)."""
    kw = {}
    if "bias" in mode.split("_"):
        kw["bias"] = x["bias"]
    if "lnfold" in mode:
        kw.update(ln_sums=x["ln_sums"], col_s=x["col_s"])
    if mode.endswith("gelu"):
        kw["gelu"] = True
    if mode.startswith("resid"):
        kw["resid"] = x["resid"]
    return kw


def emulate(mode, x, eps=1e-5):
    """The kernel's arithmetic in fp32 (gemm.cu epilogue): returns the fp32 value before the output rounding."""
    a, w = x["a"][:, :K].float(), x["w"][:, :K].float()
    v = a @ w.t()
    kw = kwargs(mode, x)
    b = kw.get("bias", torch.zeros(N))
    if "ln_sums" in kw:
        s = kw["ln_sums"]
        s1, s2 = torch.zeros(M), torch.zeros(M)
        for i in range(s.shape[1]):                     # the parts added up in order, in fp32
            s1, s2 = s1 + s[:, i, 0], s2 + s[:, i, 1]
        inv = torch.tensor(1.0 / K, dtype=torch.float32)
        mu = s1 * inv
        rstd = torch.rsqrt((s2 * inv - mu * mu).clamp_min(0) + eps)
        c = (-rstd * mu)[:, None] * kw["col_s"][None] + b[None]
        v = v * rstd[:, None] + c
    elif "bias" in kw:
        v = v + b[None]
    if kw.get("gelu"):
        v = torch.nn.functional.gelu(v)
    if "resid" in kw:
        v = v + kw["resid"][:, :N]
    return v


def emulate_stats(ob):
    """EPI_STATS in fp32 from the bf16 output."""
    x = ob.float()
    wd = Bd.stats_width(N)
    st = torch.zeros(M, stats_parts(N), 2)
    for p in range(stats_parts(N)):
        seg = x[:, p * wd:(p + 1) * wd]
        if seg.shape[1]:
            st[:, p, 0], st[:, p, 1] = seg.sum(1), (seg * seg).sum(1)
    return st


def reference(mode, x, **over):
    kw = kwargs(mode, x)
    kw.update(over)
    if "resid" in kw:
        kw["resid"] = kw["resid"][:, :N]
    ref, e = Bd.gemm_reference(x["a"][:, :K], x["w"][:, :K], **kw)
    return ref, e, Bd.bf16_bound(ref, e)


def flagged(got, ref, bound):
    return Bd.excess(got, ref, bound) > 1.0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("parts", [1, 3, 64])
def test_fp32_emulation_passes(mode, parts):
    x = inputs(parts, seed=parts)
    ref, e, e16 = reference(mode, x)
    v = emulate(mode, x)
    ob = v.bfloat16()
    r32, r16 = Bd.check(v, ref, e, "fp32"), Bd.check(ob, ref, e16, "bf16")
    assert r32 <= 1 and r16 <= 1
    if mode.startswith("resid"):
        sref, sb = Bd.stats_reference(ob, stats_parts(N))
        Bd.check(emulate_stats(ob), sref, sb, "stats")


def test_bf16_bound_is_not_half_an_ulp():
    """A bf16 rounding error reaches 2^-8 relative just above a power of two: 2^-9 would reject correct outputs."""
    v = torch.tensor([1.0 + 0.99 * 2.0 ** -8], dtype=torch.float64)
    got = v.float().bfloat16()
    assert (got.double() - v).abs().item() > 2.0 ** -9 * v.item()
    assert Bd.check(got, v, Bd.bf16_bound(v, torch.zeros_like(v))) <= 1


def test_dropped_k_step_is_flagged():
    for mode in ("bias", "lnfold_bias_gelu"):
        x = inputs()
        ref, e, e16 = reference(mode, x)
        rows, cols = tile_region(7)
        a = x["a"].clone()
        a[rows, 48:64] = 0                      # one 16-wide k step of one tile
        bad, _, _ = reference(mode, dict(x, a=a))
        got = ref.clone()
        got[rows, cols] = bad[rows, cols]
        assert not flagged(ref.float().bfloat16(), ref, e16)
        assert flagged(got.float().bfloat16(), ref, e16), mode
        assert flagged(got.float(), ref, e), mode


def test_tile_of_the_previous_iteration_is_flagged():
    x = inputs()
    ref, _, e16 = reference("lnfold_bias", x)
    t = 2 * GRID + 1
    r1, c1 = tile_region(t)
    r0, c0 = tile_region(t - GRID)
    got = ref.clone()
    got[r1, c1] = ref[r0, c0]
    assert flagged(got.float().bfloat16(), ref, e16)


def test_half_tile_of_the_previous_iteration_is_flagged():
    """Rows 64..127 (the second consumer warpgroup) of one tile from the tile its CTA computed before."""
    x = inputs()
    ref, _, e16 = reference("lnfold_bias_gelu", x)
    t = 2 * GRID
    r1, c1 = tile_region(t)
    r0, _ = tile_region(t - GRID)
    got = ref.clone()
    got[r1.start + 64:r1.start + 128, c1] = ref[r0.start + 64:r0.start + 128, c1]
    assert flagged(got.float().bfloat16(), ref, e16)


@pytest.mark.parametrize("mode", ["bias", "lnfold_bias"])
def test_bias_off_by_one_column_is_flagged(mode):
    x = inputs()
    ref, _, e16 = reference(mode, x)
    b = x["bias"].clone()
    b[128:191] = x["bias"][129:192]                 # inside the 64-column box [128, 192)
    bad, _, _ = reference(mode, x, bias=b)
    assert flagged(bad.float().bfloat16(), ref, e16)


@pytest.mark.parametrize("mode", ["resid_stats", "resid_stats_bias"])
def test_residual_of_the_neighbouring_slab_is_flagged(mode):
    x = inputs()
    ref, e, e16 = reference(mode, x)
    rows, _ = tile_region(4)
    r = x["resid"].clone()
    r[rows, 128:192] = x["resid"][rows, 192:256]
    bad, _, _ = reference(mode, x, resid=r)
    assert flagged(bad.float(), ref, e) and flagged(bad.float().bfloat16(), ref, e16)


@pytest.mark.parametrize("parts", [1, 3])
def test_layernorm_sums_of_the_next_row_are_flagged(parts):
    x = inputs(parts)
    ref, _, e16 = reference("lnfold_bias", x)
    s = x["ln_sums"].clone()
    s[200] = x["ln_sums"][201]
    bad, _, _ = reference("lnfold_bias", x, ln_sums=s)
    assert flagged(bad.float().bfloat16(), ref, e16)


def test_stats_part_shifted_by_one_is_flagged():
    x = inputs()
    ref, e, e16 = reference("resid_stats_bias", x)
    ob = emulate("resid_stats_bias", x).bfloat16()
    sref, sb = Bd.stats_reference(ob, stats_parts(N))
    st = emulate_stats(ob)
    Bd.check(st, sref, sb)
    rows, _ = tile_region(5)
    bad = st.clone()
    bad[rows, 1] = st[rows, 2]
    assert flagged(bad, sref, sb)
    unwritten = st.clone()
    unwritten[rows, stats_parts(N) - 1] = float("nan")          # a slot the kernel never wrote
    assert flagged(unwritten, sref, sb)


def patch_rows(img, p):
    return O.patchify(img.float(), p, p).reshape(-1, img.shape[1] * p * p)


@pytest.mark.parametrize("C,H,W,p", [(3, 64, 96, 16), (3, 28, 42, 14), (1, 14, 21, 7)])
def test_patch_layernorm_emulation_passes_and_previous_patch_row_is_flagged(C, H, W, p):
    g = torch.Generator().manual_seed(C + p)
    img = torch.randn(4, C, H, W, generator=g).bfloat16()
    pd = C * p * p
    gamma, beta = torch.randn(pd, generator=g), torch.randn(pd, generator=g)
    x = patch_rows(img, p)
    ref, bound = Bd.layernorm_reference(x, gamma, beta)
    mu = x.mean(1, keepdim=True)
    rstd = torch.rsqrt(((x - mu) ** 2).mean(1, keepdim=True) + 1e-5)
    emu = ((x - mu) * rstd * gamma + beta).bfloat16()
    assert Bd.check(emu, ref, bound, "patch LN") <= 1
    gw = W // p
    got = emu.clone()
    got[gw:2 * gw] = emu[0:gw]                      # patch row 1 of image 0 written with patch row 0
    assert flagged(got, ref, bound)


def test_bounds_run_in_fp64_on_the_inputs_device():
    x = Bd.gemm_inputs(7, 9, 24, parts=2)
    ref, e = Bd.gemm_reference(x["a"], x["w"], bias=x["bias"], ln_sums=x["ln_sums"], col_s=x["col_s"], gelu=True)
    assert ref.dtype == e.dtype == torch.float64 and ref.shape == e.shape == (7, 9)
    assert (e > 0).all() and math.isfinite(e.max().item())
