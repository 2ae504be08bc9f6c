"""-m gpu: the persistent kernels against fp64 references with per-element bounds (oracle/bounds.py) where production
runs them -- several tiles (or patch-row slabs) per CTA.

b200vit_gemm_bf16 launches min(tiles, SMs) CTAs and each loops over tile = blockIdx.x + i * gridDim.x: the smem ring's
stage / phase, the double-buffered bias / col_s / LN-sum vectors, the residual slab count and the TMA-store staging
all carry over from one tile to the next.  Every one of the eight kernel instances runs at 1, S - 1, S, S + 1, 2S + 1
and 4S + 3 tiles (S = the device's SM count), at k-block counts of 1, STAGES - 1, STAGES + 1 and 2 STAGES + 1, with
the epilogue flags the encoder issues.  Every output element and statistics slot must be within its bound, sentinels
past M and between N and the row stride stay untouched, and the first and last row tiles of every multi-wave launch,
launched again alone, give the same bits.  The persistent patch kernels load at least three patch-row slabs per CTA."""
import pytest
import torch
import torch.nn.functional as F

from oracle import bounds as Bd
from oracle import vit_oracle as O
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.vit_for_small_dataset import SPT_SHIFTS

pytestmark = pytest.mark.gpu
DEV = "cuda"
CHUNK = 8192            # rows per fp64 reference chunk
F32_SENT, BF16_SENT = -3.0, 7.0
WORST = {}              # worst |got - ref| / bound per kernel, printed by test_report


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def cdiv(a, b):
    return -(-a // b)


def note(name, ratio):
    WORST[name] = max(WORST.get(name, 0.0), ratio)


# ------------------------------------------------------------------------------------------------------------ GEMM
# instance -> (BLOCK_N, STAGES, kind); kind "f32": fp32 output (direct store), "tma": bf16 output through TMA
# stores, "res": residual + statistics.  Each case: (N, ldo - N, hook 12, hook 14) per tile-count index, flags mode.
INSTANCES = {
    "128x6": (128, 6, "f32", [(100, 4, 0, 0), (128, 0, 0, 0), (77, 3, 0, 0), (120, 8, 0, 0), (128, 0, 0, 0),
                              (64, 8, 0, 0)]),
    "256x4": (256, 4, "f32", [(200, 0, 0, 0), (256, 8, 0, 0), (255, 1, 0, 0), (136, 4, 0, 0), (320, 0, 0, 0),
                              (768, 16, 0, 0)]),
    "128x5_tma": (128, 5, "tma", [(128, 0, 0, 0), (96, 8, 0, 0), (64, 0, 0, 0), (120, 8, 0, 0), (128, 8, 0, 0),
                                  (72, 0, 0, 0)]),
    "256x3_tma": (256, 3, "tma", [(256, 0, 0, 0), (200, 8, 0, 0), (136, 0, 0, 0), (248, 8, 0, 0), (320, 0, 0, 0),
                                  (768, 8, 0, 0)]),
    "128x4_res_tma": (128, 4, "res", [(64, 0, 0, 0), (96, 8, 0, 0), (128, 0, 0, 0), (120, 8, 0, 0), (320, 0, 0, 0),
                                      (200, 8, 0, 0)]),
    "256x3_res": (256, 3, "res", [(200, 0, 2, 0), (250, 2, 0, 0), (256, 8, 2, 0), (201, 3, 0, 0), (320, 0, 2, 0),
                                  (330, 2, 0, 0)]),
    "128x4_res": (128, 4, "res", [(100, 4, 0, 0), (77, 3, 0, 0), (128, 0, 0, 1), (64, 8, 0, 1), (320, 0, 1, 1),
                                  (125, 3, 0, 0)]),
}
TILE_TARGETS = [lambda s: 1, lambda s: s - 1, lambda s: s, lambda s: s + 1, lambda s: 2 * s + 1,
                lambda s: 4 * s + 3]
KB = [lambda st: 2 * st + 1, lambda st: 1, lambda st: st - 1, lambda st: st + 1, lambda st: 2 * st + 1,
      lambda st: st + 1]
K_SHORT = [0, 24, 0, 7, 24, 0]             # K = 64 kb - K_SHORT: K % 64 != 0 (and odd once)
PARTS = [1, 64, "D", 1, "D", 64]           # ln_parts: one, stats_parts(K) as the layer chain passes them, the maximum
MODES = {"f32": ["bias", "lnfold_bias", "lnfold_bias_gelu"] * 2,
         "tma": ["bias", "lnfold_bias", "lnfold_bias_gelu"] * 2,
         "res": ["resid_stats_bias_separate", "resid_stats", "resid_stats_bias", "resid_stats_separate",
                 "resid_stats_bias", "resid_stats_bias_separate"]}


def route(N, ldo, res, out_f32, hook12, hook14):
    """The instance b200vit_gemm_bf16 picks (gemm.cu, the end of b200vit_gemm_bf16)."""
    tma_ok = not hook14 and (ldo | N) % 8 == 0 and (res or not out_f32)
    wide = (N > 128 and not (res and tma_ok)) if hook12 == 0 else hook12 == 2
    if tma_ok and not (res and wide):
        return "128x4_res_tma" if res else ("256x3_tma" if wide else "128x5_tma")
    if wide:
        return "256x3_res" if res else "256x4"
    return "128x4_res" if res else "128x6"


def run_gemm(x, M, N, K, ldo, mode, kind, bf16_too, hook12, hook14, rows=None):
    """One launch over rows `rows` of the inputs into sentinel-filled buffers of two extra rows and row stride ldo;
    returns (bf16 buffer, fp32 buffer or None, stats or None)."""
    rows = rows if rows is not None else slice(0, M)
    a = x["a"][rows]
    m = a.shape[0]
    res = kind == "res"
    want_f32 = kind == "f32" or res
    want_bf16 = kind != "f32" or bf16_too
    ob_full = torch.full((m + 2, ldo), BF16_SENT, device=DEV, dtype=torch.bfloat16)
    of_full = None
    kw = dict(k=K)
    if "bias" in mode.split("_"):
        kw["bias"] = x["bias"]
    if "lnfold" in mode:
        kw.update(ln_sums=x["ln_sums"][rows].contiguous(), col_s=x["col_s"])
    if mode.endswith("gelu"):
        kw["gelu"] = True
    st = None
    if res:
        in_place = not mode.endswith("separate")
        r_full = torch.cat([x["resid"][rows], torch.full((2, ldo), 11.0, device=DEV)])
        of_full = r_full.clone() if in_place else torch.full((m + 2, ldo), F32_SENT, device=DEV)
        kw["resid"] = of_full[:m, :N] if in_place else r_full[:m, :N]
        st = torch.full((m, _lib.stats_parts(N), 2), float("nan"), device=DEV)
        kw["stats_out"] = st
    elif want_f32:
        of_full = torch.full((m + 2, ldo), F32_SENT, device=DEV)
    L = _lib.lib()
    L.b200vit_debug_set(12, hook12)
    L.b200vit_debug_set(14, hook14)
    try:
        _lib.gemm(a, x["w"], out_bf16=ob_full[:m, :N] if want_bf16 else None,
                  out_f32=of_full[:m, :N] if of_full is not None else None, n=N, **kw)
        torch.cuda.synchronize()
    finally:
        L.b200vit_debug_set(12, 0)
        L.b200vit_debug_set(14, 0)
    return (ob_full if want_bf16 else None), of_full, st


def check_gemm(name, x, M, N, K, mode, ob_full, of_full, st):
    """Every element of both outputs and every statistics slot within its bound, chunk by chunk on the GPU."""
    kw = {}
    if "bias" in mode.split("_"):
        kw["bias"] = x["bias"]
    if "lnfold" in mode:
        kw.update(col_s=x["col_s"])
    for r0 in range(0, M, CHUNK):
        rs = slice(r0, min(r0 + CHUNK, M))
        ck = dict(kw)
        if "lnfold" in mode:
            ck["ln_sums"] = x["ln_sums"][rs]
        if mode.startswith("resid"):
            ck["resid"] = x["resid"][rs, :N]
        ref, e = Bd.gemm_reference(x["a"][rs, :K], x["w"][:, :K], gelu=mode.endswith("gelu"), **ck)
        if of_full is not None:
            note(name + " fp32", Bd.check(of_full[rs, :N], ref, e, f"{name} {mode} fp32 rows {r0}+"))
            if "lnfold" not in mode:
                # the accumulation error in units of K u |A||W|^T, past the fp32 adds of bias and residual (C_ACC)
                kua = K * Bd.U * (x["a"][rs, :K].double().abs() @ x["w"][:, :K].double().abs().t())
                adds = 2 * Bd.U * (ref.abs() + ck.get("bias", torch.zeros(N, device=DEV)).double().abs()
                                   + (ck["resid"].double().abs() if "resid" in ck else 0))
                d = ((of_full[rs, :N].double() - ref).abs() - adds).clamp_min(0)
                note("accumulation / (K u abs)", (d / kua).max().item())
        if ob_full is not None:
            note(name + " bf16", Bd.check(ob_full[rs, :N], ref, Bd.bf16_bound(ref, e), f"{name} {mode} bf16 rows {r0}+"))
        if st is not None:
            sref, sb = Bd.stats_reference(ob_full[rs, :N], st.shape[1])
            note(name + " stats", Bd.check(st[rs], sref, sb, f"{name} stats rows {r0}+"))


@pytest.mark.parametrize("case", range(6))
@pytest.mark.parametrize("name", list(INSTANCES))
def test_gemm_instance_persistent(name, case):
    S = sms()
    block_n, stages, kind, ns = INSTANCES[name]
    N, pad, hook12, hook14 = ns[case]
    ldo = N + pad
    mode = MODES[kind][case]
    target = TILE_TARGETS[case](S)
    kb = KB[case](stages)
    K = 64 * kb - K_SHORT[case]
    lda = cdiv(K, 8) * 8 + (8 if case % 2 == 0 else 0)
    ldw = cdiv(K, 8) * 8 + (16 if case % 3 == 0 else 0)
    parts = _lib.stats_parts(K) if PARTS[case] == "D" else PARTS[case]
    bf16_too = kind == "f32" and case % 2 == 1
    n_tiles = cdiv(N, block_n)
    m_tiles = cdiv(target, n_tiles)
    M = m_tiles * 128 - (case * 13 + 5) % 128 if target > 1 else 91
    # what this case claims to test, from launch_gemm's formulas
    assert route(N, ldo, kind == "res", kind != "tma", hook12, hook14) == name
    tiles = cdiv(M, 128) * n_tiles
    per_cta = cdiv(tiles, min(tiles, S))
    assert cdiv(K, 64) == kb and per_cta == cdiv(target, min(target, S))
    if n_tiles == 1:
        assert tiles == target
    x = Bd.gemm_inputs(M, N, K, parts=parts, lda=lda, ldw=ldw, ldo=ldo, seed=1000 * case + N, device=DEV)
    ob_full, of_full, st = run_gemm(x, M, N, K, ldo, mode, kind, bf16_too, hook12, hook14)
    check_gemm(name, x, M, N, K, mode, ob_full, of_full, st)
    note(f"{name} tiles/CTA", per_cta)
    # sentinels: rows past M, columns between N and ldo (in place: the residual that was there)
    if ob_full is not None:
        assert (ob_full[M:] == BF16_SENT).all() and (ob_full[:, N:] == BF16_SENT).all()
    if of_full is not None:
        if mode.startswith("resid") and not mode.endswith("separate"):
            assert torch.equal(of_full[:M, N:], x["resid"][:, N:]) and (of_full[M:] == 11.0).all()
        else:
            assert (of_full[M:] == F32_SENT).all() and (of_full[:, N:] == F32_SENT).all()
        if ob_full is not None:
            assert torch.equal(ob_full[:M, :N], of_full[:M, :N].bfloat16())
    if tiles <= S:
        return
    # position invariance: the first and the last row tile, launched alone, give the big launch's bits
    for rows in (slice(0, 128), slice((cdiv(M, 128) - 1) * 128, M)):
        ob1, of1, st1 = run_gemm(x, M, N, K, ldo, mode, kind, bf16_too, hook12, hook14, rows=rows)
        m = rows.stop - rows.start
        for big, one in ((ob_full, ob1), (of_full, of1)):
            if big is not None:
                assert torch.equal(big[rows, :N], one[:m, :N]), (name, rows)
        if st is not None:
            assert torch.equal(st[rows], st1), (name, rows)


def test_patch_embed_tma_persistent():
    """<256,4,PATCH>: 98-row patch tiles (7 patch rows of a 224 x 224 image), at least three tiles per CTA, against
    LayerNorm -> Linear in fp64 with the folded weights and the statistics the launch computed."""
    S = sms()
    B, C, H, W, D = S // 2 + 1, 3, 224, 224, 768
    g = torch.Generator(device=DEV).manual_seed(5)
    pd = C * 256
    img = torch.randn(B, C, H, W, device=DEV, generator=g).bfloat16()
    gamma, be = 1 + 0.2 * torch.randn(pd, device=DEV, generator=g), 0.1 * torch.randn(pd, device=DEV, generator=g)
    w = (torch.randn(D, pd, device=DEV, generator=g) / pd ** 0.5).bfloat16().float()
    b = 0.1 * torch.randn(D, device=DEV, generator=g)
    w_perm = (w * gamma[None]).view(D, 256, C).permute(0, 2, 1).reshape(D, pd).bfloat16().contiguous()
    col_s = w_perm.float().sum(1).contiguous()
    bias = (w @ be + b).contiguous()
    n = (H // 16) * (W // 16)
    # launch_gemm's tiles: 7 of the 14 patch rows per tile (7 x 14 = 98 <= 128 rows), 256-wide N tiles
    tiles = B * 2 * cdiv(D, 256)
    assert tiles // min(tiles, S) >= 3                  # every CTA computes at least three tiles
    note("256x4_patch tiles/CTA", cdiv(tiles, S))

    def launch(im):
        y = torch.full((im.shape[0] * n, D), float("nan"), device=DEV)
        stats = torch.zeros(im.shape[0] * n, 2, device=DEV)
        _lib.patch_embed_tma(im, w_perm, bias, col_s, stats, y)
        torch.cuda.synchronize()
        return y, stats

    y, stats = launch(img)
    # A in the kernel's K order (c, p1, p2)
    a = img.view(B, C, H // 16, 16, W // 16, 16).permute(0, 2, 4, 1, 3, 5).reshape(B * n, pd)
    for r0 in range(0, B * n, CHUNK):
        rs = slice(r0, min(r0 + CHUNK, B * n))
        Bd.check(stats[rs], *Bd.patch_stats_reference(a[rs]), "patch_stats")
        ref, e = Bd.gemm_reference(a[rs], w_perm, bias=bias, ln_sums=stats[rs], col_s=col_s)
        note("256x4_patch", Bd.check(y[rs], ref, e, f"patch_embed_tma rows {r0}+"))
    for i in (0, B - 1):
        y1, _ = launch(img[i:i + 1].contiguous())
        assert torch.equal(y1, y[i * n:(i + 1) * n])


# ---------------------------------------------------------------------------------------------------- patch kernels
def slab_batch(rows_per_image):
    """Images per launch for at least three patch-row slabs per CTA: the launchers run at most 8 CTAs per SM."""
    return cdiv(3 * 8 * sms(), rows_per_image) + 1


def check_patch_rows(name, got, x, gamma, beta, pd):
    for r0 in range(0, x.shape[0], CHUNK):
        rs = slice(r0, min(r0 + CHUNK, x.shape[0]))
        ref, bound = Bd.layernorm_reference(x[rs], gamma, beta)
        note(name, Bd.check(got[rs, :pd], ref, bound, f"{name} rows {r0}+"))
    assert (got[:, pd:] == 0).all()                    # K padding


@pytest.mark.parametrize("C,H,W,p,extra", [(3, 32, 96, 16, 0),     # 16 x 16 x 3 kernel
                                           (3, 28, 42, 14, 8),     # ViT-H patches: the register path
                                           (1, 14, 21, 7, 0)])     # odd patch_dim: the generic path
def test_patchify_ln_persistent(C, H, W, p, extra):
    gh, gw, pd = H // p, W // p, C * p * p
    B = slab_batch(gh)
    assert B * gh >= 3 * 8 * sms()
    note("patchify_ln slabs/CTA", (B * gh) // (8 * sms()))
    g = torch.Generator(device=DEV).manual_seed(pd)
    img = torch.randn(B, C, H, W, device=DEV, generator=g).bfloat16()
    gamma, beta = torch.randn(pd, device=DEV, generator=g), torch.randn(pd, device=DEV, generator=g)
    ldo = cdiv(pd, 64) * 64 + extra

    def launch(im):
        out = torch.full((im.shape[0] * gh * gw, ldo), BF16_SENT, device=DEV, dtype=torch.bfloat16)
        _lib.patchify_ln(im, gamma, beta, out, p, p)
        torch.cuda.synchronize()
        return out

    out = launch(img)
    check_patch_rows(f"patchify_ln p{p} C{C}", out, O.patchify(img, p, p).reshape(-1, pd), gamma, beta, pd)
    n = gh * gw
    for i in (B // 2, B - 1):
        assert torch.equal(launch(img[i:i + 1].contiguous()), out[i * n:(i + 1) * n])


@pytest.mark.parametrize("C,H,W,p", [(3, 32, 32, 4), (3, 64, 48, 16)])
def test_patchify_spt_ln_persistent(C, H, W, p):
    gh, gw, pd = H // p, W // p, 5 * C * p * p
    B = slab_batch(gh)
    note("patchify_spt_ln slabs/CTA", (B * gh) // (8 * sms()))
    g = torch.Generator(device=DEV).manual_seed(pd)
    img = torch.randn(B, C, H, W, device=DEV, generator=g).bfloat16()
    gamma, beta = torch.randn(pd, device=DEV, generator=g), torch.randn(pd, device=DEV, generator=g)
    ldo = cdiv(pd, 64) * 64

    def launch(im):
        out = torch.full((im.shape[0] * gh * gw, ldo), BF16_SENT, device=DEV, dtype=torch.bfloat16)
        _lib.patchify_spt_ln(im, gamma, beta, out, p)
        torch.cuda.synchronize()
        return out

    out = launch(img)
    xs = torch.cat([img] + [F.pad(img, s) for s in SPT_SHIFTS], dim=1)     # zero-filled shifts, exact in bf16
    check_patch_rows(f"patchify_spt_ln p{p}", out, O.patchify(xs, p, p).reshape(-1, pd), gamma, beta, pd)
    n = gh * gw
    for i in (0, B - 1):
        assert torch.equal(launch(img[i:i + 1].contiguous()), out[i * n:(i + 1) * n])


@pytest.mark.parametrize("p,sizes", [(16, [(32, 48), (64, 32), (16, 80), (48, 48)]),     # 16-wide kernel
                                     (14, [(28, 42), (56, 28), (14, 70), (42, 14)])])    # generic kernel
def test_patchify_varlen_ln_persistent(p, sizes):
    C = 3
    pd = C * p * p
    per_round = sum(h // p for h, _ in sizes)
    rounds = cdiv(3 * 8 * sms(), per_round) + 1
    g = torch.Generator(device=DEV).manual_seed(p)
    batches = [torch.randn(rounds, C, h, w, device=DEV, generator=g).bfloat16() for h, w in sizes]
    imgs = [bt[r] for r in range(rounds) for bt in batches]          # sizes interleaved
    ix = _lib.VarlenIndex(imgs, p, DEV)
    assert ix.total_rows >= 3 * 8 * sms()
    note(f"patchify_varlen_ln p{p} slabs/CTA", ix.total_rows // (8 * sms()))
    gamma = torch.randn(pd, device=DEV, generator=g)
    out = torch.full((ix.T, pd), BF16_SENT, device=DEV, dtype=torch.bfloat16)
    _lib.patchify_varlen_ln(imgs, gamma, out, ix.cu, p, index=ix)
    torch.cuda.synchronize()

    def rows_of(im):        # 'c (h p1) (w p2) -> (h w) (c p1 p2)'
        c, h, w = im.shape
        return im.view(c, h // p, p, w // p, p).permute(1, 3, 0, 2, 4).reshape(-1, pd)

    x = torch.cat([rows_of(im) for im in imgs])
    check_patch_rows(f"patchify_varlen_ln p{p}", out, x, gamma, None, pd)
    for i in (1, len(imgs) - 1):
        one = torch.full((ix.lengths[i], pd), BF16_SENT, device=DEV, dtype=torch.bfloat16)
        ix1 = _lib.VarlenIndex([imgs[i]], p, DEV)
        _lib.patchify_varlen_ln([imgs[i]], gamma, one, ix1.cu, p, index=ix1)
        torch.cuda.synchronize()
        s0 = sum(ix.lengths[:i])
        assert torch.equal(one, out[s0:s0 + ix.lengths[i]])


def test_report():
    """The worst |got - ref| / bound per kernel and the largest work per CTA of this run (printed with -s)."""
    for k in sorted(WORST):
        print(f"persistent: {k}: {WORST[k]:.4g}")
