"""-m gpu: the row kernels of rowops.cu, called through the C ABI, against the fp64 references of oracle/row_bounds.py
with a bound on every element, at the shapes where their paths split (float4 / scalar, idle lanes, partial warps,
head counts on both sides of the unroll switch).  Also bit-level properties: the statistics every writer hands to the
LN-folded GEMMs are the bits rowstats_cast writes for the same fp32 rows; repeat calls give identical bits; a NaN stays
in its own row, image or head; padding columns and rows past the outputs are never written."""
import pytest
import torch

from oracle import row_bounds as RB
from vit_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")


def report(what, r):
    print(f"excess {what}: {r:.3f}")
    return r


def nan_f32(*shape):
    return torch.full(shape, NAN, device=DEV)


def nan_bf16(*shape):
    return torch.full(shape, NAN, device=DEV, dtype=torch.bfloat16)


def same_bits(a, b):
    """bit equality (NaN == NaN)."""
    if a.dtype == torch.bfloat16:
        return torch.equal(a.view(torch.int16), b.view(torch.int16))
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def rowstats_of(x):
    """(bf16 copy, statistics) rowstats_cast writes for the fp32 rows x."""
    xb = torch.empty(x.shape, device=DEV, dtype=torch.bfloat16)
    st = torch.empty(x.shape[0], 2, device=DEV)
    _lib.rowstats_cast(x.contiguous(), xb, st)
    return xb, st


# ---------------------------------------------------------------------------------------------------- row LayerNorm
def run_layernorm(x, D, g, b, M, ldo, row_index=None, f32=True, bf16=True, pad_rows=3):
    of = nan_f32(M + pad_rows, ldo) if f32 else None
    ob = nan_bf16(M + pad_rows, ldo) if bf16 else None
    _lib.layernorm(x[:, :D], g, b, out_f32=None if of is None else of[:M],
                   out_bf16=None if ob is None else ob[:M], row_index=row_index)
    return of, ob


@pytest.mark.parametrize("D", [4, 12, 50, 64, 192, 200, 768, 1280, 4096])
def test_layernorm(D):
    torch.manual_seed(D)
    M = 77                                                        # not a multiple of the 8 rows of a CTA
    ldx = D + (4 if D % 4 == 0 else 3)
    ldo = D + (8 if D % 4 == 0 else 5)
    x = torch.randn(M, ldx, device=DEV) * 3 + 1
    g, b = torch.randn(D, device=DEV), torch.randn(D, device=DEV)
    of, ob = run_layernorm(x, D, g, b, M, ldo)
    ref, e = RB.layernorm_reference(x, g, b)
    report(f"layernorm fp32 D={D}", RB.check(of[:M, :D], ref, e, f"layernorm fp32 D={D}"))
    report(f"layernorm bf16 D={D}", RB.check(ob[:M, :D], *RB.layernorm_reference(x, g, b, bf16_out=True), "bf16"))
    assert same_bits(ob[:M, :D], of[:M, :D].bfloat16())
    assert torch.isnan(of[:M, D:]).all() and torch.isnan(of[M:]).all()          # padding never written
    assert torch.isnan(ob[:M, D:].float()).all() and torch.isnan(ob[M:].float()).all()
    of2, ob2 = run_layernorm(x, D, g, b, M, ldo)
    assert same_bits(of2, of) and same_bits(ob2, ob)                            # repeat calls: the same bits
    xn = x.clone()
    xn[5, D // 2] = NAN
    of3, _ = run_layernorm(xn, D, g, b, M, ldo)
    assert torch.isnan(of3[5, :D]).all()
    keep = torch.ones(M + 3, dtype=torch.bool, device=DEV)
    keep[5] = False
    assert same_bits(of3[keep], of[keep])                                       # the NaN stays in its row


def test_layernorm_variants():
    """ldo % 4 != 0 with D % 4 == 0 (scalar output path), a row gather, no beta, fp32-only and bf16-only output."""
    torch.manual_seed(1)
    D, M = 64, 45
    x = torch.randn(300, D, device=DEV) * 2 - 1
    g, b = torch.randn(D, device=DEV), torch.randn(D, device=DEV)
    of, ob = run_layernorm(x[:M], D, g, b, M, 66)
    RB.check(of[:M, :D], *RB.layernorm_reference(x[:M], g, b), "ldo 66 fp32")
    RB.check(ob[:M, :D], *RB.layernorm_reference(x[:M], g, b, bf16_out=True), "ldo 66 bf16")
    assert torch.isnan(of[:M, D:]).all() and torch.isnan(ob[:M, D:].float()).all()
    rows = torch.randperm(300, device=DEV)[:M].to(torch.int32)
    for beta in (b, None):
        of, _ = run_layernorm(x, D, g, beta, M, D, row_index=rows, bf16=False)
        r = RB.check(of[:M], *RB.layernorm_reference(x, g, beta, row_index=rows), "gather fp32")
        _, ob = run_layernorm(x, D, g, beta, M, D, row_index=rows, f32=False)
        RB.check(ob[:M], *RB.layernorm_reference(x, g, beta, row_index=rows, bf16_out=True), "gather bf16")
        assert torch.isnan(ob[M:].float()).all()
        report(f"layernorm gather beta={beta is not None}", r)


# ---------------------------------------------------------------------------------------------------- token assembly
# (D, groups, n, ncls, ntail, LN, POS, pos_period, cls_pos): every row kind at D % 4 == 0 and != 0
EMBED = {
    "vit": (768, 5, 49, 1, 0, True, True, 1, True),
    "vit_odd_d": (202, 3, 21, 1, 0, True, True, 1, True),
    "two_cls": (192, 3, 16, 2, 0, True, True, 1, True),
    "registers": (384, 3, 16, 0, 4, True, True, 1, True),
    "registers_odd_d": (198, 3, 16, 1, 3, True, True, 1, True),
    "no_ln": (256, 4, 25, 1, 0, False, True, 1, True),
    "no_ln_odd_d": (90, 3, 25, 1, 0, False, True, 1, True),
    "no_pos": (192, 3, 16, 1, 0, True, False, 1, True),
    "no_ln_no_pos_odd_d": (66, 3, 9, 0, 0, False, False, 1, True),
    "grouped_cls_pos": (192, 8, 16, 1, 0, True, True, 4, True),
    "grouped_no_cls_pos": (192, 8, 16, 1, 0, True, True, 4, False),
    "grouped_odd_d": (150, 6, 9, 1, 0, True, True, 3, False),
}


def embed_inputs(case, seed=0):
    D, groups, n, ncls, ntail, ln, has_pos, period, cls_pos = EMBED[case]
    g = torch.Generator(device=DEV).manual_seed(seed)
    stride = n + (ncls if cls_pos else 0)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    return dict(y=rn(groups * n, D) * 2 + 0.5, gamma=rn(D) if ln else None, beta=rn(D) if ln else None,
                cls=rn(ncls, D) if ncls else None, pos=rn(period * stride + 2, D) if has_pos else None,
                tail=rn(ntail, D) if ntail else None, groups=groups, n=n, ncls=ncls, pos_period=period,
                pos_stride=stride if period > 1 else 0, cls_pos=cls_pos)


def run_embed(a, pad_rows=5):
    D = a["y"].shape[1]
    N = a["ncls"] + a["n"] + (0 if a["tail"] is None else a["tail"].shape[0])
    R = a["groups"] * N
    x, xb, st = nan_f32(R + pad_rows, D), nan_bf16(R + pad_rows, D), nan_f32(R + pad_rows, 2)
    if a["pos_period"] > 1 or not a["cls_pos"]:
        _lib.embed_tokens_grouped(a["y"], a["gamma"], a["beta"], a["cls"], a["pos"], x[:R], a["groups"], a["n"],
                                  a["ncls"], a["pos_period"], a["pos_stride"], a["cls_pos"], xb=xb[:R], stats=st[:R])
    else:
        _lib.embed_tokens(a["y"], a["gamma"], a["beta"], a["cls"], a["pos"], x[:R], a["groups"], a["n"], a["ncls"],
                          xb=xb[:R], stats=st[:R], tail=a["tail"])
    return x, xb, st, R


@pytest.mark.parametrize("case", list(EMBED))
def test_embed_tokens(case):
    a = embed_inputs(case)
    x, xb, st, R = run_embed(a)
    ref, e = RB.embed_tokens_reference(a["y"], a["gamma"], a["beta"], a["cls"], a["pos"], a["groups"], a["n"],
                                       a["ncls"], tail=a["tail"], pos_period=a["pos_period"],
                                       pos_stride=a["pos_stride"], cls_pos=a["cls_pos"])
    report(f"embed_tokens {case}", RB.check(x[:R], ref, e, case))
    report(f"embed_tokens stats {case}", RB.check(st[:R], *RB.row_stats_reference(xb[:R]), case + " stats"))
    assert torch.isnan(x[R:]).all() and torch.isnan(xb[R:].float()).all() and torch.isnan(st[R:]).all()
    x2, xb2, st2, _ = run_embed(a)
    assert same_bits(x2, x) and same_bits(xb2, xb) and same_bits(st2, st)
    # a NaN in one image's patches stays in that image
    if a["groups"] > 1:
        N = R // a["groups"]
        yn = a["y"].clone()
        yn[a["n"] + 1] = NAN                                     # patch 1 of image 1
        xn, _, stn, _ = run_embed(dict(a, y=yn))
        other = torch.ones(R, dtype=torch.bool, device=DEV)
        other[N:2 * N] = False
        assert same_bits(xn[:R][other], x[:R][other]) and same_bits(stn[:R][other], st[:R][other])
        assert torch.isnan(xn[N + a["ncls"] + 1]).all()


@pytest.mark.parametrize("case", list(EMBED))
def test_embed_tokens_statistics_are_rowstats_cast_bits(case):
    """Every row kind hands the first LN-folded GEMM the bf16 copy and statistics rowstats_cast writes for the same
    fp32 rows, so a model's first layer starts from the same bits whichever way its tokens arrive."""
    x, xb, st, R = run_embed(embed_inputs(case, seed=1))
    xb_ref, st_ref = rowstats_of(x[:R])
    assert same_bits(xb[:R], xb_ref) and same_bits(xb[:R], x[:R].bfloat16())
    bad = (st[:R].view(torch.int32) != st_ref.view(torch.int32)).any(1).nonzero().flatten().tolist()
    assert not bad, f"{len(bad)} of {R} rows differ from rowstats_cast, first {bad[:8]}"


# ---------------------------------------------------------------------------------------------------- embed_varlen
def varlen_case(seed=0):
    p, D = 4, 192
    # 11 images (bisection over more than 8), one-patch images, grids of every shape; T = 51 (not a multiple of 8)
    dims = [(8, 12), (4, 4), (12, 8), (4, 20), (4, 4), (16, 16), (8, 4), (4, 8), (20, 4), (8, 8), (4, 12)]
    imgs = [torch.zeros(1, h, w, device=DEV, dtype=torch.bfloat16) for h, w in dims]
    index = _lib.VarlenIndex(imgs, p, DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    y = torch.randn(index.T, D, generator=g, device=DEV) * 2 + 0.5
    gm = torch.randn(D, generator=g, device=DEV)
    ph, pw = torch.randn(6, D, generator=g, device=DEV), torch.randn(6, D, generator=g, device=DEV)
    return dict(y=y, gamma=gm, pos_h=ph, pos_w=pw, index=index, dims=dims, p=p, imgs=imgs)


def run_varlen(c, y=None):
    y = c["y"] if y is None else y
    T, D = y.shape
    x, xb, st = nan_f32(T + 3, D), nan_bf16(T + 3, D), nan_f32(T + 3, 2)
    _lib.embed_varlen(y, c["gamma"], c["pos_h"], c["pos_w"], c["index"], x[:T], c["p"], xb=xb[:T], stats=st[:T])
    return x, xb, st


def test_embed_varlen():
    c = varlen_case()
    T = c["index"].T
    assert T % 8 != 0 and c["index"].S > 8 and 1 in c["index"].lengths
    x, xb, st = run_varlen(c)
    ref, e = RB.embed_varlen_reference(c["y"], c["gamma"], c["pos_h"], c["pos_w"], c["index"].lengths, c["dims"],
                                       c["p"])
    report("embed_varlen", RB.check(x[:T], ref, e, "embed_varlen"))
    report("embed_varlen stats", RB.check(st[:T], *RB.row_stats_reference(xb[:T]), "stats"))
    assert torch.isnan(x[T:]).all() and torch.isnan(xb[T:].float()).all() and torch.isnan(st[T:]).all()
    xb_ref, st_ref = rowstats_of(x[:T])
    assert same_bits(xb[:T], xb_ref) and same_bits(st[:T], st_ref)
    x2, xb2, st2 = run_varlen(c)
    assert same_bits(x2, x) and same_bits(xb2, xb) and same_bits(st2, st)
    cu = [0]
    for L in c["index"].lengths:
        cu.append(cu[-1] + L)
    yn = c["y"].clone()
    yn[cu[5] + 3] = NAN                                           # one token of image 5
    xn, _, _ = run_varlen(c, yn)
    other = torch.ones(T, dtype=torch.bool, device=DEV)
    other[cu[5]:cu[6]] = False
    assert same_bits(xn[:T][other], x[:T][other])


# ---------------------------------------------------------------------------------------------------- head norms
def layernorm_heads(buf, gamma, nheads, dh, eps=1e-5):
    rc = _lib.lib().b200vit_layernorm_heads(buf.data_ptr(), buf.stride(0), gamma.data_ptr(), buf.shape[0], nheads, dh,
                                            float(eps), _lib._stream())
    assert rc == 0, _lib.lib().b200vit_last_error()


def head_buffer(T, H, dh, seed):
    """kv-like buffer [T, 2 H dh + 8] (the k half is normalised; the v half and the 8 padding columns must not
    change) with an all-zero head, a constant head and ill-conditioned heads (|mean| / std of several hundred)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    I = H * dh
    buf = torch.randn(T, 2 * I + 8, generator=g, device=DEV).bfloat16()
    buf[:, 2 * I:] = NAN
    k = buf[:, :I].view(T, H, dh)
    k[3, H - 1] = 0
    k[4, 0] = 0.75
    k[7:40:3] = (torch.randn(k[7:40:3].shape, generator=g, device=DEV) * 0.5 + 300).bfloat16()
    return buf, torch.randn(H, dh, generator=g, device=DEV)


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("H", [1, 3, 8, 9, 17, 33])
@pytest.mark.parametrize("norm", ["rms", "ln"])
def test_head_norms(norm, H, dh):
    """rmsnorm_heads / layernorm_heads on the k half of a kv buffer: head counts on both sides of the U = 2 / 4 switch
    (> 8) and not multiples of the heads per step."""
    T = 301
    I = H * dh
    buf0, g = head_buffer(T, H, dh, H * dh)
    x = buf0[:, :I].view(T, H, dh)
    gf = g.reshape(-1).contiguous()

    def run(b):
        out = b.clone()
        if norm == "rms":
            _lib.rmsnorm_heads(out, gf, H, dh)
        else:
            layernorm_heads(out, gf, H, dh)
        return out

    out = run(buf0)
    ref, e = (RB.rmsnorm_heads_reference(x, g) if norm == "rms" else RB.layernorm_heads_reference(x, g))
    report(f"{norm}_heads dh={dh} H={H}", RB.check(out[:, :I].view(T, H, dh), ref, e, f"{norm} dh={dh} H={H}"))
    assert same_bits(out[:, I:], buf0[:, I:])                                  # v and padding untouched
    if norm == "rms":
        assert (out[3, (H - 1) * dh:I] == 0).all()                             # an all-zero head gives exactly 0
    assert same_bits(run(buf0), out)
    bn = buf0.clone()
    bn[10, (H // 2) * dh + 1] = NAN
    outn = run(bn)
    assert torch.isnan(outn[10, (H // 2) * dh:(H // 2 + 1) * dh].float()).all()
    keep = torch.ones_like(out, dtype=torch.bool)
    keep[10, (H // 2) * dh:(H // 2 + 1) * dh] = False
    assert same_bits(outn[keep], out[keep])                                    # the NaN stays in its head


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_qk_rmsnorm_leaves_v_untouched(dh):
    torch.manual_seed(dh)
    T, H = 203, 5
    I = H * dh
    qkv = torch.randn(T, 3 * I, device=DEV).bfloat16()
    gqk = torch.randn(2, H, dh, device=DEV)
    out = qkv.clone()
    _lib.qk_rmsnorm(out, gqk.reshape(-1).contiguous(), H, dh)
    for s in (0, 1):
        x = qkv[:, s * I:(s + 1) * I].view(T, H, dh)
        got = out[:, s * I:(s + 1) * I].view(T, H, dh)
        report(f"qk_rmsnorm dh={dh} {'qk'[s]}", RB.check(got, *RB.rmsnorm_heads_reference(x, gqk[s]), "qk"))
    assert same_bits(out[:, 2 * I:], qkv[:, 2 * I:])


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("headln", [False, True])
def test_gemm_headnorm_norm_half(dh, headln):
    """QKV GEMM + per-head norm of the q and k heads, against the reference norm of the kernel's own plain-GEMM bf16
    output (the same GEMM instance: its bits are deterministic)."""
    torch.manual_seed(dh + headln)
    M, H, K = 700, 3, 256
    I = H * dh
    a = torch.randn(M, K, device=DEV).bfloat16()
    w = (torch.randn(3 * I, K, device=DEV) / K ** 0.5).bfloat16()
    g = torch.randn(2 * H, dh, device=DEV)
    plain = torch.empty(M, 3 * I, device=DEV, dtype=torch.bfloat16)
    _lib.gemm(a, w, out_bf16=plain)
    got = torch.empty_like(plain)
    _lib.gemm_headnorm(a, w, out_bf16=got, head_gamma=g.reshape(-1).contiguous(), norm_heads=2 * H, dh=dh,
                       head_layernorm_eps=1e-5 if headln else None)
    x = plain[:, :2 * I].view(M, 2 * H, dh)
    ref, e = RB.layernorm_heads_reference(x, g) if headln else RB.rmsnorm_heads_reference(x, g)
    report(f"gemm_headnorm dh={dh} ln={headln}", RB.check(got[:, :2 * I].view(M, 2 * H, dh), ref, e, "headnorm"))
    assert same_bits(got[:, 2 * I:], plain[:, 2 * I:])                         # v columns untouched

