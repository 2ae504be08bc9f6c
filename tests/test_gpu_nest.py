"""-m gpu: NesT on the H100.  b200vit_nest_level_entry against an fp64 reference with per-element bounds in the style
of oracle/row_bounds.py (the LayerNorm term of every window pixel, an exact max, one rounding for the position add)
for both pool settings, odd and even maps and D on the vector and scalar paths; its bf16 copy and row statistics
bit-identical to b200vit_rowstats_cast on the written stream; a NaN pixel reaching only its own pool windows and its
own image; nothing written outside the addressed rows; identical bits on repeat calls.  b200vit_nest_im2col bit-exact
against a torch gather, with zero padding columns.  Then the model: every case of tests/golden/nest_spec.py through the
comparison of test_gpu_family_parity.py in both LayerNorm modes (against the reference's logits and the module's own
bf16 graph), CUDA-graph replay, weight updates through `.data` + refresh_fused_weights and in place, and the eager
fall-backs."""
import sys

import pytest
import torch
import torch.nn.functional as F

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR
from oracle.bounds import U, check
from oracle.row_bounds import layernorm_e32, ln_depth
from vit_pytorch_b200 import _lib
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from nest_spec import FAMILY, NEST_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = dict(device=DEV, dtype=torch.float32)
NAN = float("nan")
PAD = 8          # poisoned rows before and after the addressed ones (keeps every row offset 16-byte aligned)


def block_rows(B, H, W, nb):
    """Per map-order row (b*H + y)*W + x, its row in the block-major stream of nb x nb blocks."""
    sh, sw = H // nb, W // nb
    b, y, x = torch.meshgrid(torch.arange(B, device=DEV), torch.arange(H, device=DEV), torch.arange(W, device=DEV),
                             indexing="ij")
    return (((b * nb + y // sh) * nb + x // sw) * (sh * sw) + (y % sh) * sw + x % sw).reshape(-1)


def poisoned(rows, cols, dtype):
    return torch.full((rows + 2 * PAD, cols), NAN, device=DEV, dtype=dtype)


# ========================================================================================= level entry
def level_entry_reference(y, g, b, pos, B, H, W, k, s, p, nb, eps=1e-5):
    """(ref, bound) fp64 [B*oh*ow, D] in block-major rows: per window the max of the window pixels' LayerNorm values
    (an exact max, so off by at most the largest LayerNorm bound E32 in the window), then + pos (one fp32 rounding)."""
    D = y.shape[1]
    ln, e32 = layernorm_e32(y, g, b, eps, ln_depth(D))

    def pool(t, fill):
        t = t.view(B, H, W, D).permute(0, 3, 1, 2)
        return F.pad(t, (p, p, p, p), value=fill).unfold(2, k, s).unfold(3, k, s).amax(dim=(-1, -2))
    m, e = pool(ln, float("-inf")), pool(e32, 0.0)
    oh, ow = m.shape[2], m.shape[3]
    sh, sw = oh // nb, ow // nb
    r, q = torch.meshgrid(torch.arange(oh, device=DEV), torch.arange(ow, device=DEV), indexing="ij")
    ref = m + pos.double()[(r % sh) * sw + q % sw]
    bound = e + U * (ref.abs() + e)
    rows = block_rows(B, oh, ow, nb)
    out_r = torch.empty(B * oh * ow, D, dtype=torch.float64, device=DEV)
    out_b = torch.empty_like(out_r)
    out_r[rows], out_b[rows] = ref.permute(0, 2, 3, 1).reshape(-1, D), bound.permute(0, 2, 3, 1).reshape(-1, D)
    return out_r, out_b


def run_level_entry(y, g, b, pos, B, H, W, k, s, p, nb, fold):
    """The kernel writing between NaN rows of x (and xb, stats); asserts the padding kept.  Returns (x, xb, stats)."""
    D = y.shape[1]
    rows = B * _lib.conv_out_size(H, k, s, p) * _lib.conv_out_size(W, k, s, p)
    xbig = poisoned(rows, D, torch.float32)
    bbig = poisoned(rows, D, torch.bfloat16) if fold else None
    sbig = poisoned(rows, 2, torch.float32) if fold else None
    cut = lambda t: None if t is None else t[PAD:PAD + rows]        # noqa: E731
    _lib.nest_level_entry(y, g, b, pos, cut(xbig), B, H, W, k, s, p, nb, xb=cut(bbig), stats=cut(sbig))
    torch.cuda.synchronize()
    for t in (xbig, bbig, sbig):
        if t is not None:
            assert torch.isnan(t[:PAD]).all() and torch.isnan(t[PAD + rows:]).all()
    return tuple(None if t is None else t.clone() for t in (cut(xbig), cut(bbig), cut(sbig)))


def entry_inputs(B, H, W, D, seed, n_pos):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    y = torch.randn(B * H * W, D, device=DEV, generator=gen) * 2 + 0.5
    g = 1 + 0.2 * torch.randn(D, device=DEV, generator=gen)
    b = 0.1 * torch.randn(D, device=DEV, generator=gen)
    pos = torch.randn(n_pos, device=DEV, generator=gen)
    return y, g, b, pos


ENTRY_SHAPES = [  # B, H, W, (k, s, p), nb: the patch embedding's entry, then Aggregate's on even and odd maps
    (2, 56, 56, (1, 1, 0), 4), (3, 7, 7, (1, 1, 0), 1), (1, 12, 20, (1, 1, 0), 2),
    (2, 56, 56, (3, 2, 1), 2), (2, 28, 14, (3, 2, 1), 1), (2, 7, 7, (3, 2, 1), 1), (1, 13, 9, (3, 2, 1), 1),
    (2, 16, 16, (2, 2, 0), 2),
]


@pytest.mark.parametrize("fold", [True, False])
@pytest.mark.parametrize("D", [96, 384, 36, 30])      # float4 path (D % 4 == 0) and scalar path
@pytest.mark.parametrize("B,H,W,pool,nb", ENTRY_SHAPES)
def test_level_entry_within_bounds_with_rowstats_bits_and_repeatable(B, H, W, pool, nb, D, fold):
    k, s, p = pool
    oh, ow = _lib.conv_out_size(H, k, s, p), _lib.conv_out_size(W, k, s, p)
    n_pos = (oh // nb) * (ow // nb) + 3                      # a longer table: only its prefix is read
    y, g, b, pos = entry_inputs(B, H, W, D, 7 * H + D + k, n_pos)
    x, xb, st = run_level_entry(y, g, b, pos, B, H, W, k, s, p, nb, fold)
    ref, bound = level_entry_reference(y, g, b, pos, B, H, W, k, s, p, nb)
    check(x, ref, bound, f"level entry {B}x{H}x{W} D={D} pool={pool} nb={nb}")
    if fold:
        assert torch.equal(xb, x.bfloat16())
        xb2 = torch.empty_like(xb)
        st2 = torch.empty(x.shape[0], 1, 2, **F32)
        _lib.rowstats_cast(x, xb2, st2)
        torch.cuda.synchronize()
        assert torch.equal(xb2, xb) and torch.equal(st2.view(-1, 2), st)
    again = run_level_entry(y, g, b, pos, B, H, W, k, s, p, nb, fold)
    for t0, t1 in zip((x, xb, st), again):
        assert t0 is None or torch.equal(t0, t1)


@pytest.mark.parametrize("pool,nb", [((1, 1, 0), 2), ((3, 2, 1), 1)])
def test_level_entry_nan_pixel_reaches_only_its_pool_windows_and_image(pool, nb):
    B, H, W, D = 2, 8, 8, 64
    k, s, p = pool
    y, g, b, pos = entry_inputs(B, H, W, D, 3, 64)
    clean = run_level_entry(y, g, b, pos, B, H, W, k, s, p, nb, True)
    yy, xx, c = 3, 4, 17
    y[(0 * H + yy) * W + xx, c] = NAN
    x, xb, st = run_level_entry(y, g, b, pos, B, H, W, k, s, p, nb, True)
    oh, ow = _lib.conv_out_size(H, k, s, p), _lib.conv_out_size(W, k, s, p)
    r, q = torch.meshgrid(torch.arange(oh, device=DEV), torch.arange(ow, device=DEV), indexing="ij")
    hit = ((r * s - p <= yy) & (yy < r * s - p + k) & (q * s - p <= xx) & (xx < q * s - p + k)).reshape(-1)
    rows = block_rows(B, oh, ow, nb).view(B, -1)
    assert hit.any()
    assert torch.isnan(x[rows[0][hit]]).all() and torch.isnan(st[rows[0][hit]]).all()
    assert torch.equal(x[rows[0][~hit]], clean[0][rows[0][~hit]])
    assert torch.equal(x[rows[1]], clean[0][rows[1]]) and torch.equal(st[rows[1]], clean[2][rows[1]])


# ========================================================================================= im2col
@pytest.mark.parametrize("B,H,W,D,nb,extra", [(2, 56, 56, 96, 4, 0), (1, 28, 14, 192, 2, 8), (3, 7, 7, 32, 1, 16),
                                              (2, 8, 8, 8, 4, 24)])
def test_im2col_bit_exact_against_a_torch_gather(B, H, W, D, nb, extra):
    gen = torch.Generator(device=DEV).manual_seed(H + D)
    x = torch.randn(B * H * W, D, device=DEV, generator=gen)
    M, ldo = B * H * W, 9 * D + extra
    big = torch.full((M + 2 * PAD, ldo), NAN, device=DEV, dtype=torch.bfloat16)
    _lib.nest_im2col(x, big[PAD:PAD + M], B, H, W, nb)
    torch.cuda.synchronize()
    assert torch.isnan(big[:PAD]).all() and torch.isnan(big[PAD + M:]).all()
    m = torch.zeros(B, H + 2, W + 2, D, device=DEV)
    m[:, 1:-1, 1:-1] = x[block_rows(B, H, W, nb)].view(B, H, W, D)
    want = torch.cat([m[:, i:i + H, j:j + W] for i in range(3) for j in range(3)], -1).reshape(M, 9 * D)
    got = big[PAD:PAD + M]
    assert torch.equal(got[:, :9 * D], want.bfloat16())
    assert (got[:, 9 * D:] == 0).all()


# ========================================================================================= the model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(NEST_CASES))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec against the reference's stored logits and the module's own bf16 graph with the shared
    comparison (fused_reason is None, launches counted, tol 3e-2), in both LayerNorm modes."""
    monkeypatch.setitem(P.FAMILIES, "nest", FAMILY)
    monkeypatch.setitem(P.GPU, "nest", dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens("nest", name, ln_mode, monkeypatch)


def small_model(seed=0, name="int_repeats_mlp2"):
    spec = dict(NEST_CASES[name], seed=seed)
    return FAMILY.build(spec).to(DEV, torch.bfloat16), FAMILY.input(spec).to(DEV)


def test_graphed_forward_replays_the_eager_launches_bit_for_bit():
    m, x = small_model()
    with torch.inference_mode():
        want = m(x).clone()
    fwd = GraphedForward(m, x)
    got = fwd(x)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_weight_updates_change_the_output():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
        m.layers[1][0].pos_emb.data.mul_(-1.5)            # through .data: the version counter does not move
        m.refresh_fused_weights()
        after = m(x).clone()
        want = m.forward_eager(x)
    assert not torch.equal(after, before)
    assert (after.float() - want.float()).abs().max().item() < 3e-2
    with torch.no_grad():
        m.layers[0][1][1].g.mul_(0.5)                     # in place: the version counter moves
        m.layers[0][0].layers[0][1].net[1].weight.mul_(-1.0)
    with torch.inference_mode():
        again = m(x).clone()
        want = m.forward_eager(x)
    assert not torch.equal(again, after)
    assert (again.float() - want.float()).abs().max().item() < 3e-2


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
        h = m.layers[1][0].layers[0][0].to_qkv.register_forward_hook(lambda mod, i, o: seen.append(tuple(o.shape)))
        assert "hooks" in m.fused_reason(x)
        got = m(x)
        assert seen == [(2 * 4, 3 * 64, 4, 4)]          # level 2: 8 x 8 map in 2 x 2 blocks of 4 x 4
        assert (got.float() - m.forward_eager(x).float()).abs().max().item() < 5e-2
        h.remove()
        assert m.fused_reason(x) is None
        m.train()
        assert "training" in m.fused_reason(x)
        m.eval()
        assert m.fused_reason(x.float()) is not None
        assert "seq_len" in m.fused_reason(torch.zeros(1, 3, 128, 128, device=DEV, dtype=torch.bfloat16))
