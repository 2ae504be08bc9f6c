"""-m gpu: Twins-SVT on the H100.  Its four kernels (window attention in csrc/attention_tile64.cu, the other three in
csrc/twins.cu) against fp64 references with per-element bounds
(the attention kernels through oracle/attention_bounds.py, the patch merging through oracle.bounds.layernorm_reference,
the positional encoding with a bound built like test_gpu_pit.pool_reference), what they write and which rows they
read; then the model: every case of tests/golden/twins_svt_spec.py through the comparison of
test_gpu_family_parity.py, CUDA-graph replay, weight refresh and the eager fall-backs."""
import sys

import pytest
import torch

import test_gpu_family_parity as P
from conftest import GOLDEN_DIR
from oracle.bounds import check, layernorm_reference
from oracle.grid_attention_bounds import kv_reference, peg_reference, window_reference, window_rows
from vit_pytorch_b200 import _lib

sys.path.insert(0, GOLDEN_DIR)
from twins_svt_spec import FAMILY, TWINS_CASES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
HEAD_WIDTHS = [32, 64, 80, 128]


def rows_equal(a, b):
    return ((a == b) | (torch.isnan(a) & torch.isnan(b))).all(1)


# ================================================================================================ attention_window
def run_window(qkv, B, gh, gw, p, H, dh, pad_rows=3):
    """attention_window into a view of a NaN-poisoned buffer longer than the output: (whole buffer, output view)."""
    big = torch.full((B * gh * gw + pad_rows, H * dh), NAN, device=DEV, dtype=torch.bfloat16)
    out = big[:B * gh * gw]
    _lib.attention_window(qkv, out, B, gh, gw, p, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    return big, out


@pytest.mark.parametrize("p,gh,gw", [(1, 3, 5), (2, 4, 4), (2, 6, 10), (3, 9, 6), (4, 8, 8), (4, 4, 12), (5, 10, 5),
                                     (6, 6, 12), (7, 14, 7), (7, 7, 7), (8, 8, 16), (8, 16, 8)])
@pytest.mark.parametrize("dh", HEAD_WIDTHS)
def test_attention_window_within_bounds(dh, p, gh, gw):
    B, H = 3, 2
    g = torch.Generator(device=DEV).manual_seed(dh * 100 + p * 10 + gw)
    qkv = torch.randn(B * gh * gw, 3 * H * dh, device=DEV, generator=g).bfloat16()
    big, out = run_window(qkv, B, gh, gw, p, H, dh)
    assert torch.isnan(big[B * gh * gw:].float()).all(), "rows past the output were written"
    ref, bound = window_reference(qkv, B, gh, gw, p, H, dh)
    check(out, ref, bound, f"attention_window dh={dh} p={p} {gh}x{gw}")


@pytest.mark.parametrize("p,gh,gw", [(1, 3, 5), (2, 6, 10), (4, 8, 8), (7, 14, 7), (8, 8, 16)])
@pytest.mark.parametrize("dh", [32, 64])
def test_attention_window_isolation(dh, p, gh, gw):
    """A NaN image leaves the other images bit-identical; so does a NaN window where a window has a tile of its own,
    and a window of huge finite values where windows share a tile; NaN past the view passed in is never read."""
    B, H = 3, 2
    I, n = H * dh, gh * gw
    g = torch.Generator(device=DEV).manual_seed(dh + p)
    qkv = torch.randn(B * n, 3 * I, device=DEV, generator=g).bfloat16()
    clean = run_window(qkv, B, gh, gw, p, H, dh)[1]
    assert torch.isfinite(clean.float()).all()
    image = torch.arange(B * n, device=DEV) // n
    for b in range(B):
        bad = qkv.clone()
        bad[b * n:(b + 1) * n] = NAN
        assert rows_equal(run_window(bad, B, gh, gw, p, H, dh)[1], clean)[image != b].all(), f"NaN image {b}"
    rows = window_rows(B, gh, gw, p, p, DEV)
    for wi in (0, rows.shape[0] // 2, rows.shape[0] - 1):
        bad = qkv.clone()
        bad[rows[wi]] = NAN if p * p > 32 else 3.0e38
        keep = torch.ones(B * n, dtype=torch.bool, device=DEV)
        keep[rows[wi]] = False
        assert rows_equal(run_window(bad, B, gh, gw, p, H, dh)[1], clean)[keep].all(), f"poisoned window {wi}"
    buf = torch.full((B * n + 70, 3 * I), NAN, device=DEV, dtype=torch.bfloat16)
    buf[:B * n] = qkv
    assert torch.equal(run_window(buf[:B * n], B, gh, gw, p, H, dh)[1], clean)


# ==================================================================================================== attention_kv
def run_kv(q, kv, B, Nq, Nk, H, dh, pad_rows=3):
    big = torch.full((B * Nq + pad_rows, H * dh), NAN, device=DEV, dtype=torch.bfloat16)
    out = big[:B * Nq]
    _lib.attention_kv(q, kv, out, B, Nq, Nk, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    return big, out


def kv_inputs(B, Nq, Nk, H, dh, seed, strided=True):
    """q and kv as views of wider buffers (their own row strides) when `strided`."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    I = H * dh
    qb = torch.randn(B * Nq, 3 * I if strided else I, device=DEV, generator=g).bfloat16()
    kb = torch.randn(B * Nk, 2 * I + (8 if strided else 0), device=DEV, generator=g).bfloat16()
    return qb[:, :I], kb[:, :2 * I]


@pytest.mark.parametrize("Nk", [1, 4, 63, 64, 65, 784, 1024])
@pytest.mark.parametrize("Nq", [1, 200, 300])
@pytest.mark.parametrize("dh", HEAD_WIDTHS)
def test_attention_kv_within_bounds(dh, Nq, Nk):
    B, H = 2, 2
    q, kv = kv_inputs(B, Nq, Nk, H, dh, dh * 1000 + Nq + Nk)
    big, out = run_kv(q, kv, B, Nq, Nk, H, dh)
    assert torch.isnan(big[B * Nq:].float()).all(), "rows past the output were written"
    ref, bound = kv_reference(q, kv, B, Nq, Nk, H, dh)
    check(out, ref, bound, f"attention_kv dh={dh} Nq={Nq} Nk={Nk}")


def test_attention_kv_one_key_returns_the_value_row():
    B, Nq, H, dh = 3, 130, 2, 64
    q, kv = kv_inputs(B, Nq, 1, H, dh, 7)
    out = run_kv(q, kv, B, Nq, 1, H, dh)[1]
    assert torch.equal(out.view(B, Nq, H * dh), kv[:, H * dh:].reshape(B, 1, H * dh).expand(B, Nq, H * dh))


@pytest.mark.parametrize("Nq,Nk", [(130, 1), (300, 65), (257, 784)])
@pytest.mark.parametrize("dh", [64, 128])
def test_attention_kv_isolation(dh, Nq, Nk):
    """A NaN image (queries, keys and values) leaves the other images bit-identical, and NaN rows past the views
    passed in are never read."""
    B, H = 3, 2
    I = H * dh
    q, kv = kv_inputs(B, Nq, Nk, H, dh, dh + Nq, strided=False)
    clean = run_kv(q, kv, B, Nq, Nk, H, dh)[1]
    assert torch.isfinite(clean.float()).all()
    image = torch.arange(B * Nq, device=DEV) // Nq
    for b in range(B):
        qb, kb = q.clone(), kv.clone()
        qb[b * Nq:(b + 1) * Nq] = NAN
        kb[b * Nk:(b + 1) * Nk] = NAN
        assert rows_equal(run_kv(qb, kb, B, Nq, Nk, H, dh)[1], clean)[image != b].all(), f"NaN image {b}"
    qbuf = torch.full((B * Nq + 130, I), NAN, device=DEV, dtype=torch.bfloat16)
    kbuf = torch.full((B * Nk + 70, 2 * I), NAN, device=DEV, dtype=torch.bfloat16)
    qbuf[:B * Nq], kbuf[:B * Nk] = q, kv
    assert torch.equal(run_kv(qbuf[:B * Nq], kbuf[:B * Nk], B, Nq, Nk, H, dh)[1], clean)


# ============================================================================================ merge_patches_ln, peg
@pytest.mark.parametrize("p,gh,gw,C", [(1, 7, 7, 40), (2, 4, 6, 16), (2, 28, 28, 64), (3, 6, 9, 8), (4, 8, 4, 24)])
def test_merge_patches_ln_within_bounds(p, gh, gw, C):
    B, K = 2, p * p * C
    ldo = (K + 63) // 64 * 64 + 8
    g = torch.Generator(device=DEV).manual_seed(p * 100 + C)
    x = torch.randn(B * gh * gw, C, device=DEV, generator=g) * 2 + 0.5
    gamma = 1 + 0.2 * torch.randn(K, device=DEV, generator=g)
    beta = 0.1 * torch.randn(K, device=DEV, generator=g)
    rows = B * (gh // p) * (gw // p)
    big = torch.full((rows + 2, ldo), NAN, device=DEV, dtype=torch.bfloat16)
    out = big[:rows]
    _lib.merge_patches_ln(x, gamma, beta, out, B, gh, gw, p)
    torch.cuda.synchronize()
    merged = x.view(B, gh // p, p, gw // p, p, C).permute(0, 1, 3, 2, 4, 5).reshape(rows, K)      # (p1 p2 c)
    ref, bound = layernorm_reference(merged, gamma, beta, eps=1e-5)
    check(out[:, :K], ref, bound, f"merge_patches_ln p={p} {gh}x{gw} C={C}")
    assert (out[:, K:] == 0).all(), "the K padding is not zero"
    assert torch.isnan(big[rows:].float()).all(), "rows past the output were written"


@pytest.mark.parametrize("gh,gw", [(1, 1), (2, 5), (7, 7), (14, 9)])
@pytest.mark.parametrize("k", [1, 3, 5, 7])
def test_peg_within_bounds_and_isolated(k, gh, gw):
    B, C = 3, 24
    g = torch.Generator(device=DEV).manual_seed(k * 100 + gh * 10 + gw)
    x = torch.randn(B * gh * gw, C, device=DEV, generator=g)
    w = 0.4 * torch.randn(k * k, C, device=DEV, generator=g)
    b = 0.2 * torch.randn(C, device=DEV, generator=g)

    def run(xin):
        big = torch.full((B * gh * gw + 2, C), NAN, device=DEV)
        _lib.peg(xin, w, b, big[:B * gh * gw], B, gh, gw, k)
        torch.cuda.synchronize()
        return big
    big = run(x)
    y = big[:B * gh * gw]
    assert torch.isnan(big[B * gh * gw:]).all()
    ref, bound = peg_reference(x, w, b, B, gh, gw, k)
    check(y, ref, bound, f"peg k={k} {gh}x{gw}")
    bad = x.clone()
    bad[gh * gw:2 * gh * gw] = NAN
    image = torch.arange(B * gh * gw, device=DEV) // (gh * gw)
    assert rows_equal(run(bad)[:B * gh * gw], y)[image != 1].all()


# ============================================================================================================ model
@pytest.mark.parametrize("ln_mode", P.BOTH)
@pytest.mark.parametrize("name", sorted(TWINS_CASES))
def test_fused_against_reference_goldens(name, ln_mode, monkeypatch):
    """Every case of the spec against the reference's stored logits and the module's own bf16 graph, in both
    LayerNorm modes, with the shared comparison (fused_reason is None, launches counted, tol 3e-2)."""
    monkeypatch.setitem(P.FAMILIES, "twins_svt", FAMILY)
    monkeypatch.setitem(P.GPU, "twins_svt", dict(tol=3e-2, ln_modes=P.BOTH, second="eager bf16"))
    P.test_fused_against_reference_goldens("twins_svt", name, ln_mode, monkeypatch)


def small_model(seed=0):
    f = FAMILY
    spec = dict(TWINS_CASES["nonsquare_packed"], seed=seed)
    return f.build(spec).to(DEV, torch.bfloat16), f.input(spec).to(DEV)


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


def test_weight_update_needs_refresh():
    m, x = small_model()
    with torch.inference_mode():
        before = m(x).clone()
        m.layers[6].bias.data.add_(1.0)                   # through .data: the version counter does not move
        m.refresh_fused_weights()
        after = m(x)
    assert torch.allclose(after.float(), before.float() + 1.0, atol=5e-2)
    with torch.no_grad():
        m.layers[0][1].layers[0][2].fn.to_kv.weight.mul_(0.0)      # in place: picked up by the version counter
        assert not torch.equal(m(x), after)


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
        h = m.layers[1][2].register_forward_hook(lambda mod, i, o: seen.append(tuple(o.shape)))
        assert "hooks" in m.fused_reason(x)
        m(x)
        assert seen == [(2, 24, 16, 8)]
        h.remove()
        assert m.fused_reason(x) is None
