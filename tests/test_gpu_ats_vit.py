"""Adaptive Token Sampling ViT on the GPU: the select kernel against the fp64 oracle oracle/ats_bounds.py on bf16 qkv,
the gather as bit copies, the per-image-key-count attention against oracle/attention_bounds.py (and plain
b200vit_attention_kv unchanged), NaN / Inf kept inside one image, the model against the reference fixture with its
uniforms replayed in both LayerNorm modes, repeats, CUDA-graph replay, and the fall-backs."""
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, load_golden
from oracle import ats_bounds as AT
from vit_pytorch_b200 import _lib
from vit_pytorch_b200 import ats_vit as A
from vit_pytorch_b200.graph import GraphedForward

sys.path.insert(0, GOLDEN_DIR)
from ats_vit_spec import ATS_CASES, FAMILY  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
NEW_KERNELS = ("ats_select", "ats_gather", "attention_kv_lens")


def _qkv(B, S, H, dh, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B * S, 3 * H * dh, generator=g) * 0.8).bfloat16().to(DEV)


def _select(qkv, lens, u, B, S, K, H, dh, scale):
    S_out = min(S, K + 1)
    ids = torch.arange(S, dtype=torch.int32).repeat(B).to(DEV) * 3 + 7     # any ids: they travel with the rows
    src = torch.empty(B * S_out, dtype=torch.int32, device=DEV)
    lo = torch.empty(B, dtype=torch.int32, device=DEV)
    io = torch.empty(B * S_out, dtype=torch.int32, device=DEV)
    _lib.ats_select(qkv, torch.tensor(lens, dtype=torch.int32, device=DEV), ids, u, src, lo, io, B, S, K, H, dh, scale)
    torch.cuda.synchronize()
    return src.cpu(), lo.cpu(), io.cpu(), ids.cpu()


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
@pytest.mark.parametrize("u_dtype", [torch.float32, torch.bfloat16])
def test_select_against_fp64_oracle(dh, u_dtype):
    B, S, K, H = 3, 70, 12, 3
    lens = [70, 41, 2]
    qkv = _qkv(B, S, H, dh, seed=dh)
    g = torch.Generator().manual_seed(7 + dh)
    u = torch.rand(B, K, S - 1, generator=g).to(u_dtype).to(DEV)
    scale = dh ** -0.5
    src, lo, io, ids = _select(qkv, lens, u, B, S, K, H, dh, scale)
    ref = AT.select_reference(qkv.cpu(), lens, u.cpu().float(), B, S, K, H, dh, scale)
    ok = AT.allowed_draws(ref)
    S_out = K + 1
    for b in range(B):
        kept = [int(s) - b * S for s in src[b * S_out:b * S_out + int(lo[b])]]
        assert kept[0] == 0 and kept == sorted(set(kept)), kept
        cand = set(c - 1 for c in kept[1:])
        # every unambiguous draw is the fp64 argmax and is kept; every kept candidate is an allowed draw
        for k in range(K):
            if ref["gap"][b, k] > 2 * ref["bound"][b, k].max():
                assert int(ref["argmax"][b, k]) in cand, (b, k)
        assert all(bool(ok[b, :, c].any()) for c in cand), (b, cand)
        # the rest of the outputs are an exact function of the kept set
        draws = torch.tensor(sorted(cand) + [min(cand)] * (K - len(cand)))
        want_src, want_lo, want_io, sampled = AT.select_outputs(draws[None].expand(B, -1), lens, ids, B, S, K)
        assert sampled
        sl = slice(b * S_out, (b + 1) * S_out)
        assert torch.equal(src[sl], want_src[sl]) and int(lo[b]) == int(want_lo[b]) and torch.equal(io[sl], want_io[sl])


def test_select_without_sampling_is_the_identity():
    B, S, K, H, dh = 2, 20, 16, 2, 64
    qkv = _qkv(B, S, H, dh, seed=3)
    u = torch.rand(B, K, S - 1, device=DEV)
    src, lo, io, ids = _select(qkv, [17, 12], u, B, S, K, H, dh, 0.125)
    for b, L in enumerate([17, 12]):
        row = src[b * 17:(b + 1) * 17] - b * S
        assert row[:L].tolist() == list(range(L)) and (row[L:] == 0).all() and int(lo[b]) == L


def test_gather_rows_are_bit_copies():
    rows, D, W = 50, 96, 192
    x = torch.randn(80, D, device=DEV)
    a = torch.randn(80, W, device=DEV).bfloat16()
    src = torch.randint(0, 80, (rows,), dtype=torch.int32, device=DEV)
    xo = torch.empty(rows, D, device=DEV)
    ao = torch.zeros(rows, 64, device=DEV, dtype=torch.bfloat16)
    _lib.ats_gather(src, x=x, x_out=xo, a=a, a_out=ao, ncols=64)
    torch.cuda.synchronize()
    assert torch.equal(xo, x[src.long()]) and torch.equal(ao, a[src.long(), :64])


@pytest.mark.parametrize("dh", [32, 64, 80, 128])
def test_kv_lens_attention_within_bounds(dh):
    B, Nq, Nk, H = 3, 33, 130, 2
    lens = [130, 61, 1]
    qkv = _qkv(B, Nk, H, dh, seed=20 + dh)
    I = H * dh
    q = torch.randn(B * Nq, I, device=DEV).bfloat16()
    out = torch.empty(B * Nq, I, device=DEV, dtype=torch.bfloat16)
    _lib.attention_kv_lens(q, qkv[:, I:], out, torch.tensor(lens, dtype=torch.int32, device=DEV), B, Nq, Nk, H, dh,
                           dh ** -0.5)
    torch.cuda.synchronize()
    ref, bound = AT.kv_lens_reference(q.cpu(), qkv[:, I:].cpu(), lens, B, Nq, Nk, H, dh, dh ** -0.5)
    err = (out.cpu().double() - ref).abs()
    assert bool((err <= bound).all()), float((err - bound).max())
    # every key: the plain kernel's bits
    plain = torch.empty_like(out)
    full = torch.full((B,), Nk, dtype=torch.int32, device=DEV)
    _lib.attention_kv(q, qkv[:, I:], plain, B, Nq, Nk, H, dh, dh ** -0.5)
    _lib.attention_kv_lens(q, qkv[:, I:], out, full, B, Nq, Nk, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    assert torch.equal(out, plain)


def test_nan_and_inf_stay_in_their_image():
    B, S, K, H, dh = 3, 40, 8, 2, 64
    I = H * dh
    lens = torch.tensor([40, 30, 40], dtype=torch.int32, device=DEV)
    u = torch.rand(B, K, S - 1, device=DEV)
    outs = []
    for poison in (None, float("nan"), float("inf")):
        qkv = _qkv(B, S, H, dh, seed=5)
        if poison is not None:
            qkv[S + 3] = poison
            qkv[S + 35] = poison                          # past image 1's valid keys
        src, lo, io, _ = _select(qkv, lens.tolist(), u, B, S, K, H, dh, 0.125)
        o = torch.empty(B * S, I, device=DEV, dtype=torch.bfloat16)
        _lib.attention_kv_lens(qkv[:, :I], qkv[:, I:], o, lens, B, S, S, H, dh, 0.125)
        torch.cuda.synchronize()
        outs.append((src.view(B, -1), lo, io.view(B, -1), o.view(B, S, I).cpu()))
    for got in outs[1:]:
        for b in (0, 2):
            assert torch.equal(got[0][b], outs[0][0][b]) and got[1][b] == outs[0][1][b]
            assert torch.equal(got[2][b], outs[0][2][b]) and torch.equal(got[3][b], outs[0][3][b])


def test_poison_past_an_images_valid_rows_leaves_its_selection_unchanged():
    """Rows of image 1's slot past its valid length hold NaN or Inf: its own selection reads none of them."""
    B, S, K, H, dh = 3, 40, 8, 2, 64
    lens = [40, 30, 40]
    u = torch.rand(B, K, S - 1, device=DEV)
    outs = []
    for poison in (None, float("nan"), float("inf")):
        qkv = _qkv(B, S, H, dh, seed=6)
        if poison is not None:
            qkv[S + 30:2 * S] = poison
        src, lo, io, _ = _select(qkv, lens, u, B, S, K, H, dh, 0.125)
        outs.append((src, lo, io))
    for got in outs[1:]:
        assert all(torch.equal(g, w) for g, w in zip(got, outs[0]))


def _replay(case):
    """draw_uniform replaying the fixture's uniforms (device tensors made up front, so a capture can use them)."""
    cache = {}

    def draw(shape, device, dtype, layer):
        key = (tuple(shape), layer)
        if key not in cache:
            u = torch.full(shape, 0.5, dtype=torch.float32)
            rec = case["uniforms"].get(f"layer{layer}")
            if rec is not None:
                u[:, :, :rec.shape[2]] = rec.float()
            cache[key] = u.to(device)
        return cache[key]
    return draw


def _model(name):
    spec = ATS_CASES[name]
    return FAMILY.build(spec).to(DEV, torch.bfloat16), FAMILY.input(spec).to(DEV), load_golden("ats_vit")["cases"][name]


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", [n for n in ATS_CASES if n != "fallback_dh16"])
def test_model_matches_reference_fixture(name, ln_mode, monkeypatch):
    monkeypatch.setenv("B200VIT_LN_MODE", ln_mode)
    m, x, case = _model(name)
    monkeypatch.setattr(A, "draw_uniform", _replay(case))
    _lib.reset_launch_count()
    with torch.inference_mode():
        assert m.fused_reason(x) is None
        logits, ids = m(x, return_sampled_token_ids=True)
    torch.cuda.synchronize()
    assert _lib.launch_count() > 0
    assert torch.equal(ids.cpu(), case["token_ids"]), (ids, case["token_ids"])
    d = (logits.float().cpu() - case["logits_sampled"]).abs().max().item()
    assert d < 3e-2, (name, ln_mode, d)


class _SelectLog:
    """ats_vit's view of the library that keeps every select call's operands and outputs (cloned after the call)."""

    def __init__(self, lib, layer):
        self.lib, self.layer, self.calls = lib, layer, []

    def __getattr__(self, name):
        return getattr(self.lib, name)

    def ats_select(self, qkv, lens, ids, u, src, lens_out, ids_out, B, S_in, K, H, dh, scale):
        self.lib.ats_select(qkv, lens, ids, u, src, lens_out, ids_out, B, S_in, K, H, dh, scale)
        self.calls.append(dict(layer=self.layer["i"], qkv=qkv.cpu(), lens=lens.cpu(), u=u.float().cpu(),
                               src=src.cpu(), lens_out=lens_out.cpu(), B=B, S_in=S_in, K=K, H=H, dh=dh, scale=scale))


def _logged_fused(name, monkeypatch):
    """(model, input, fixture case, fused logits, fused ids, select calls) of one fused forward on replayed draws."""
    m, x, case = _model(name)
    current = {"i": None}
    draw = _replay(case)

    def draw_logged(shape, device, dtype, layer):
        current["i"] = layer
        return draw(shape, device, dtype, layer)
    log = _SelectLog(A._lib, current)
    monkeypatch.setattr(A, "draw_uniform", draw_logged)
    monkeypatch.setattr(A, "_lib", log)
    with torch.inference_mode():
        logits, ids = m(x, return_sampled_token_ids=True)
    torch.cuda.synchronize()
    return m, x, case, logits.float().cpu(), ids.cpu(), log.calls


FUSED = [n for n in ATS_CASES if n != "fallback_dh16"]


@pytest.mark.parametrize("name", FUSED)
def test_logits_match_fp64_replay_of_the_fused_ids(name, monkeypatch):
    """The module's PyTorch graph in fp64, made to keep exactly the rows each select kernel kept (its Gumbel noise
    replaced by a draw that lands on them), reproduces the fused path's ids and, within the family tolerance, its
    logits: selection and arithmetic are checked apart."""
    _, x, _, logits, ids, calls = _logged_fused(name, monkeypatch)
    kept = {}
    for c in calls:
        if max(int(v) for v in c["lens"]) - 1 > c["K"]:
            S_out = min(c["S_in"], c["K"] + 1)
            kept[c["layer"]] = [[int(v) - b * c["S_in"] - 1 for v in c["src"][b * S_out + 1:b * S_out + int(c["lens_out"][b])]]
                                for b in range(c["B"])]
    m64 = FAMILY.build(ATS_CASES[name]).double()
    state = {}

    def forced(shape, device, dtype, eps=1e-6):
        g = torch.zeros(shape, dtype=dtype)
        for b, cand in enumerate(kept[state["layer"]]):
            for k in range(shape[1]):
                g[b, k, cand[k % len(cand)]] = 1e6
        return g
    hooks = [attn.register_forward_pre_hook(lambda mod, a, kw, i=i: state.__setitem__("layer", i), with_kwargs=True)
             for i, (attn, _) in enumerate(m64.transformer.layers)]
    monkeypatch.setattr(A, "sample_gumbel", forced)
    try:
        with torch.inference_mode():
            want, want_ids = m64(x.cpu().double(), return_sampled_token_ids=True)
    finally:
        for h in hooks:
            h.remove()
    assert torch.equal(ids, want_ids)
    d = (logits - want).abs().max().item()
    assert d < 3e-2, (name, d)


@pytest.mark.parametrize("name", FUSED)
def test_pseudo_logits_stay_within_half_the_fixture_margin(name, monkeypatch):
    """The pseudo-logits the select kernel draws from -- the fp64 values of its own bf16 qkv -- differ from the fp32
    reference graph's by less than half the fixture's smallest Gumbel-max margin, so no draw of the fixture can flip.
    The deviation is printed next to the margin."""
    _, x, case, _, _, calls = _logged_fused(name, monkeypatch)
    ref = {}
    m = FAMILY.build(ATS_CASES[name])
    state = {}

    def pre_attention(i):
        return lambda mod, a, kw: state.__setitem__("layer", i)

    def pre_ats(mod, args, kwargs):
        attn, value, mask = args[0], args[1], kwargs["mask"]
        scores = torch.einsum('b h n, b h n -> b n', attn[..., 0, 1:], value[..., 1:, :].norm(dim=-1))
        lg = torch.log(scores / (scores.sum(dim=-1, keepdim=True) + mod.eps) + mod.eps)
        ref[state["layer"]] = lg.masked_fill(~mask[:, 1:], -float("inf")).double()
    hooks = []
    for i, (attn, _) in enumerate(m.transformer.layers):
        hooks.append(attn.register_forward_pre_hook(pre_attention(i), with_kwargs=True))
        if attn.ats is not None:
            hooks.append(attn.ats.register_forward_pre_hook(pre_ats, with_kwargs=True))
    try:
        torch.manual_seed(ATS_CASES[name]["noise_seed"])
        with torch.inference_mode():
            m(x.cpu().float())
    finally:
        for h in hooks:
            h.remove()
    dev = 0.0
    for c in calls:
        if c["layer"] not in ref:
            continue
        got = AT.select_reference(c["qkv"], [int(v) for v in c["lens"]], c["u"], c["B"], c["S_in"], c["K"], c["H"],
                                  c["dh"], c["scale"])["logit"]
        want = ref[c["layer"]]
        n = want.shape[1]
        valid = torch.isfinite(want)
        assert torch.equal(valid, torch.isfinite(got[:, :n])), name
        dev = max(dev, float((got[:, :n] - want)[valid].abs().max()))
    print(f"{name}: pseudo-logit deviation {dev:.4f}, fixture margin {case['margin']:.4f}")
    assert dev < case["margin"] / 2, (name, dev, case["margin"])


def test_repeats_and_graph_replay_are_bit_identical(monkeypatch):
    m, x, case = _model("readme")
    monkeypatch.setattr(A, "draw_uniform", _replay(case))
    with torch.inference_mode():
        a = m(x)
        b = m(x)
    assert torch.equal(a, b)
    g = GraphedForward(m, x)
    got = g(x).clone()
    torch.cuda.synchronize()
    assert torch.equal(got, a)


def test_graph_replay_with_torch_generator_runs():
    m, x, _ = _model("readme")
    g = GraphedForward(m, x)
    for _ in range(3):
        out = g(x)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out.float()).all())


def test_fallback_launches_none_of_the_new_kernels(monkeypatch):
    m, x, case = _model("fallback_dh16")
    assert m.fused_reason(x) is not None
    called = []
    for k in NEW_KERNELS:
        monkeypatch.setattr(_lib, k, lambda *a, _k=k, **kw: called.append(_k))
    with torch.inference_mode():
        torch.manual_seed(ATS_CASES["fallback_dh16"]["noise_seed"])
        out = m(x)
    assert not called and out.shape == case["logits_fp32"].shape
