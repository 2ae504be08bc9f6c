"""Adaptive Token Sampling ViT (vit_pytorch_b200.ats_vit) without a GPU.

* The fused dataflow: ViT.forward_fused runs on CPU with every library launch traced (oracle/layer_trace.tracer) and
  emulated -- the encoder kernels by their fp64 references (oracle/layer_trace.emulate_impl), the select, gather and
  per-image-key-count attention by oracle/ats_bounds.py -- with the fixture's uniforms replayed through
  ats_vit.draw_uniform.  Its token ids must be the reference's and its logits within the family tolerance of the
  reference's fp32 logits, in both LayerNorm modes; the launch sequence must follow the layers' slot plan.
* Dispatch: the slot plan, fused_reason's fall-backs.
* The new entry points: the header declares them and their limits, the library exports them, the wrappers check their
  arguments."""
import os
import re
import sys

import pytest
import torch

from conftest import GOLDEN_DIR, load_golden
from oracle import ats_bounds as AT
from oracle import layer_trace as LT
from vit_pytorch_b200 import _lib
from vit_pytorch_b200 import ats_vit as A

sys.path.insert(0, GOLDEN_DIR)
import make_engine_schedule as S  # noqa: E402
from ats_vit_spec import ATS_CASES, FAMILY  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ATS_ENTRY_POINTS = ("ats_select", "ats_gather", "attention_kv_lens")
ATS_OUTPUTS = {"ats_select": ("src", "lens_out", "ids_out"), "ats_gather": ("x_out", "a_out"),
               "attention_kv_lens": ("out",)}
FUSED_CASES = ["readme", "stays_off", "ragged", "no_sampling", "dh80", "smaller_input"]


def replay(case: dict):
    """A draw_uniform that returns the fixture's uniforms of the layers where the reference sampled, padded from its
    padded length to the fused path's slot (the padding is never read), and 0.5 where it did not (no draw is read)."""
    drawn = case["uniforms"]

    def draw(shape, device, dtype, layer):
        u = torch.full(shape, 0.5, dtype=torch.float32)
        rec = drawn.get(f"layer{layer}")
        if rec is not None:
            u[:, :, :rec.shape[2]] = rec.float()
        return u.to(device)
    return draw


def ats_impl(name, real):
    if name == "ats_select":
        def run(qkv, lens, ids, u, src, lens_out, ids_out, B, S_in, K, H, dh, scale):
            s, lo, io = AT.emulate_select(qkv, lens, ids, u, B, S_in, K, H, dh, scale)
            src.copy_(s), lens_out.copy_(lo), ids_out.copy_(io)
        return run
    if name == "ats_gather":
        def run(src, x=None, x_out=None, a=None, a_out=None, ncols=0):
            idx = src.long()
            if x is not None:
                x_out.copy_(x[idx])
            if a is not None:
                a_out[:, :ncols] = a[idx, :ncols]
        return run
    if name == "attention_kv_lens":
        def run(q, kv, out, lens, B, Nq, Nk, H, dh, scale):
            ref, _ = AT.kv_lens_reference(q, kv, [int(v) for v in lens], B, Nq, Nk, H, dh, LT.f32(scale))
            out.copy_(ref.bfloat16())
        return run
    return LT.emulate_impl(name, real)


def trace(model, img, ln_mode, monkeypatch, case, impl=ats_impl):
    """(launches, (logits, ids, lens)) of model.forward_fused(img) with the case's uniforms replayed."""
    for k, v in ATS_OUTPUTS.items():
        monkeypatch.setitem(LT.OUTPUTS, k, v)
    monkeypatch.setattr(A, "draw_uniform", replay(case))
    outs = []
    with S.recording(None, lambda: [], ln_mode, "python", LT.FRONT_ENTRY_POINTS + ATS_ENTRY_POINTS,
                     recorder=LT.tracer(impl)) as rec:
        with torch.inference_mode():
            outs.append(model.forward_fused(img))
    return rec.launches, outs[0]


def returned_ids(ids: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
    """What ViT.forward returns for the fused path's ids and lengths."""
    return ids[:, 1:int(lens.max())].long() - 1


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", FUSED_CASES)
def test_emulated_fused_forward_matches_reference(name, ln_mode, monkeypatch):
    spec, case = ATS_CASES[name], load_golden("ats_vit")["cases"][name]
    model = FAMILY.build(spec).bfloat16()
    img = FAMILY.input(spec)
    launches, (logits, ids, lens) = trace(model, img, ln_mode, monkeypatch, case)
    assert torch.equal(returned_ids(ids, lens), case["token_ids"])
    d = (logits.float() - case["logits_sampled"]).abs().max().item()
    assert d < 3e-2, (name, ln_mode, d)
    # the launch sequence follows the slot plan: one select + gather per layer that may sample, one key-count
    # attention per layer from the first of them on, plain attention before it
    n = img.shape[2] // 8 * img.shape[3] // 8 + 1
    plan = A.slot_plan(n, FAMILY.case_kwargs(spec)["max_tokens_per_depth"])
    first = next((i for i, p in enumerate(plan) if p[2]), len(plan))
    names = [c.name for c in launches]
    assert names.count("ats_select") == names.count("ats_gather") == sum(p[2] for p in plan)
    assert names.count("attention_kv_lens") == len(plan) - first
    assert names.count("attention") == first
    # the ids are an exact function of the draws: lengths, padding at the cls row, -1 in the returned ids
    for b in range(lens.shape[0]):
        L = int(lens[b])
        assert (ids[b, L:] == 0).all()


def test_dispatch():
    m = A.ViT(image_size=32, patch_size=8, num_classes=3, dim=64, depth=2, max_tokens_per_depth=(8, 4), heads=2,
              mlp_dim=64, dim_head=32)
    img = torch.zeros(1, 3, 32, 32)
    assert m.fused_reason(img) == "input is not on a CUDA device"
    assert m.fused_reason(torch.zeros(1, 3, 32)) == "input is not (B, C, H, W)"
    assert A.slot_plan(17, (8, 4)) == [(17, 9, True), (9, 5, True)]
    assert A.slot_plan(17, (16, 8, 8)) == [(17, 17, False), (17, 9, True), (9, 9, False)]
    assert A.slot_plan(65, (256, 128, 64, 32, 16, 8))[2:] == [(65, 65, False), (65, 33, True), (33, 17, True),
                                                            (17, 9, True)]


def test_fused_reason_names_the_select_limits(monkeypatch):
    m = A.ViT(image_size=32, patch_size=8, num_classes=3, dim=64, depth=1, max_tokens_per_depth=(4,), heads=2,
              mlp_dim=64, dim_head=32).bfloat16()
    img = torch.zeros(1, 3, 32, 32, dtype=torch.bfloat16)
    import vit_pytorch_b200.engine as E
    monkeypatch.setattr(E, "why_not_fused", lambda *a, **k: None)       # as on an H100
    assert m.fused_reason(img) is None
    monkeypatch.setattr(_lib, "ATS_MAX_TOKENS", 16)
    assert "select kernel takes at most 16" in m.fused_reason(img)
    monkeypatch.setattr(_lib, "ATS_MAX_TOKENS", 4096)
    monkeypatch.setattr(_lib, "ATS_MAX_HEAD_TOKENS", 32)
    assert "2 heads x 17 tokens" in m.fused_reason(img)
    m16 = A.ViT(image_size=32, patch_size=8, num_classes=3, dim=64, depth=1, max_tokens_per_depth=(4,), heads=4,
                mlp_dim=64, dim_head=16).bfloat16()
    assert m16.fused_reason(img) == "dim_head=16 (the attention kernels are built for 32, 64, 80 and 128)"


def test_header_declares_the_entry_points():
    h = open(os.path.join(ROOT, "include", "b200vit.h")).read()
    for sym in ("b200vit_ats_select", "b200vit_ats_gather", "b200vit_attention_kv_lens"):
        assert re.search(rf"\bint {sym}\(", h), sym
        assert sym in _lib.SYMBOLS
    assert int(re.search(r"#define B200VIT_ATS_MAX_TOKENS (\d+)", h).group(1)) == _lib.ATS_MAX_TOKENS
    assert int(re.search(r"#define B200VIT_ATS_MAX_HEAD_TOKENS (\d+)", h).group(1)) == _lib.ATS_MAX_HEAD_TOKENS


def test_library_exports_the_entry_points():
    if not _lib.LIB_PATH.exists():
        pytest.skip("library not built")
    L = _lib.lib()
    for sym in ("b200vit_ats_select", "b200vit_ats_gather", "b200vit_attention_kv_lens"):
        assert hasattr(L, sym)


def _bf(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


def _i32(n):
    return torch.zeros(n, dtype=torch.int32)


# B = 2 images of S = 5 rows, K = 2 (S_out = 3), H = 2 heads of 32: every call breaks one rule and must be refused
# with that rule's message before the library (or a device) is reached
SELECT_OK = dict(qkv=_bf(10, 192), lens=_i32(2), ids=_i32(10), u=torch.zeros(2, 2, 4), src=_i32(6), lens_out=_i32(2),
                 ids_out=_i32(6), B=2, S_in=5, K=2, H=2, dh=32, scale=1.0)
SELECT_BAD = [
    (dict(qkv=_bf(9, 192)), "qkv must be"),
    (dict(qkv=_bf(10, 191)), "qkv must be"),
    (dict(u=torch.zeros(2, 2, 5)), "u must be contiguous"),
    (dict(u=torch.zeros(2, 2, 4, dtype=torch.float64)), "u must be fp32 or bf16"),
    (dict(lens=torch.zeros(2, dtype=torch.int64)), "lens must be contiguous int32"),
    (dict(ids=_i32(9)), "ids must be contiguous int32"),
    (dict(src=_i32(10)), "src must be contiguous int32"),
    (dict(ids_out=_i32(10)), "ids_out must be contiguous int32"),
]
KV_OK = dict(q=_bf(6, 64), kv=_bf(8, 128), out=_bf(6, 64), lens=_i32(2), B=2, Nq=3, Nk=4, H=2, dh=32, scale=1.0)
KV_BAD = [
    (dict(q=_bf(6, 32)), "q must be"),
    (dict(kv=_bf(8, 64)), "kv must be"),
    (dict(out=_bf(64, 6).t()), "out must be contiguous"),
    (dict(lens=_i32(3)), "lens must be contiguous int32"),
    (dict(lens=torch.zeros(2)), "lens must be contiguous int32"),
]
GATHER_OK = dict(src=_i32(3), x=torch.zeros(5, 8), x_out=torch.zeros(3, 8), a=_bf(5, 16), a_out=_bf(3, 16), ncols=16)
GATHER_BAD = [
    (dict(src=torch.zeros(3)), "src must be a contiguous int32"),
    (dict(x_out=None), "give x with x_out"),
    (dict(x_out=torch.zeros(4, 8)), "x_out must be"),
    (dict(x=torch.zeros(5, 8, dtype=torch.float64), x_out=torch.zeros(3, 8, dtype=torch.float64)), "must be fp32"),
    (dict(ncols=24), "at least ncols"),
    (dict(a=torch.zeros(5, 16), a_out=torch.zeros(3, 16)), "must be bf16"),
]


@pytest.mark.parametrize("bad,msg", SELECT_BAD)
def test_ats_select_checks_its_arguments(bad, msg):
    with pytest.raises(_lib.B200VitError, match=msg):
        _lib.ats_select(**dict(SELECT_OK, **bad))


@pytest.mark.parametrize("bad,msg", KV_BAD)
def test_attention_kv_lens_checks_its_arguments(bad, msg):
    with pytest.raises(_lib.B200VitError, match=msg):
        _lib.attention_kv_lens(**dict(KV_OK, **bad))


@pytest.mark.parametrize("bad,msg", GATHER_BAD)
def test_ats_gather_checks_its_arguments(bad, msg):
    with pytest.raises(_lib.B200VitError, match=msg):
        _lib.ats_gather(**dict(GATHER_OK, **bad))


def test_valid_arguments_pass_the_shape_checks():
    """The valid calls above get past every shape rule: on a CPU tensor the first refusal is the device check."""
    for fn, kw in ((_lib.ats_select, SELECT_OK), (_lib.attention_kv_lens, KV_OK), (_lib.ats_gather, GATHER_OK)):
        with pytest.raises(_lib.B200VitError, match="expected CUDA"):
            fn(**kw)


# ------------------------------------------------------------------------------------------------------ launch sequence
import json  # noqa: E402

import make_ats_vit_schedule as AS  # noqa: E402


@pytest.fixture(scope="module")
def schedule():
    with open(AS.FIXTURE) as f:
        return json.load(f)


def test_schedule_fixture_lists_every_run(schedule):
    assert list(schedule) == [AS.run_name(m, h) for m, h in AS.RUNS]


@pytest.mark.parametrize("ln_mode,host_loop", AS.RUNS)
def test_fused_forward_schedule_matches_fixture(schedule, ln_mode, host_loop):
    """Every launch of ViT.forward_fused, recorded on CPU: its entry point, its scalars, the buffer (and offset, shape,
    stride) of every tensor and the digest of every prepared weight, against tests/golden/ats_vit_schedule.json."""
    name = AS.run_name(ln_mode, host_loop)
    got, want = AS.record(ln_mode, host_loop), schedule[name]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: call {i} differs"
    assert len(got) == len(want), f"{name}: {len(got)} calls, {len(want)} expected"
