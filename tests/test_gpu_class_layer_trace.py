"""-m gpu: the encoders of tests/test_class_layer_trace.py on the real kernels at production-like widths (D 384 in 6
heads of 64, as tests/test_gpu_layer_trace.py), traced back to their reference layers: SimpleViT, flash-attention
SimpleViT, PiT and NesT through run_blocks; CrossViT's MultiScaleEncoder with sm_dim != lg_dim (the projection path)
and cross depth 2; CaiT (talking heads, layer subsets in both stages) and XCiT (class depth 2) through their
forward_fused after the patch embedding; and LeViT's whole forward with a downsampling layer and a distill head.

For each case and LayerNorm mode every operand of every launch is what the reference module's forward defines
(provenance) and every output is within its kernel's fp64 bound on the operands it received.  The worst
|got - ref| / bound per (case, launch kind) is printed at the end of the module.  Every planted defect of
tests/test_class_layer_trace.py is re-run through the real kernels: the walk must name it; how far it moves the
output from the module's own fp32 forward, against the family's parity tolerance, is printed, not asserted."""
import pytest
import torch

import test_class_layer_trace as C
from oracle import layer_trace as LT
from test_gpu_layer_trace import DH, H, MLP, D, perturbed, rerun_plain, traced
from vit_pytorch_b200 import _lib, cait, cross_vit, engine, levit, xcit
from vit_pytorch_b200 import nest, pit, simple_flash_attn_vit, simple_vit

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst |got - ref| / bound per case, LayerNorm mode and launch kind:")
    for key in sorted(WORST):
        print(f"  {' | '.join(key)}: {WORST[key]:.3f}")


def _record(name, ln_mode, launches):
    for kind, r in LT.check_accuracy(launches, f"{name} | {ln_mode}", rerun_plain=rerun_plain).items():
        WORST[(name, ln_mode, kind)] = max(WORST.get((name, ln_mode, kind), 0.0), r)


def _x(rows, width, seed):
    return torch.randn(rows, width, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))


# name: (module, B, N) of one run_blocks call
BLOCKS = {
    "simple_vit": (lambda: simple_vit.Transformer(D, 2, H, DH, MLP), 3, 196),
    "simple_flash_attn_vit": (lambda: simple_flash_attn_vit.Transformer(D, 2, H, DH, MLP, True), 3, 196),
    "pit stage": (lambda: pit.Transformer(D, 2, H, DH, MLP), 3, 1 + 27 * 27),
    # 2 images of 4 x 4 blocks of 7 x 7 tokens
    "nest level": (lambda: nest.Transformer(D, 49, 2, H, 4), 2 * 16, 49),
}


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", list(BLOCKS))
def test_block_launches_trace_back_and_stay_within_bounds(name, ln_mode):
    build, B, N = BLOCKS[name]
    mod = perturbed(build)
    x = _x(B * N, D, N)
    kw = dict(B=B, N=N, primed=True)
    x0 = x.clone()
    with torch.no_grad():
        launches = traced(mod, x, kw, ln_mode)
        assert LT.check_provenance(mod, x0, kw, launches, ln_mode, f"{name} | {ln_mode}") == len(launches) > 0
        _record(name, ln_mode, launches)


def _mse():
    return cross_vit.MultiScaleEncoder(depth=2, sm_dim=192, lg_dim=D, cross_attn_heads=H, cross_attn_depth=2,
                                       cross_attn_dim_head=DH, sm_enc_params=dict(depth=1, heads=3, mlp_dim=768,
                                                                                  dim_head=DH),
                                       lg_enc_params=dict(depth=2, heads=H, mlp_dim=MLP, dim_head=DH))


CROSS_B, CROSS_NS, CROSS_NL = 3, 1 + 14 * 14, 1 + 7 * 7


def cross_vit_run(ln_mode, plant=None):
    """(module, xs0, xl0, launches, fused output streams) of fused_two_streams on the real kernels."""
    B, Ns, Nl = CROSS_B, CROSS_NS, CROSS_NL
    mse = perturbed(_mse)
    if plant is not None:
        plant(mse)
    xs, xl = _x(B * Ns, 192, 1), _x(B * Nl, D, 2)
    xs0, xl0 = xs.clone(), xl.clone()
    stages = mse.stages()
    outs = []

    def setup():
        for eng, x in ((stages[0][0], xs), (stages[0][1], xl)):
            for buf in eng.workspace(x.shape[0], x.device).values():
                buf.fill_(float("nan"))
    launches = LT.trace_call(lambda: outs.append(engine.fused_two_streams(
        stages, xs, xl, B, Ns, Nl, False, mse.cls_rows(B, Ns, Nl, xs.device))[0]), ln_mode, setup=setup)
    torch.cuda.synchronize()
    return mse, xs0, xl0, launches, [o.clone() for o in outs[0]]


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
def test_cross_vit_launches_trace_back_and_stay_within_bounds(ln_mode):
    name = "cross_vit sm 192 lg 384 cross depth 2"
    with torch.no_grad():
        mse, xs0, xl0, launches, _ = cross_vit_run(ln_mode)
        n = LT.check_cross_vit_provenance(mse, xs0, xl0, CROSS_B, CROSS_NS, CROSS_NL, False, launches, ln_mode,
                                          f"{name} | {ln_mode}")
        assert n == len(launches) > 0
        _record(name, ln_mode, launches)


# family: (model, patch grid (h, w), layers the patch encoder runs, layers the class stage runs)
CLASS_MODELS = {
    "cait": (lambda: cait.CaiT(image_size=224, patch_size=16, num_classes=1000, dim=D, depth=3, cls_depth=3, heads=H,
                               mlp_dim=MLP, dim_head=DH), (14, 14), [0, 2], [0, 2]),
    "xcit": (lambda: xcit.XCiT(image_size=224, patch_size=16, num_classes=1000, dim=D, depth=2, cls_depth=2, heads=H,
                               mlp_dim=MLP, dim_head=DH), (14, 14), [0, 1], [0, 1]),
}
B_CLS = 3
REAL_ROWSTATS = _lib.rowstats_cast


def class_run(mp, family, ln_mode, plant=None):
    """(model, x0, launches, logits) of CaiT's or XCiT's forward_fused after the patch embedding, on the real kernels."""
    build, (gh, gw), patch, cls = CLASS_MODELS[family]
    model = C._kept(perturbed(build), patch, cls)
    if plant is not None:
        plant(model)
    img = torch.zeros(B_CLS, 3, 16 * gh, 16 * gw, device=DEV, dtype=torch.bfloat16)
    x0 = _x(B_CLS * gh * gw, D, 3)
    launches, out = C.trace_class_model(mp, model, img, x0, ln_mode, impl=LT.real_impl,
                                        prime=lambda a, b, st: REAL_ROWSTATS(a, b, st))
    torch.cuda.synchronize()
    return model, x0, launches, out


def class_eager(model, x0):
    """cait.py:246-255 / xcit.py:380-393 in fp32 from the embedded tokens x0, the layers kept_layers() names."""
    is_xcit = isinstance(model, xcit.XCiT)
    enc = model.xcit_transformer if is_xcit else model.patch_transformer
    gh, gw = CLASS_MODELS["xcit" if is_xcit else "cait"][1]
    x = x0.view(B_CLS, gh, gw, D) if is_xcit else x0.view(B_CLS, gh * gw, D)
    for i in enc.kept_layers():
        for blk in enc.layers[i]:
            x = blk(x) + x
    if is_xcit:
        x = model.final_norm(x).reshape(B_CLS, gh * gw, D)
    c = model.cls_token.reshape(1, 1, D).expand(B_CLS, 1, D)
    for i in model.cls_transformer.kept_layers():
        ls_attn, ls_ff = model.cls_transformer.layers[i]
        c = ls_attn(c, context=x) + c
        c = ls_ff(c) + c
    return model.mlp_head(c[:, 0])


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("family", list(CLASS_MODELS))
def test_class_attention_traces_back_and_stays_within_bounds(family, ln_mode, monkeypatch):
    with torch.no_grad():
        model, x0, launches, _ = class_run(monkeypatch, family, ln_mode)
        name = f"{family} class stage"
        n = LT.check_class_stage_provenance(model, x0, B_CLS, CLASS_MODELS[family][1], launches, ln_mode,
                                            f"{name} | {ln_mode}")
        assert n == len(launches) > 0
        _record(name, ln_mode, launches)


LEVIT = dict(image_size=224, num_classes=1000, dim=(256, D), depth=(2, 2), heads=(4, H), mlp_mult=2, stages=2,
             dim_key=32, dim_value=64, num_distill_classes=1000)


def levit_run(ln_mode="fold", plant=None):
    mod = perturbed(lambda: levit.LeViT(**LEVIT))
    if plant is not None:
        plant(mod)
    img = torch.randn(3, 3, 224, 224, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9)).bfloat16()
    outs = []
    launches = LT.trace_call(lambda: outs.append(mod.forward_fused(img)), ln_mode)
    torch.cuda.synchronize()
    return mod, img, launches, outs[0]


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
def test_levit_forward_traces_back_and_stays_within_bounds(ln_mode):
    with torch.no_grad():
        mod, img, launches, _ = levit_run(ln_mode)
        assert LT.check_levit_provenance(mod, img, launches, f"levit | {ln_mode}") == len(launches) > 0
        assert sum(c.name == "attention_posbias" and c.args["s"] == 2 for c in launches) == 1
        _record("levit downsampling distill", ln_mode, launches)


# ------------------------------------------------------------------------------------------------------ planted defects
# the parity tolerance of each family on its logits (tests/test_gpu_family_parity.py, tests/test_gpu_levit.py)
TOL = {"cross_vit": 2e-2, "cait": 3e-2, "xcit": 3e-2, "levit": 3e-2}


def _family(kind, case):
    return case.split()[0] if kind == "class" else kind


def _defect_run(mp, kind, case, ln_mode, plant_mod):
    """(check(): the walk of the trace, max |fused - the module's own fp32 forward|, what that difference is over)."""
    if kind == "cross_vit":
        mse, xs0, xl0, launches, out = cross_vit_run(ln_mode, plant_mod)
        with mp.context() as eager:                 # the branch Transformers' own PyTorch graph
            eager.setenv("B200VIT_DISABLE_FUSED", "1")
            want = mse.forward_eager(xs0.view(CROSS_B, CROSS_NS, -1), xl0.view(CROSS_B, CROSS_NL, -1))
        diff = max((o - w.reshape(o.shape)).abs().max().item() for o, w in zip(out, want))
        return (lambda: LT.check_cross_vit_provenance(mse, xs0, xl0, CROSS_B, CROSS_NS, CROSS_NL, False, launches,
                                                      ln_mode, case)), diff, "the encoder's output streams"
    if kind == "class":
        family = _family(kind, case)
        model, x0, launches, out = class_run(mp, family, ln_mode, plant_mod)
        diff = (out.float() - class_eager(model, x0)).abs().max().item()
        return (lambda: LT.check_class_stage_provenance(model, x0, B_CLS, CLASS_MODELS[family][1], launches, ln_mode,
                                                        case)), diff, "the logits"
    mod, img, launches, (out, distill) = levit_run(ln_mode, plant_mod)
    eo, ed = mod.forward_eager(img.float())
    diff = max((out.float() - eo).abs().max().item(), (distill.float() - ed).abs().max().item())
    return (lambda: LT.check_levit_provenance(mod, img, launches, case)), diff, "the logits"


@pytest.mark.parametrize("defect", list(C.DEFECTS))
def test_planted_defect_is_named_on_the_real_kernels(defect, monkeypatch):
    kind, case, ln_mode, plant, plant_mod, want = C.DEFECTS[defect]
    family = _family(kind, case)
    with torch.no_grad():
        check, clean, what = _defect_run(monkeypatch, kind, case, ln_mode, None)
        check()
        if plant is not None:
            plant(monkeypatch)
        try:
            check, bad, what = _defect_run(monkeypatch, kind, case, ln_mode, plant_mod)
        except AssertionError as e:               # the library's own argument checks refuse the launch
            print(f"\n{defect}: refused before any launch by the library's argument check ({e!r})")
            return
        with pytest.raises(LT.ProvenanceError) as e:
            check()
    assert all(w in str(e.value) for w in want), str(e.value)
    tol = TOL[family]
    print(f"\n{defect} ({family}): max |fused - eager fp32| over {what} {clean:.3e} without the defect, {bad:.3e} "
          f"with it; the family's {tol:g} parity tolerance would {'miss' if bad < tol else 'catch'} it")
