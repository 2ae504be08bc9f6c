"""-m gpu: the encoder layers on token grids traced back to their reference layers on the real kernels
(oracle/layer_trace.py, tests/test_grid_layer_trace.py on CPU), at the first two stages of each family's README model
with two images: Twins-SVT (56 x 56 at dim 64, 28 x 28 at dim 128; windows 7, global k 7), MaxViT (dim 96 and 192,
windows 7), CrossFormer (dim 64 and 128, local windows 7, long windows 8 and 4), CvT (dim 64 and 192, projection 3,
key / value stride 2) and MobileViT-XS (dim 96 on 32 x 32 and 120 on 16 x 16, 2 x 2 patches); ScalableViT-S at 256 x
256 (64 x 64 at dim 64, 2 heads, dim_key 40, reduction 8, one 4096-token window; 32 x 32 at dim 128, 4 heads, reduction
4, windows 32) and its last stage (8 x 8 at dim 512, 16 heads, dim_key 32, reduction 1, the whole map), each through
Transformer.run_fused with its PEG; SepViT's stages 1, 2 and 4 (56 x 56 at dim 32 in 64 windows, 28 x 28 at dim 64,
7 x 7 at dim 256 in one window); RegionViT's stages 1 and 2 at depth 2 (56 x 56 / 8 x 8 at dim 64, 28 x 28 / 4 x 4 at
dim 128, windows 7), and one image of 7 x 7 / 1 x 1, whose 49 local rows put the region rows at an odd row offset.

For each case and LayerNorm mode: every operand of every launch is what the reference module's forward defines there,
and every output is within its kernel's fp64 bound on the operands it received.  The worst |got - ref| / bound per
(case, LayerNorm mode, launch kind) is printed at the end of the module.  Two planted defects are re-run through the
real kernels: the walk must name them; whether a model-level max-abs criterion would have seen them is printed, not
asserted."""
import pytest
import torch

from oracle import layer_trace as LT
from test_gpu_layer_trace import perturbed, rerun_plain, traced
from test_grid_layer_trace import (MaxViTBlock, _bn_default_eps, _dilated_swapped, _head_ln_default_eps,
                                   _iwsa_scale_padded)
from vit_pytorch_b200 import crossformer, cvt, mobile_vit, regionvit, scalable_vit, sep_vit, twins_svt

pytestmark = pytest.mark.gpu
DEV = "cuda"
B = 2
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst |got - ref| / bound per case, LayerNorm mode and launch kind:")
    for key in sorted(WORST):
        print(f"  {' | '.join(key)}: {WORST[key]:.3f}")


# name: (module, width, grid, extra run_blocks arguments)
CASES = {
    "twins stage 1": (lambda: twins_svt.Transformer(64, 1, local_patch_size=7, global_k=7), 64, (56, 56), {}),
    "twins stage 2": (lambda: twins_svt.Transformer(128, 1, local_patch_size=7, global_k=7), 128, (28, 28), {}),
    "max_vit stage 1": (lambda: MaxViTBlock(7, 96, 32, 4), 96, (56, 56), {}),
    "max_vit stage 2": (lambda: MaxViTBlock(7, 192, 32, 4), 192, (28, 28), {}),
    "crossformer stage 1": (lambda: crossformer.Transformer(64, local_window_size=7, global_window_size=8, depth=1),
                            64, (56, 56), {}),
    "crossformer stage 2": (lambda: crossformer.Transformer(128, local_window_size=7, global_window_size=4, depth=1),
                            128, (28, 28), {}),
    "cvt stage 1": (lambda: cvt.Transformer(64, 3, 2, 1, heads=1, dim_head=64, mlp_mult=4), 64, (56, 56), {}),
    "cvt stage 2": (lambda: cvt.Transformer(192, 3, 2, 2, heads=3, dim_head=64, mlp_mult=4), 192, (28, 28), {}),
    "mobile_vit xs stage 1": (lambda: mobile_vit.Transformer(96, 2, 4, 8, 192), 96, (32, 32), dict(groups=(2, 2))),
    "mobile_vit xs stage 2": (lambda: mobile_vit.Transformer(120, 4, 4, 8, 240), 120, (16, 16), dict(groups=(2, 2))),
    "scalable_vit s stage 1": (lambda: _scalable(64, 2, 40, 8, 64), 64, (64, 64), {}),
    "scalable_vit s stage 2": (lambda: _scalable(128, 4, 40, 4, 32), 128, (32, 32), {}),
    "scalable_vit s stage 4": (lambda: _scalable(512, 16, 32, 1, None), 512, (8, 8), {}),
    "sep_vit stage 1": (lambda: sep_vit.Transformer(32, 1, heads=1, norm_output=False), 32, (56, 56), {}),
    "sep_vit stage 2": (lambda: sep_vit.Transformer(64, 1, heads=2, norm_output=False), 64, (28, 28), {}),
    "sep_vit stage 4": (lambda: sep_vit.Transformer(256, 1, heads=8, norm_output=False), 256, (7, 7), {}),
    "regionvit stage 1": (lambda: regionvit.R2LTransformer(64, window_size=7, depth=2), 64, (56, 56),
                          dict(regions=(8, 8))),
    "regionvit stage 2": (lambda: regionvit.R2LTransformer(128, window_size=7, depth=2), 128, (28, 28),
                          dict(regions=(4, 4))),
    "regionvit one image 7x7 / 1x1": (lambda: regionvit.R2LTransformer(64, window_size=7, depth=2), 64, (7, 7),
                                      dict(regions=(1, 1), B=1)),
}


def _scalable(dim, heads, dk, r, window):
    return scalable_vit.Transformer(dim, 1, heads=heads, ssa_dim_key=dk, ssa_reduction_factor=r, iwsa_dim_key=dk,
                                    iwsa_window_size=window, norm_output=False)


def inputs(name):
    """(x, run_blocks' arguments): `B` images of the case's grid, then with `regions` their region maps."""
    _, D, (gh, gw), extra = CASES[name]
    kw = dict(dict(B=B, N=gh * gw, grid=(gh, gw)), **extra)
    rows = kw["B"] * gh * gw
    if "regions" in kw:
        rows += kw["B"] * kw["regions"][0] * kw["regions"][1]
    x = torch.randn(rows, D, device=DEV, generator=torch.Generator(device=DEV).manual_seed(gh * D))
    return x, kw


def run_traced(mod, x, kw, ln_mode):
    """(launches, the encoder's output stream): ScalableViT through Transformer.run_fused, the rest run_blocks."""
    if not isinstance(mod, scalable_vit.Transformer):
        return traced(mod, x, kw, ln_mode), x
    out = []
    launches = traced(mod, x, kw, ln_mode,
                      call=lambda: out.append(mod.run_fused(x, kw["B"], kw["grid"][0], kw["grid"][1])))
    return launches, out[0]


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", list(CASES))
def test_grid_layer_launches_trace_back_and_stay_within_bounds(name, ln_mode):
    mod = perturbed(CASES[name][0])
    x, kw = inputs(name)
    x0 = x.clone()
    with torch.no_grad():
        launches, _ = run_traced(mod, x, kw, ln_mode)
        n = LT.check_provenance(mod, x0, kw, launches, ln_mode, f"{name} | {ln_mode}")
        assert n == len(launches) > 0
        for kind, r in LT.check_accuracy(launches, f"{name} | {ln_mode}", rerun_plain=rerun_plain).items():
            WORST[(name, ln_mode, kind)] = max(WORST.get((name, ln_mode, kind), 0.0), r)


def _eager(name, mod, x0, kw):
    """The module's own fp32 forward over the same token map (the reference's operator sequence), as tokens."""
    (gh, gw), D = kw["grid"], x0.shape[1]
    fmap = x0.view(B, gh, gw, D).permute(0, 3, 1, 2)
    out = mod.block[1:](fmap) if isinstance(mod, MaxViTBlock) else mod.forward_eager(fmap) \
        if isinstance(mod, (scalable_vit.Transformer, sep_vit.Transformer)) else mod(fmap)
    return out.permute(0, 2, 3, 1).reshape(B * gh * gw, D)


# name: (case, plant(monkeypatch), what the failure must name)
GPU_DEFECTS = {
    "CvT BatchNorm folded with eps 1e-5 instead of the module's":
        ("cvt stage 1", _bn_default_eps, ("layer 0 convolutional projection", "operand wq")),
    "MaxViT block and grid windows swapped":
        ("max_vit stage 1", _dilated_swapped, ("layer 0 attention", "operand dilated")),
    "ScalableViT IWSA scale from the padded key width (48, not dim_key 40)":
        ("scalable_vit s stage 2", _iwsa_scale_padded, ("layer 1 attention", "operand scale")),
    "SepViT window-token LayerNorm at the default eps":
        ("sep_vit stage 2", _head_ln_default_eps, ("layer 0 window tokens", "operand eps")),
}


@pytest.mark.parametrize("defect", list(GPU_DEFECTS))
def test_planted_defect_is_named_on_the_real_kernels(defect, monkeypatch):
    name, plant, want = GPU_DEFECTS[defect]
    x0, kw = inputs(name)
    res = {}
    with torch.no_grad():
        for planted in (False, True):
            mod = perturbed(CASES[name][0])
            if planted:
                plant(monkeypatch)
            launches, got = run_traced(mod, x0.clone(), kw, "fold")
            want_out = _eager(name, mod, x0, kw)
            res[planted] = ((got - want_out).abs().max().item(), want_out.abs().max().item())
            if planted:
                with pytest.raises(AssertionError) as e:
                    LT.check_provenance(mod, x0, kw, launches, "fold", name)
                assert all(w in str(e.value) for w in want), str(e.value)
                monkeypatch.undo()
    (clean, scale), (bad, _) = res[False], res[True]
    verdict = "miss it" if bad < 3e-2 else "catch it" if clean < 3e-2 else \
        "not tell it from the run without it, which it fails too"
    print(f"\n{defect} ({name}): max |fused - eager fp32| over the encoder output {clean:.3e} without the defect, "
          f"{bad:.3e} with it (max |eager| {scale:.3e}); a 3e-2 max-abs criterion would {verdict}")
