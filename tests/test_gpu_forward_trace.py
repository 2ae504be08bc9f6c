"""-m gpu: the whole forwards of tests/test_forward_trace.py on the real kernels, traced from the pixels to the logits
(oracle/layer_trace.check_forward_provenance) at production-like shapes: 224 x 224 images in 16 x 16 patches, D 384 in
6 heads of 64, 3 inputs (images, N-d volumes, 1-D series, videos of 2 to 8 frames); NaViT over five resolutions, four
of them non-square.  Both LayerNorm modes, and both patch modes where the TMA patch embedding applies.

For each case every operand of every launch is what the reference module's forward defines (provenance), every output
is within its kernel's fp64 bound on the operands it received, and the worst |got - ref| / bound per (case, launch kind)
-- and of each operand the walk checks within a bound -- is printed at the end of the module, with each case's
max |fused - eager fp32| over the logits.  Every planted defect of tests/test_forward_trace.py is re-run through the
real kernels: the walk must name it; how far it moves the logits from the module's own fp32 forward is printed, not
asserted.  T2T-ViT's soft-split walk (tests/test_t2t_trace.py) runs on the real kernels too."""
import pytest
import torch

import test_forward_trace as F
import test_t2t_trace as T2T
from oracle import layer_trace as LT
from test_gpu_layer_trace import rerun_plain
from vit_pytorch_b200 import deepvit, na_vit, simple_flash_attn_vit, simple_vit, simple_vit_1d, simple_vit_3d
from vit_pytorch_b200 import simple_vit_with_patch_dropout, simple_vit_with_qk_norm, simple_vit_with_register_tokens
from vit_pytorch_b200 import vit, vit_for_small_dataset, vit_nd, vit_nd_rotary, vivit

pytestmark = pytest.mark.gpu
DEV = "cuda"
D, H, DH, MLP = 384, 6, 64, 1536
B = 3
WORST = {}
LOGITS = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst |got - ref| / bound per case, patch mode, LayerNorm mode and launch kind (walk: an operand the "
          "walk checks within a bound):")
    for key in sorted(WORST):
        print(f"  {' | '.join(key)}: {WORST[key]:.3f}")
    print("\nmax |fused - eager fp32| over the logits per case, patch mode and LayerNorm mode:")
    for key in sorted(LOGITS):
        print(f"  {' | '.join(key)}: {LOGITS[key]:.3e}")


def _kw(**extra):
    return dict(num_classes=1000, dim=D, depth=2, heads=H, dim_head=DH, mlp_dim=MLP, **extra)


def _video_kw(temporal_depth=1, **extra):
    kw = _kw(**extra)
    kw.pop("depth")
    return dict(kw, spatial_depth=2, temporal_depth=temporal_depth)


# name: (model, image (h, w) -- NaViT: the list of image sizes); the names of tests/test_forward_trace.py
CASES = {
    "vit cls": (lambda: vit.ViT(image_size=224, patch_size=16, pool="cls", **_kw()), (224, 224)),
    "vit mean": (lambda: vit.ViT(image_size=224, patch_size=16, pool="mean", **_kw()), (224, 224)),
    "vit patch 8": (lambda: vit.ViT(image_size=112, patch_size=8, pool="cls", **_kw()), (112, 112)),
    "simple_vit": (lambda: simple_vit.SimpleViT(image_size=224, patch_size=16, **_kw()), (224, 224)),
    "simple_vit register tokens": (lambda: simple_vit_with_register_tokens.SimpleViT(
        image_size=224, patch_size=16, num_register_tokens=4, **_kw()), (224, 224)),
    "simple_vit qk norm": (lambda: simple_vit_with_qk_norm.SimpleViT(image_size=224, patch_size=16, **_kw()),
                           (224, 224)),
    "simple_vit patch dropout (eval)": (lambda: simple_vit_with_patch_dropout.SimpleViT(
        image_size=224, patch_size=16, patch_dropout=0.5, **_kw()), (224, 224)),
    "simple_flash_attn_vit": (lambda: simple_flash_attn_vit.SimpleViT(image_size=224, patch_size=16, **_kw()),
                              (224, 160)),
    "vit small dataset (SPT)": (lambda: vit_for_small_dataset.ViT(image_size=224, patch_size=16, pool="cls", **_kw()),
                                (224, 224)),
    "vit small dataset mean": (lambda: vit_for_small_dataset.ViT(image_size=224, patch_size=16, pool="mean",
                                                                  **_kw()), (224, 224)),
    "deepvit": (lambda: deepvit.DeepViT(image_size=224, patch_size=16, pool="cls", **_kw()), (224, 224)),
    "navit": (lambda: na_vit.NaViT(image_size=224, patch_size=16, **_kw()),
              [(224, 224), (128, 224), (96, 160), (48, 80), (160, 96)]),
    "vit_nd 3-d cls": (lambda: vit_nd.ViTND(ndim=3, input_shape=(8, 112, 112), patch_size=(2, 16, 16), pool="cls",
                                            **_kw()), (8, 112, 112)),
    "vit_nd 2-d mean": (lambda: vit_nd.ViTND(ndim=2, input_shape=224, patch_size=16, pool="mean", **_kw()),
                        (224, 224)),
    "vit_nd_rotary 3-d": (lambda: vit_nd_rotary.ViTND(ndim=3, input_shape=(8, 112, 112), patch_size=(2, 16, 16),
                                                      **_kw()), (8, 112, 112)),
    "simple_vit_1d": (lambda: simple_vit_1d.SimpleViT(seq_len=3136, patch_size=16, **_kw()), (3136,)),
    "simple_vit_3d": (lambda: simple_vit_3d.SimpleViT(image_size=224, image_patch_size=16, frames=2,
                                                      frame_patch_size=1, **_kw()), (2, 224, 224)),
    "simple_vit_3d frame patch 2": (lambda: simple_vit_3d.SimpleViT(image_size=224, image_patch_size=16, frames=4,
                                                                    frame_patch_size=2, **_kw()), (4, 224, 224)),
    "vivit factorized encoder cls": (lambda: vivit.ViViT(image_size=224, image_patch_size=16, frames=8,
                                                         frame_patch_size=2, pool="cls", **_video_kw()),
                                     (8, 224, 224)),
    "vivit factorized encoder mean": (lambda: vivit.ViViT(image_size=224, image_patch_size=16, frames=4,
                                                          frame_patch_size=1, pool="mean", **_video_kw()),
                                      (4, 224, 224)),
    "vivit factorized self-attention cls": (lambda: vivit.ViViT(
        image_size=224, image_patch_size=16, frames=4, frame_patch_size=1, pool="cls",
        variant="factorized_self_attention", **_video_kw(temporal_depth=2)), (4, 224, 224)),
    "vivit factorized self-attention mean": (lambda: vivit.ViViT(
        image_size=224, image_patch_size=16, frames=8, frame_patch_size=2, pool="mean",
        variant="factorized_self_attention", **_video_kw(temporal_depth=2)), (8, 224, 224)),
}


def inputs(name):
    size = CASES[name][1]
    g = torch.Generator(device=DEV).manual_seed(len(name))
    if isinstance(size, list):
        return [torch.randn(3, h, w, device=DEV, generator=g).bfloat16() for h, w in size]
    return torch.randn(B, 3, *size, device=DEV, generator=g).bfloat16()


def run(name, ln_mode, patch_mode, mp):
    mp.setenv("B200VIT_PATCH_MODE", patch_mode)
    # the host prepares NaViT's pooling query with an fp32 matmul, which the walk bounds as fp32, not TF32
    mp.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    model = F.perturbed(CASES[name][0], device=DEV)
    img = inputs(name)
    launches, logits = F.trace(model, img, ln_mode, impl=LT.real_impl)
    torch.cuda.synchronize()
    return model, img, launches, logits


PARAMS = F.patch_modes(CASES)


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name,patch_mode", PARAMS, ids=[f"{n} | {m}" for n, m in PARAMS])
def test_forward_traces_back_and_stays_within_bounds(name, patch_mode, ln_mode, monkeypatch):
    with torch.no_grad():
        model, img, launches, logits = run(name, ln_mode, patch_mode, monkeypatch)
        case = f"{name} | {patch_mode} | {ln_mode}"
        ratios = {}
        assert LT.check_forward_provenance(model, img, launches, ln_mode, case, ratios) == len(launches) > 0
        kinds = {c.name for c in launches}
        assert ("patch_embed_tma" in kinds) == (patch_mode == "tma"), kinds
        worst = LT.check_accuracy(launches, case, rerun_plain=rerun_plain)
        worst.update({f"walk: {op}": r for op, r in ratios.items()})
        for kind, r in worst.items():
            key = (name, patch_mode, ln_mode, kind)
            WORST[key] = max(WORST.get(key, 0.0), r)
        assert torch.isfinite(logits.float()).all()
        LOGITS[(name, patch_mode, ln_mode)] = (logits.float() - F.eager(model, img)).abs().max().item()


@pytest.mark.parametrize("defect", list(F.DEFECTS))
def test_planted_defect_is_named_on_the_real_kernels(defect, monkeypatch):
    name, ln_mode, plant, want = F.DEFECTS[defect]
    mode = "tma"                          # the TMA embedding where it applies, else the patchify kernels
    diff = {}
    with torch.no_grad():
        for planted in (False, True):
            if planted:
                plant(monkeypatch)
            model, img, launches, logits = run(name, ln_mode, mode, monkeypatch)
            diff[planted] = (logits.float() - F.eager(model, img)).abs().max().item()
            if planted:
                with pytest.raises(LT.ProvenanceError) as e:
                    LT.check_forward_provenance(model, img, launches, ln_mode, name)
            else:
                assert LT.check_forward_provenance(model, img, launches, ln_mode, name) == len(launches)
    assert all(w in str(e.value) for w in want), str(e.value)
    print(f"\n{defect} ({name}, {ln_mode}): max |fused - eager fp32| over the logits {diff[False]:.3e} without the "
          f"defect, {diff[True]:.3e} with it")


@pytest.mark.parametrize("ln_mode", ["fold", "exact"])
@pytest.mark.parametrize("name", sorted(T2T.CASES))
def test_t2t_soft_splits_trace_back_on_the_real_kernels(name, ln_mode, monkeypatch):
    spec = T2T.CASES[name]
    with torch.no_grad():
        ref = T2T.FAMILY.build(spec).to(DEV)
        model = T2T.FAMILY.build(spec).bfloat16().to(DEV)
        img = T2T.FAMILY.input(spec).to(DEV)
        launches, logits = T2T.trace(model, img, ln_mode, monkeypatch, impl=LT.real_impl)
        torch.cuda.synchronize()
        case = f"t2t {name} | {ln_mode}"
        first_main = T2T.check_soft_splits(model, img, launches, case)
        assert first_main < len(launches) and launches[-1].name == "gemm"
        # the launches with an fp64 oracle here: every one but the soft splits' unfold and wide attention kernels
        known = [c for c in launches if c.name not in T2T.T2T_ENTRY_POINTS]
        for kind, r in LT.check_accuracy(known, case, rerun_plain=rerun_plain).items():
            key = (f"t2t {name}", "-", ln_mode, kind)
            WORST[key] = max(WORST.get(key, 0.0), r)
        d = (logits.float() - ref(img.float())).abs().max().item()
    assert d < 5e-2, (case, d)
