"""MobileViT parity cases (reference mobile_vit.py), on the shared recipe of parity.py.  Its own rule, LeViT's: every
BatchNorm's weight, bias, running mean and running variance are perturbed (the default statistics would leave the
BatchNorm folds of every convolution untested) and the statistics rounded to bf16 like the parameters."""
from levit_spec import perturb_batchnorms
from parity import Family

SMALL = dict(num_classes=7, dims=(32, 40, 48), channels=[16, 16, 24, 24, 32, 32, 40, 40, 48, 48, 96], depths=(1, 1, 1))
BATCH = 2
# constructor keywords (on top of SMALL unless `readme`; image_size is the input's); `input` = (height, width) of the
# image, `batch` its batch size.  The comments give the maps of the three MobileViT blocks and the tokens per group.
MOBILE_VIT_CASES = {
    # the README mbvit_xs at 256, batch 1: 32 x 32, 16 x 16, 8 x 8 -> 256, 64 and 16 tokens per group
    "readme_xs_256": dict(seed=901, readme=True, dims=[96, 120, 144],
                          channels=[16, 32, 48, 48, 64, 64, 80, 80, 96, 96, 384], num_classes=1000, input=(256, 256),
                          batch=1),
    # XXS widths with expansion 2 (stem.0 adds its input): 16 x 16, 8 x 8, 4 x 4 -> 64, 16, 4
    "xxs_expansion2": dict(seed=902, dims=(64, 80, 96), channels=[16, 16, 24, 24, 48, 48, 64, 64, 80, 80, 320],
                           expansion=2, input=(128, 128)),
    # patch (1, 1): one group per map, 16 x 16, 8 x 8, 4 x 4 -> 256, 64, 16
    "patch11_whole_map": dict(seed=903, patch_size=(1, 1), input=(128, 128)),
    # patch (2, 4) on a 128 x 256 image, depths (1, 2, 1), batch 3: 16 x 32, 8 x 16, 4 x 8 -> 64, 16, 4
    "rect_patch_nonsquare": dict(seed=904, patch_size=(2, 4), depths=(1, 2, 1), input=(128, 256), batch=3),
    # expansion 1 (the depthwise-first MV2Block): 8 x 8, 4 x 4, 2 x 2 -> 16, 4, 1
    "expansion1": dict(seed=905, expansion=1, input=(64, 64)),
    # patch (1, 1) on a 100 x 68 image, maps rounded up by the strided convolutions: 13 x 9, 7 x 5, 4 x 3 -> 117, 35, 12
    "odd_input_patch11": dict(seed=906, patch_size=(1, 1), input=(100, 68)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 921
INIT_KWARGS = dict(SMALL, image_size=(64, 64), expansion=2)

_SPEC_KEYS = ("seed", "input", "batch", "readme")


def case_kwargs(spec: dict) -> dict:
    kw = {} if spec.get("readme") else dict(SMALL)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    kw["image_size"] = tuple(spec["input"])
    return kw


def input_shape(spec: dict) -> tuple:
    return (spec.get("batch", BATCH), 3, *spec["input"])


FAMILY = Family(
    name="mobile_vit", model="mobile_vit.MobileViT", cases=MOBILE_VIT_CASES, case_kwargs=case_kwargs,
    input_shape=input_shape, init_seed=INIT_SEED, init={None: INIT_KWARGS}, after=perturb_batchnorms)
