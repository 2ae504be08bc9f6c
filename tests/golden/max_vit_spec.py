"""MaxViT parity cases (reference max_vit.py), on the shared recipe of parity.py.  Its own rule, LeViT's: every
BatchNorm's weight, bias, running mean and running variance are perturbed (the default statistics would leave the
three BatchNorm folds of every MBConv untested) and the statistics rounded to bf16 like the parameters."""
from levit_spec import perturb_batchnorms
from parity import Family

SMALL = dict(num_classes=7, dim=32, depth=(1, 1), dim_head=32, window_size=2)
BATCH = 2
# constructor keywords (on top of SMALL unless `readme`); `input` = (height, width) of the image, `batch` its batch
# size.  The comments give the token map of every stage: the stem halves the image (rounding up), every stage's first
# MBConv halves the map again.
MAX_VIT_CASES = {
    # the README MaxViT-S at 224, dropout 0.1, batch 1: 56 x 56 -> 28 x 28 -> 14 x 14 -> 7 x 7, 7 x 7 windows
    "readme_224": dict(seed=601, readme=True, num_classes=1000, dim_conv_stem=64, dim=96, dim_head=32,
                       depth=(2, 2, 5, 2), window_size=7, mbconv_expansion_rate=4, mbconv_shrinkage_rate=0.25,
                       dropout=0.1, input=(224, 224), batch=1),
    # window 8 (full 64-row tiles), dim_head 64: 32 x 32 (4 x 4 windows, block and grid differ) -> 16 x 16 (2 x 2)
    "window8_dh64": dict(seed=602, dim=64, dim_head=64, window_size=8, depth=(2, 1), input=(128, 128)),
    # odd maps that the stride-2 convolutions round up, a non-square image, one channel, dim_conv_stem != dim, stage
    # depth 2: 53 x 109 -> stem 27 x 55 -> 14 x 28 (2 x 4 windows of 7) -> 7 x 14
    "odd_nonsquare_c1": dict(seed=603, window_size=7, dim_conv_stem=16, depth=(1, 2), channels=1, input=(53, 109)),
    # dim_head 128, window 3, non-default expansion and shrinkage rates (hidden 384, squeeze 192): 12 x 12 -> 6 x 6
    "dh128_w3_rates": dict(seed=604, dim=128, dim_head=128, window_size=3, depth=(1, 2), mbconv_expansion_rate=3,
                           mbconv_shrinkage_rate=0.5, input=(48, 48)),
    # three stages at window 2, dim_conv_stem 24: 16 x 16 -> 8 x 8 -> 4 x 4, batch 3
    "w2_three_stages": dict(seed=605, dim_conv_stem=24, depth=(1, 1, 1), input=(64, 64), batch=3),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 621
INIT_KWARGS = dict(SMALL, depth=(2, 1), dim_conv_stem=16)

_SPEC_KEYS = ("seed", "input", "batch", "readme")


def case_kwargs(spec: dict) -> dict:
    kw = {} if spec.get("readme") else dict(SMALL)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def input_shape(spec: dict) -> tuple:
    return (spec.get("batch", BATCH), spec.get("channels", 3), *spec["input"])


FAMILY = Family(
    name="max_vit", model="max_vit.MaxViT", cases=MAX_VIT_CASES, case_kwargs=case_kwargs, input_shape=input_shape,
    init_seed=INIT_SEED, init={None: INIT_KWARGS}, after=perturb_batchnorms)
