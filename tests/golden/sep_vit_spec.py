"""SepViT parity cases (reference sep_vit.py), on the shared recipe of parity.py.  The reference's SepViT passes
neither `window_size` nor `dim_head` to its DSSA layers (sep_vit.py:224, 274): every DSSA attends inside 7 x 7
windows with heads 32 wide, so a stage's map must be a multiple of 7 and the keywords are accepted and ignored; one
case passes both to pin that.  The window token is the one parameter the 1-D rules of parity.py skip (its name ends in
neither `weight` nor `bias`); it keeps its N(0, 1) init."""
from parity import Family

BATCH = 2
# constructor keywords (dim, depth, heads and num_classes given per case); `input` = (height, width) of the image,
# `batch` its batch size.  The comments give every stage's map and its number of 7 x 7 windows.
SEP_VIT_CASES = {
    # the README config at 224, batch 1: 56 x 56, 28 x 28, 14 x 14, 7 x 7 -> 64, 16, 4, 1 windows
    "readme_224": dict(seed=1001, num_classes=1000, dim=32, dim_head=32, heads=(1, 2, 4, 8), depth=(1, 2, 6, 2),
                       window_size=7, input=(224, 224), batch=1),
    # non-square, three stages: 56 x 28, 28 x 14, 14 x 7 -> 32, 8, 2 windows
    "nonsquare_224x112": dict(seed=1002, num_classes=10, dim=32, heads=(1, 2, 4), depth=(1, 1, 1),
                              input=(224, 112)),
    # two stages at batch 3: 28 x 28, 14 x 14 -> 16, 4 windows; two heads of 32 in stage 1
    "two_stage_batch3": dict(seed=1003, num_classes=5, dim=64, heads=(2, 4), depth=(2, 1), input=(112, 112),
                             batch=3),
    # two stages ending in one window: 14 x 14, 7 x 7 -> 4, 1 windows
    "single_window_last": dict(seed=1004, num_classes=6, dim=48, heads=(1, 3), depth=(1, 2), ff_mult=2,
                               input=(56, 56)),
    # window_size and dim_head given, and ignored as by the reference: 28 x 56, 14 x 28 -> 8, 2 windows
    "ignored_window_and_dim_head": dict(seed=1005, num_classes=4, dim=32, heads=(1, 2), depth=(1, 1),
                                        window_size=(4, 2), dim_head=64, input=(112, 224)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 1021
INIT_KWARGS = dict(num_classes=10, dim=32, heads=(1, 2), depth=(1, 2), window_size=7)

_SPEC_KEYS = ("seed", "input", "batch")


def case_kwargs(spec: dict) -> dict:
    return {k: v for k, v in spec.items() if k not in _SPEC_KEYS}


def input_shape(spec: dict) -> tuple:
    return (spec.get("batch", BATCH), 3, *spec["input"])


FAMILY = Family(
    name="sep_vit", model="sep_vit.SepViT", cases=SEP_VIT_CASES, case_kwargs=case_kwargs, input_shape=input_shape,
    init_seed=INIT_SEED, init={None: INIT_KWARGS})
