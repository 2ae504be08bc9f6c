"""PiT parity cases (reference pit.py), on the shared recipe of parity.py."""
from parity import Family

BASE = dict(num_classes=7, dim=32, depth=(1, 1), heads=2, mlp_dim=64, dim_head=32, dropout=0., emb_dropout=0.,
            channels=3)
BATCH = 2
# constructor keywords on top of BASE; `input` = (height, width) of the image fed to it.  The comments give the token
# grid of every stage (unfold grid, then what each Pool makes of it).
README = dict(image_size=224, patch_size=14, num_classes=1000, dim=256, depth=(3, 3, 3), heads=16, mlp_dim=2048,
              dim_head=64, dropout=0.1, emb_dropout=0.1, input=(224, 224))
PIT_CASES = {
    # the README config: 31 x 31 (961 patches + cls: the key-block attention) -> 16 x 16 -> 8 x 8
    "readme": dict(README, seed=301),
    # one head count per stage: 9 x 9 -> 5 x 5 -> 3 x 3
    "heads_tuple": dict(seed=302, image_size=40, patch_size=8, depth=(1, 2, 1), heads=(1, 2, 4), input=(40, 40)),
    # a single stage, no Pool
    "single_stage": dict(seed=303, image_size=32, patch_size=8, depth=(2,), input=(32, 32)),
    # an odd patch size (stride 3) and four channels: 8 x 8 -> 4 x 4
    "p7_c4": dict(seed=304, image_size=28, patch_size=7, channels=4, input=(28, 28)),
    # p 2 (stride 1): an odd 7 x 7 grid -> 4 x 4
    "p2_odd_grid": dict(seed=305, image_size=8, patch_size=2, input=(8, 8)),
    # 30 x 30 with p 8 (stride 4): the last 2 pixel rows and columns fill no stride step; 6 x 6 -> 3 x 3
    "trailing_pixels": dict(seed=306, image_size=32, patch_size=8, input=(30, 30)),
    # an image smaller than the constructed one: the first n + 1 rows of the positional table; 7 x 7 -> 4 x 4
    "smaller_input": dict(seed=307, image_size=64, patch_size=8, input=(32, 32)),
    # one patch: 1 x 1 -> 1 x 1 -> 1 x 1 (every tap but the centre one falls on padding)
    "one_patch": dict(seed=308, image_size=8, patch_size=8, depth=(1, 1, 1), input=(8, 8)),
    # 2 x 2 -> 1 x 1
    "grid_2x2": dict(seed=309, image_size=8, patch_size=4, input=(6, 6)),
    # a 4 x 16 unfold grid: the reference's Pool reads its 64 tokens as 8 x 8 (int(sqrt(n))), then 4 x 4
    "isqrt_4x16": dict(seed=310, image_size=36, patch_size=4, input=(10, 34)),
    "dh80": dict(seed=311, image_size=16, patch_size=4, heads=(2, 1), dim_head=80, input=(16, 16)),
    "dh128": dict(seed=312, image_size=16, patch_size=4, heads=1, dim_head=128, input=(16, 16)),
    # heads 1 and dim_head == dim in the first stage: its to_out is the identity; the second stage (dim 64) projects
    "identity_out": dict(seed=313, image_size=16, patch_size=4, heads=(1, 2), dim_head=32, input=(16, 16)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 321
INIT_KWARGS = dict(image_size=32, patch_size=8, **{**BASE, "depth": (2, 1, 1), "heads": (2, 2, 4)})

_SPEC_KEYS = ("seed", "input")


def case_kwargs(spec: dict) -> dict:
    kw = dict(BASE)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


FAMILY = Family(
    name="pit", model="pit.PiT", cases=PIT_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (BATCH, case_kwargs(spec)["channels"], *spec["input"]),
    init_seed=INIT_SEED, init={None: INIT_KWARGS})
