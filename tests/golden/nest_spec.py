"""NesT parity cases (reference nest.py), on the shared recipe of parity.py.  Every level attends inside blocks of the
map with heads dim // heads wide (`dim_head` is accepted and ignored, nest.py:121-125, 43-44); one case passes it to
pin that.  The LayerNorm's `g` and `b` are 4-D, so the 1-D rules of parity.py skip them: `extra` perturbs them, or the
affines of every level entry and of the head would go untested.  `pos_emb` keeps its N(0, 1) init."""
import torch

from parity import Family

BATCH = 2
# constructor keywords; `input` = (height, width) of the image, `batch` its batch size.  The comments give every
# level's map, its blocks and their tokens.
NEST_CASES = {
    # the README config at 224, batch 1: 56 x 56 (4 x 4 blocks), 28 x 28 (2 x 2), 14 x 14 (1): 196-token blocks
    "readme_224": dict(seed=1101, image_size=224, patch_size=4, dim=96, heads=3, num_hierarchies=3,
                       block_repeats=(2, 2, 8), num_classes=1000, input=(224, 224), batch=1),
    # four hierarchies at 224: 56 x 56 (8 x 8 blocks), 28 x 28 (4 x 4), 14 x 14 (2 x 2), 7 x 7: 49-token blocks
    "hier4_224": dict(seed=1102, image_size=224, patch_size=4, dim=32, heads=1, num_hierarchies=4,
                      block_repeats=(1, 1, 1, 1), num_classes=10, input=(224, 224), batch=1),
    # 32 x 32, patch 4: 8 x 8 (4 x 4 blocks), 4 x 4 (2 x 2), 2 x 2: 4-token blocks
    "tiny_32": dict(seed=1103, image_size=32, patch_size=4, dim=32, heads=1, num_hierarchies=3,
                    block_repeats=(1, 1, 2), num_classes=5, input=(32, 32)),
    # one level, no Aggregate: 8 x 8 in one block of 64 tokens
    "one_level": dict(seed=1104, image_size=32, patch_size=4, dim=64, heads=2, num_hierarchies=1, block_repeats=2,
                      num_classes=7, input=(32, 32)),
    # heads 64 wide (dim 128, heads 2): 16 x 16 (4 x 4 blocks), 8 x 8 (2 x 2), 4 x 4: 16-token blocks
    "dim_head_64": dict(seed=1105, image_size=64, patch_size=4, dim=128, heads=2, num_hierarchies=3,
                        block_repeats=(1, 1, 1), num_classes=6, input=(64, 64)),
    # an int block_repeats and mlp_mult 2: two layers at every level
    "int_repeats_mlp2": dict(seed=1106, image_size=64, patch_size=4, dim=32, heads=1, num_hierarchies=3,
                             block_repeats=2, mlp_mult=2, num_classes=4, input=(64, 64)),
    # non-square 224 x 112: 56 x 28 (4 x 4 blocks), 28 x 14 (2 x 2), 14 x 7: 98-token blocks
    "nonsquare_224x112": dict(seed=1107, image_size=224, patch_size=4, dim=32, heads=1, num_hierarchies=3,
                              block_repeats=(1, 1, 1), num_classes=5, input=(224, 112), batch=1),
    # a 112 input to a model built for 224: 28 x 28 (4 x 4 blocks of 49 tokens, the first 49 of 196 positions)
    "smaller_input": dict(seed=1108, image_size=224, patch_size=4, dim=32, heads=1, num_hierarchies=3,
                          block_repeats=(1, 1, 1), num_classes=5, input=(112, 112)),
    # dim_head given, and ignored: heads of 64 // 2 = 32; 16 x 16 (2 x 2 blocks), 8 x 8
    "ignored_dim_head": dict(seed=1109, image_size=64, patch_size=4, dim=64, heads=2, num_hierarchies=2,
                             block_repeats=(1, 2), dim_head=16, num_classes=3, input=(64, 64)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 1121
INIT_KWARGS = dict(image_size=64, patch_size=4, dim=32, heads=1, num_hierarchies=3, block_repeats=(1, 1, 2),
                   num_classes=10)

_SPEC_KEYS = ("seed", "input", "batch")


def case_kwargs(spec: dict) -> dict:
    return {k: v for k, v in spec.items() if k not in _SPEC_KEYS}


def input_shape(spec: dict) -> tuple:
    return (spec.get("batch", BATCH), 3, *spec["input"])


def perturb_layer_norms(name, p, g, spec) -> None:
    if p.dim() == 4 and p.shape[0] == 1 and name.endswith((".g", ".b")):
        p.add_(torch.randn(p.shape, generator=g) * (0.1 if name.endswith(".g") else 0.05))


FAMILY = Family(
    name="nest", model="nest.NesT", cases=NEST_CASES, case_kwargs=case_kwargs, input_shape=input_shape,
    init_seed=INIT_SEED, init={None: INIT_KWARGS}, extra=perturb_layer_norms)
