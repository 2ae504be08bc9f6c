"""RegionViT parity cases (reference regionvit.py), on the shared recipe of parity.py.  Every R2LTransformer of the
reference is built without `heads` or `dim_head` (regionvit.py:255), so every stage attends with 4 heads of 32.
ChanLayerNorm's `g` and `b` are 4-D, so the 1-D rules of parity.py skip them: `extra` perturbs them, or the affine of
the 3-conv local tokenizer would go untested.  The relative-position bias tables are Embedding weights (2-D) and keep
their N(0, 1) init."""
import torch

from parity import Family

BATCH = 2
# constructor keywords; `input` = (height, width) of the image, `batch` its batch size.  The comments give every
# stage's local map / region map (window = local / region).
REGIONVIT_CASES = {
    # the README config at 224, batch 1: 56 / 8, 28 / 4, 14 / 2, 7 / 1 -> 7 x 7 windows
    "readme_224": dict(seed=1101, dim=(64, 128, 256, 512), depth=(2, 2, 8, 2), window_size=7, num_classes=1000,
                       tokenize_local_3_conv=False, use_peg=False, input=(224, 224), batch=1),
    # window_size 14 at 224: 56 / 4, 28 / 2, 14 / 1, 7 / 1 -> windows 14, 14, 14, 7 (197-token windows)
    "window14_224": dict(seed=1102, dim=(32, 64, 64, 96), depth=(1, 1, 1, 1), window_size=14, num_classes=10,
                         input=(224, 224)),
    # the 3-conv local tokenizer and the PEGs at 112, batch 3: 28 / 4, 14 / 2, 7 / 1, 4 / 1 -> windows 7, 7, 7, 4
    "three_conv_peg_112": dict(seed=1103, dim=(32, 64, 64, 128), depth=(1, 2, 1, 1), num_classes=7,
                               tokenize_local_3_conv=True, use_peg=True, input=(112, 112), batch=3),
    # non-square 224 x 112: 56 x 28 / 8 x 4, ..., 7 x 4 / 1 x 1 -> the last window 7 x 4
    "nonsquare_224x112": dict(seed=1104, dim=(32, 32, 64, 64), depth=(1, 1, 1, 2), num_classes=5,
                              input=(224, 112)),
    # 56 x 56: 14 / 2, 7 / 1, 4 / 1, 2 / 1 -> windows 7, 7, 4, 2, a 1 x 1 region map from stage 2 on
    "small_56": dict(seed=1105, dim=(32, 64, 64, 96), depth=(1, 1, 2, 1), num_classes=6, input=(56, 56)),
    # an int dim and depth: every stage 64 wide, one layer each
    "int_dim": dict(seed=1106, dim=64, depth=1, num_classes=4, input=(112, 112)),
    # dropout > 0 in eval mode: the same logits
    "dropout_eval": dict(seed=1107, dim=(32, 64, 64, 96), depth=(1, 1, 1, 1), num_classes=3, attn_dropout=0.2,
                         ff_dropout=0.1, input=(112, 112)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 1121
INIT_KWARGS = dict(dim=(32, 64, 64, 96), depth=(1, 2, 1, 1), num_classes=10, tokenize_local_3_conv=True, use_peg=True)

_SPEC_KEYS = ("seed", "input", "batch")


def case_kwargs(spec: dict) -> dict:
    return {k: v for k, v in spec.items() if k not in _SPEC_KEYS}


def input_shape(spec: dict) -> tuple:
    return (spec.get("batch", BATCH), 3, *spec["input"])


def perturb_channel_norms(name, p, g, spec) -> None:
    if p.dim() == 4 and p.shape[0] == 1 and name.endswith((".g", ".b")):
        p.add_(torch.randn(p.shape, generator=g) * (0.1 if name.endswith(".g") else 0.05))


FAMILY = Family(
    name="regionvit", model="regionvit.RegionViT", cases=REGIONVIT_CASES, case_kwargs=case_kwargs,
    input_shape=input_shape, init_seed=INIT_SEED, init={None: INIT_KWARGS}, extra=perturb_channel_norms)
