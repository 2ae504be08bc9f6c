"""CrossFormer parity cases (reference crossformer.py), on the shared recipe of parity.py.  Its own rule: the channel
LayerNorms' 4-D affines `g` / `b` (shape (1, dim, 1, 1)), which the 1-D rules skip, get the same perturbations as a
1-D weight and bias, so the folded LayerNorms are exercised."""
import torch

from parity import Family

SMALL = dict(num_classes=7, dim=(64, 64, 96, 128), depth=(1, 1, 1, 1), local_window_size=2)
BATCH = 2
# constructor keywords (on top of SMALL unless `readme`); `input` = (height, width) of the image, `batch` its batch
# size.  The comments give the stage maps and the stage-1 scale widths.
CROSSFORMER_CASES = {
    # the README CrossFormer at 224, batch 1: 56 x 56 -> 28 x 28 -> 14 x 14 -> 7 x 7; stem scales 32 / 16 / 8 / 8
    "readme_224": dict(seed=801, readme=True, num_classes=1000, dim=(64, 128, 256, 512), depth=(2, 2, 8, 2),
                       global_window_size=(8, 4, 2, 1), local_window_size=7, input=(224, 224), batch=1),
    # 16 x 16 -> 8 x 8 -> 4 x 4 -> 2 x 2; a 3-head stage (dim 96)
    "small_64": dict(seed=802, global_window_size=(4, 2, 2, 1), input=(64, 64)),
    # one channel, a 16 x 32 map under window 8, then 8 x 16, 4 x 8, 2 x 4; 1-token windows at the end, batch 3
    "nonsquare_c1": dict(seed=803, global_window_size=(8, 4, 2, 1), channels=1, input=(64, 128), batch=3),
    # inner width < dim (dim 80: 2 heads of 32), stage widths 40 / 56 / 72 at the later scales
    "inner_lt_dim": dict(seed=804, dim=(64, 80, 112, 144), global_window_size=(4, 2, 2, 1), input=(64, 64)),
    # three stem scales (widths 32 / 16 / 16), strides 2: 16 x 16 -> 8 x 8 -> 4 x 4 -> 2 x 2, full 64-token windows
    "three_scale_s2_w8": dict(seed=805, cross_embed_kernel_sizes=((2, 4, 8), (2, 4), (2, 4), (2, 4)),
                              cross_embed_strides=(2, 2, 2, 2), local_window_size=(8, 8, 4, 2),
                              global_window_size=(2, 1, 1, 1), input=(32, 32)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 821
INIT_KWARGS = dict(SMALL, depth=(1, 2, 1, 1))

_SPEC_KEYS = ("seed", "input", "batch", "readme")


def case_kwargs(spec: dict) -> dict:
    kw = {} if spec.get("readme") else dict(SMALL)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def input_shape(spec: dict) -> tuple:
    return (spec.get("batch", BATCH), spec.get("channels", 3), *spec["input"])


def perturb_channel_norms(name, p, g, spec) -> None:
    if p.dim() == 4 and p.shape[0] == 1 and name.endswith((".g", ".b")):
        p.add_(torch.randn(p.shape, generator=g) * (0.1 if name.endswith(".g") else 0.05))


FAMILY = Family(
    name="crossformer", model="crossformer.CrossFormer", cases=CROSSFORMER_CASES, case_kwargs=case_kwargs,
    input_shape=input_shape, init_seed=INIT_SEED, init={None: INIT_KWARGS}, extra=perturb_channel_norms)
