"""LeViT parity cases (reference levit.py), on the shared recipe of parity.py.  Its own rule: every BatchNorm's weight,
bias, running mean and running variance are perturbed (the zero-initialised to_out BatchNorm and the default
statistics would otherwise leave the folding untested) and the statistics rounded to bf16 like the parameters.  The
model with a distill head returns a tuple, which the shared single-logit outputs do not take: its case is DISTILL,
stored under the fixture's "distill" key by make_levit_golden.py."""
import torch

from parity import Family, round_buffers

SMALL = dict(num_classes=7, dim=(32, 48, 64), depth=1, heads=2, mlp_mult=2)
BATCH = 2
# constructor keywords (on top of SMALL unless `readme`); `input` = (height, width) of the image, `batch` its batch size.
# The comments give the grid F of each stage; a downsampling layer takes the stage's F x F keys and ceil(F / 2)^2
# queries.
LEVIT_CASES = {
    # the README config at 224: 14 -> 7 -> 4 (196 -> 49 and 49 -> 16 queries, an odd grid)
    "readme_224": dict(seed=501, readme=True, image_size=224, num_classes=1000, dim=(256, 384, 512), depth=4,
                       heads=(4, 6, 8), mlp_mult=2, input=(224, 224)),
    # 7 -> 4 -> 2, dim_key 16, dim_value 32, tuple depths and heads, mlp_mult 3
    "dk16_dv32_112": dict(seed=502, image_size=112, dim_key=16, dim_value=32, depth=(1, 2, 1), heads=(2, 3, 4),
                          mlp_mult=3, input=(112, 112)),
    # 24 -> 12 -> 6: 576 keys, batch 1
    "keys_576": dict(seed=503, image_size=384, input=(384, 384), batch=1),
    # four stages at 64: 4 -> 2 -> 1 -> 1 (one-token maps)
    "stages4_64": dict(seed=504, image_size=64, stages=4, dim=(32, 48, 64, 80), input=(64, 64)),
    # 4 -> 2 -> 1 with dim_key 64, dim_value 128
    "dk64_dv128": dict(seed=505, image_size=64, dim_key=64, dim_value=128, input=(64, 64), batch=3),
    # a 224 x 216 input into an image_size=224 model: the convolutions still give 14 x 14
    "input_224x216": dict(seed=506, image_size=224, input=(224, 216)),
}
# the model with a distill head: (out, distill); 4 -> 2 -> 1
DISTILL = dict(seed=507, image_size=64, num_distill_classes=5, input=(64, 64), batch=3)
# the seeded-init (unperturbed) comparison
INIT_SEED = 521
INIT_KWARGS = dict(SMALL, image_size=64, num_distill_classes=5)

_SPEC_KEYS = ("seed", "input", "batch", "readme")


def case_kwargs(spec: dict) -> dict:
    kw = {} if spec.get("readme") else dict(SMALL)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def input_shape(spec: dict) -> tuple:
    return (spec.get("batch", BATCH), 3, *spec["input"])


def perturb_batchnorms(model, g: torch.Generator, spec: dict) -> None:
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.add_(0.5 * torch.randn(m.weight.shape, generator=g))
            m.bias.add_(0.1 * torch.randn(m.bias.shape, generator=g))
            m.running_mean.add_(0.2 * torch.randn(m.running_mean.shape, generator=g))
            m.running_var.mul_(0.5 + torch.rand(m.running_var.shape, generator=g))
    round_buffers(model)


FAMILY = Family(
    name="levit", model="levit.LeViT", cases=LEVIT_CASES, case_kwargs=case_kwargs, input_shape=input_shape,
    init_seed=INIT_SEED, init={None: INIT_KWARGS}, after=perturb_batchnorms)
