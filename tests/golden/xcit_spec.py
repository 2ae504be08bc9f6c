"""XCiT parity cases (reference xcit.py), on the shared recipe of parity.py.  Its own rules: the LayerScale vectors
are scaled by 1 + 0.5 N(0, 1), every temperature gets `tau` plus N(0, 0.3), the BatchNorm running statistics are
perturbed and rounded to bf16 like the parameters, and layer dropout is seeded right before every forward."""
import torch

from parity import Family, round_buffers, seed_layer_dropout

BASE = dict(num_classes=7, dim=64, depth=2, cls_depth=2, heads=4, mlp_dim=96, dim_head=32, dropout=0.,
            emb_dropout=0., local_patch_kernel_size=3, layer_dropout=0.)
BATCH = 2
# constructor keywords on top of BASE; `input` = (height, width) of the image fed to it; `tau` = value added to every
# temperature parameter before its N(0, 0.3) noise (tau = temperature.exp(): 3.0 makes the channel softmax peaky);
# `drop_seed` = the torch / random seed set right before the forward (layer dropout draws from both)
README = dict(image_size=256, patch_size=32, num_classes=1000, dim=1024, depth=12, cls_depth=2, heads=16, mlp_dim=2048,
              dim_head=64, dropout=0.1, emb_dropout=0.1, local_patch_kernel_size=3, input=(256, 256))
XCIT_CASES = {
    # the README config (256 / 32, dim 1024, depth 12 + 2, 16 x 64 heads): an 8 x 8 grid
    "readme": dict(README, seed=201, layer_dropout=0.0),
    # the same with the README's layer dropout raised so that a seeded subset of the 12 + 2 layers runs
    "readme_layer_dropout": dict(README, seed=202, layer_dropout=0.25, drop_seed=7),
    "dh32": dict(seed=203, image_size=32, patch_size=4, input=(32, 32)),
    # the paper's head width (XCiT-T/S/L), 196 tokens
    "dh48_n196": dict(seed=204, image_size=56, patch_size=4, heads=6, dim_head=48, dim=96, input=(56, 56)),
    "dh80": dict(seed=205, image_size=32, patch_size=8, heads=3, dim_head=80, input=(32, 32)),
    "dh128": dict(seed=206, image_size=32, patch_size=8, heads=2, dim_head=128, input=(32, 32)),
    # large temperatures: tau near 20, a peaky softmax over the channels
    "peaky_tau": dict(seed=207, image_size=32, patch_size=4, input=(32, 32), tau=3.0),
    # a 6 x 8 grid: rows and columns differ, so a transposed grid would fail
    "nonsquare_6x8": dict(seed=208, image_size=64, patch_size=8, input=(48, 64)),
    # an image smaller than the constructed one: the first n rows of the positional table
    "smaller_input": dict(seed=209, image_size=64, patch_size=8, input=(32, 32)),
    # one patch: every tap of both convolutions but the centre one falls on padding
    "one_patch": dict(seed=210, image_size=8, patch_size=8, input=(8, 8)),
    # a 1 x 7 strip: every token is a border token vertically
    "strip_1x7": dict(seed=211, image_size=56, patch_size=8, input=(8, 56)),
    "kernel1": dict(seed=212, image_size=32, patch_size=4, input=(32, 32), local_patch_kernel_size=1),
    "kernel5": dict(seed=213, image_size=32, patch_size=4, input=(32, 32), local_patch_kernel_size=5),
    "kernel7_2x2": dict(seed=214, image_size=16, patch_size=8, input=(16, 16), local_patch_kernel_size=7),
    "kernel7": dict(seed=215, image_size=48, patch_size=4, input=(48, 48), local_patch_kernel_size=7),
    # 28 x 28 = 784 tokens: the channel attention streams several token tiles with a ragged tail
    "grid28": dict(seed=216, image_size=112, patch_size=4, heads=2, dim_head=48, dim=96, input=(112, 112)),
    "depth1_cls1": dict(seed=217, image_size=32, patch_size=4, depth=1, cls_depth=1, input=(32, 32)),
}
# the seeded-init (unperturbed) comparison; depth 20 puts layers 19 and 20 on LayerScale's 1e-6 branch
INIT_SEED = 321
INIT_KWARGS = dict(image_size=32, patch_size=8, **{**BASE, "depth": 20})

_SPEC_KEYS = ("seed", "input", "tau", "drop_seed")


def case_kwargs(spec: dict) -> dict:
    kw = dict(BASE)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def extra(n, p, g, spec) -> None:
    if n.endswith(".scale"):                                    # LayerScale (dim,)
        p.mul_(1 + 0.5 * torch.randn(p.shape, generator=g))
    elif n.endswith("temperature"):
        p.add_(spec.get("tau", 0.0) + 0.3 * torch.randn(p.shape, generator=g))


def after(model, g, spec) -> None:
    for n, b in model.named_buffers():
        if n.endswith("running_mean"):
            b.add_(0.2 * torch.randn(b.shape, generator=g))
        elif n.endswith("running_var"):
            b.mul_(0.5 + torch.rand(b.shape, generator=g))
    round_buffers(model)


FAMILY = Family(
    name="xcit", model="xcit.XCiT", cases=XCIT_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (BATCH, 3, *spec["input"]),
    init_seed=INIT_SEED, init={None: INIT_KWARGS}, extra=extra, after=after, before_forward=seed_layer_dropout)
