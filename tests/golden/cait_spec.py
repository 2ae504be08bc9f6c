"""CaiT parity cases (reference cait.py), on the shared recipe of parity.py.  Its own rules: the LayerScale vectors
are scaled by 1 + 0.5 N(0, 1), each layer's mixing matrices get `mix` times N(0, 1) noise, and layer dropout is seeded
right before every forward."""
import torch

from parity import Family, seed_layer_dropout

BASE = dict(num_classes=7, dim=64, depth=2, cls_depth=2, heads=4, mlp_dim=96, dim_head=32, dropout=0.,
            emb_dropout=0., layer_dropout=0.)
BATCH = 2
# constructor keywords on top of BASE; `input` = side of the square image fed to it; `mix` = scale of the noise added to
# every layer's two mixing matrices (0: the reference's own N(0, 1) init); `pre_sign` = -1 makes every pre-softmax
# weight negative; `drop_seed` = the torch / random seed set right before the forward (layer dropout draws from both)
README = dict(image_size=256, patch_size=32, num_classes=1000, dim=1024, depth=12, cls_depth=2, heads=16, mlp_dim=2048,
              dim_head=64, dropout=0.1, emb_dropout=0.1, input=256, mix=0.0)
CAIT_CASES = {
    # the README config (256 / 32, dim 1024, depth 12 + 2, 16 x 64 heads): 64 patches, reference init of the mixing
    "readme": dict(README, seed=91, layer_dropout=0.0),
    # the same with layer dropout: a seeded subset of the 12 + 2 layers runs
    "readme_layer_dropout": dict(README, seed=92, layer_dropout=0.25, drop_seed=7),
    "dh32_n64": dict(seed=93, image_size=32, patch_size=4, input=32, mix=0.5),
    # CaiT's paper head width (three 16-wide slabs), 196 patches
    "dh48_n196": dict(seed=94, image_size=56, patch_size=4, heads=6, dim_head=48, input=56, mix=0.5),
    "dh80": dict(seed=95, image_size=32, patch_size=8, heads=3, dim_head=80, input=32, mix=0.5),
    "dh128": dict(seed=96, image_size=32, patch_size=8, heads=2, dim_head=128, input=32, mix=0.5),
    # 576 patches: 36 key blocks, one CTA of output heads per row tile
    "n576_h8": dict(seed=97, image_size=96, patch_size=4, heads=8, dim_head=32, input=96, mix=0.5),
    # 224 / 16: 196 patches, 16 heads
    "p16_h16": dict(seed=98, image_size=224, patch_size=16, heads=16, dim_head=32, dim=96, input=224, mix=0.5),
    # one head: a negative pre weight turns the softmax around (the most negative score gets the most weight)
    "heads1_negative_pre": dict(seed=99, image_size=32, patch_size=4, heads=1, dim_head=64, input=32, mix=0.5,
                                pre_sign=-1),
    # image size equal to the patch size: one patch
    "one_patch": dict(seed=100, image_size=8, patch_size=8, input=8, mix=0.5),
    # an image smaller than the constructed one: the first n rows of the positional table
    "smaller_input": dict(seed=101, image_size=64, patch_size=8, input=32, mix=0.5),
    "depth1_cls1": dict(seed=102, image_size=32, patch_size=4, depth=1, cls_depth=1, input=32, mix=0.5),
}
# the seeded-init (unperturbed) comparison; depth 20 puts layers 19 and 20 on LayerScale's 1e-5 branch
INIT_SEED = 123
INIT_KWARGS = dict(image_size=32, patch_size=8, **{**BASE, "depth": 20})

_SPEC_KEYS = ("seed", "input", "mix", "pre_sign", "drop_seed")


def case_kwargs(spec: dict) -> dict:
    kw = dict(BASE)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def extra(n, p, g, spec) -> None:
    if n.endswith(".scale"):                                    # LayerScale [1, 1, dim]
        p.mul_(1 + 0.5 * torch.randn(p.shape, generator=g))
    elif n.endswith("mix_heads_pre_attn") or n.endswith("mix_heads_post_attn"):
        p.add_(spec["mix"] * torch.randn(p.shape, generator=g))
        if n.endswith("mix_heads_pre_attn") and spec.get("pre_sign", 1) < 0:
            p.copy_(-p.abs())


FAMILY = Family(
    name="cait", model="cait.CaiT", cases=CAIT_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (BATCH, 3, spec["input"], spec["input"]),
    init_seed=INIT_SEED, init={None: INIT_KWARGS}, extra=extra, before_forward=seed_layer_dropout)
