"""vit_for_small_dataset parity cases (reference vit_for_small_dataset.py), on the shared recipe of parity.py.  Its own
rule: every layer's `temperature` moves by a different amount per layer, since its default is exactly
log(dim_head ** -0.5) and a path that ignored it would match."""
from parity import Family

BASE = dict(num_classes=7, dim=64, depth=2, heads=2, dim_head=32, mlp_dim=96)
BATCH = 3
# image_size / patch_size / channels of the constructor; `input` = (height, width) of the image fed to it
VIT_SMALL_CASES = {
    # CIFAR geometry: K = 5*3*4*4 = 240, padded to 256 on the fused path
    "c32_p4_cls": dict(seed=61, image_size=32, patch_size=4, channels=3, pool="cls", input=(32, 32)),
    "c32_p4_mean": dict(seed=62, image_size=32, patch_size=4, channels=3, pool="mean", input=(32, 32)),
    "nonsquare_24x32": dict(seed=63, image_size=(24, 32), patch_size=4, channels=3, pool="cls", input=(24, 32)),
    "c1_p8": dict(seed=64, image_size=32, patch_size=8, channels=1, pool="mean", input=(32, 32)),
    "p16_k3840": dict(seed=65, image_size=32, patch_size=16, channels=3, pool="cls", input=(32, 32)),
    "dh64": dict(seed=66, image_size=32, patch_size=4, channels=3, pool="cls", input=(32, 32), dim_head=64),
    "dh80": dict(seed=67, image_size=32, patch_size=8, channels=3, pool="mean", input=(32, 32), dim_head=80),
    "dh128": dict(seed=68, image_size=32, patch_size=8, channels=3, pool="cls", input=(32, 32), dim_head=128),
    # 24 x 24 patches + cls = 577 tokens: the self-masked key-block (varlen) attention
    "long_577": dict(seed=69, image_size=96, patch_size=4, channels=3, pool="mean", input=(96, 96), depth=1),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 123
INIT_KWARGS = dict(image_size=32, patch_size=4, channels=3, **BASE)


def case_kwargs(spec: dict) -> dict:
    kw = dict(BASE)
    for k in ("dim_head", "depth"):
        if k in spec:
            kw[k] = spec[k]
    return dict(image_size=spec["image_size"], patch_size=spec["patch_size"], channels=spec["channels"],
                pool=spec["pool"], **kw)


def after(model, g, spec) -> None:
    for i, layer in enumerate(model.transformer.layers):
        layer[0].temperature.add_(0.3 * (i + 1) * (-1) ** i)


FAMILY = Family(
    name="vit_small", model="vit_for_small_dataset.ViT", cases=VIT_SMALL_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (BATCH, spec["channels"], *spec["input"]),
    init_seed=INIT_SEED, init={pool: dict(INIT_KWARGS, pool=pool) for pool in ("cls", "mean")}, after=after)
