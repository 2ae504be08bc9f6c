"""ScalableViT parity cases (reference scalable_vit.py), on the shared recipe of parity.py.  ChanLayerNorm's `g` and
`b` are 4-D, so the 1-D rules of parity.py skip them: `extra` perturbs them, or every LayerNorm affine of the encoder
would go untested.  The comments give every stage's map, its IWSA windows and its SSA key map."""
import torch

from parity import Family

BATCH = 2
# constructor keywords; `input` = (height, width) of the image, `batch` its batch size
SCALABLE_VIT_CASES = {
    # the README ScalableViT-S at 256, batch 1: 64², 32², 16², 8² maps, every IWSA window the whole map (4096, 1024,
    # 256, 64 tokens), every SSA over 8 x 8 keys; ssa_dim_key 40 runs padded to 48
    "readme_256": dict(seed=1201, num_classes=1000, dim=64, heads=(2, 4, 8, 16), depth=(2, 2, 20, 2),
                       ssa_dim_key=(40, 40, 40, 32), reduction_factor=(8, 4, 2, 1), window_size=(64, 32, None, None),
                       input=(256, 256), batch=1),
    # 8 x 8 windows (64 tokens) on a 64 x 64 map
    "window8_64map": dict(seed=1202, num_classes=10, dim=32, heads=1, depth=(1,), reduction_factor=8, window_size=8,
                          input=(256, 256), batch=1),
    # 16 x 16 windows (256 tokens) on 64 x 64 and 32 x 32 maps
    "window16": dict(seed=1203, num_classes=10, dim=32, heads=1, depth=(1, 1), reduction_factor=(8, 4),
                     window_size=16, input=(256, 256), batch=1),
    # non-square: 32 x 24 and 16 x 12 maps, whole-map windows
    "nonsquare_128x96": dict(seed=1204, num_classes=7, dim=32, heads=(1, 2), depth=(1, 2), reduction_factor=(4, 2),
                             input=(128, 96)),
    # reduction 3 does not divide the 32 x 32 and 16 x 16 maps: 10 x 10 and 5 x 5 keys
    "floor_keys": dict(seed=1205, num_classes=5, dim=32, heads=2, depth=(1, 1), reduction_factor=3, input=(128, 128)),
    # key and value heads 64 wide in both attentions
    "dim_64": dict(seed=1206, num_classes=6, dim=64, heads=(1, 2), depth=(1, 1), reduction_factor=(4, 2),
                   ssa_dim_key=64, ssa_dim_value=64, iwsa_dim_key=64, iwsa_dim_value=64, input=(128, 128)),
    # IWSA key heads 24 wide (run at 32) and value heads 64 wide; SSA keys 16 wide
    "iwsa_key24_value64": dict(seed=1207, num_classes=4, dim=32, heads=2, depth=(1, 1), reduction_factor=(4, 2),
                               iwsa_dim_key=24, iwsa_dim_value=64, ssa_dim_key=16, window_size=(16, None),
                               input=(128, 128)),
    # one stage only: no Downsample, no Transformer norm
    "one_stage": dict(seed=1208, num_classes=3, dim=32, heads=2, depth=(2,), reduction_factor=4, input=(64, 64)),
    # ff_expansion_factor 2 and a one-channel image
    "ff2_channels1": dict(seed=1209, num_classes=5, dim=32, heads=1, depth=(1, 1), reduction_factor=(2, 1),
                          ff_expansion_factor=2, channels=1, input=(64, 64)),
    # batch 3
    "batch3": dict(seed=1210, num_classes=8, dim=32, heads=(1, 2), depth=(1, 1), reduction_factor=(4, 2),
                   window_size=(8, None), input=(64, 64), batch=3),
    # value heads 48 wide: no kernel is built for them, so the fused forward falls back to the PyTorch graph
    "fallback_value48": dict(seed=1211, num_classes=4, dim=32, heads=1, depth=(1,), reduction_factor=2,
                             ssa_dim_value=48, input=(64, 64)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 1221
INIT_KWARGS = dict(num_classes=10, dim=32, heads=(1, 2), depth=(1, 2), reduction_factor=(4, 2), ssa_dim_key=40,
                   window_size=(8, None))

_SPEC_KEYS = ("seed", "input", "batch")


def case_kwargs(spec: dict) -> dict:
    return {k: v for k, v in spec.items() if k not in _SPEC_KEYS}


def input_shape(spec: dict) -> tuple:
    return (spec.get("batch", BATCH), spec.get("channels", 3), *spec["input"])


def perturb_layer_norms(name, p, g, spec) -> None:
    if p.dim() == 4 and p.shape[0] == 1 and name.endswith((".g", ".b")):
        p.add_(torch.randn(p.shape, generator=g) * (0.1 if name.endswith(".g") else 0.05))


FAMILY = Family(
    name="scalable_vit", model="scalable_vit.ScalableViT", cases=SCALABLE_VIT_CASES, case_kwargs=case_kwargs,
    input_shape=input_shape, init_seed=INIT_SEED, init={None: INIT_KWARGS}, extra=perturb_layer_norms)
