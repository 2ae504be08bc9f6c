"""ViViT parity cases (reference vivit.py), on the shared recipe of parity.py.  Every case stores the logits of each
frame-mask kind."""
import torch

from parity import Family

BASE = dict(num_classes=7, dim=64, spatial_depth=2, temporal_depth=2, heads=2, dim_head=32, mlp_dim=96)
BATCH = 3
# geometry: constructor sizes, and the input's (frames, height, width) when it is smaller than those
_GEO = dict(image_size=(16, 24), image_patch_size=8, frames=8, frame_patch_size=2, channels=3)
VIVIT_CASES = {}
_seed = 40
for _variant, _v in (("factorized_encoder", "fe"), ("factorized_self_attention", "fsa")):
    for _pool in ("cls", "mean"):
        for _flash in (True, False):
            _seed += 1
            VIVIT_CASES[f"{_v}_{_pool}_{'sdpa' if _flash else 'softmax'}"] = dict(
                seed=_seed, variant=_variant, pool=_pool, use_flash_attn=_flash, input=(8, 16, 24), **_GEO)
# a clip shorter and smaller than the constructed size: pos_embedding[:, :frames, :seq] takes a corner of the table
VIVIT_CASES["fe_cls_short"] = dict(seed=51, variant="factorized_encoder", pool="cls", use_flash_attn=True,
                                   input=(4, 16, 16), image_size=24, image_patch_size=8, frames=8, frame_patch_size=2,
                                   channels=3)
VIVIT_CASES["fsa_mean_short"] = dict(seed=52, variant="factorized_self_attention", pool="mean", use_flash_attn=False,
                                     input=(4, 16, 16), image_size=24, image_patch_size=8, frames=8,
                                     frame_patch_size=2, channels=3)
# one frame per patch and 16 x 16 patches (the TMA patch embedding on the fused path)
VIVIT_CASES["fe_cls_pf1_p16"] = dict(seed=53, variant="factorized_encoder", pool="cls", use_flash_attn=True,
                                     input=(3, 32, 32), image_size=32, image_patch_size=16, frames=3,
                                     frame_patch_size=1, channels=3)
MASK_KINDS = ("none", "partial", "full")
VARIANTS = ("factorized_encoder", "factorized_self_attention")
# the seeded-init (unperturbed) comparison
INIT_SEED = 123
INIT_KWARGS = dict(image_size=(16, 24), image_patch_size=8, frames=8, frame_patch_size=2, channels=3, **BASE)


def case_kwargs(spec: dict) -> dict:
    return dict(image_size=spec["image_size"], image_patch_size=spec["image_patch_size"], frames=spec["frames"],
                frame_patch_size=spec["frame_patch_size"], channels=spec["channels"], pool=spec["pool"],
                variant=spec["variant"], use_flash_attn=spec["use_flash_attn"], **BASE)


def vivit_mask(spec: dict, kind: str):
    """Frame mask [BATCH, frames] (True = keep) of a mask kind:
      none:    no mask;
      partial: clip 0 loses its first frame patch, clip 1 one frame of its second frame patch (the reference reduces
               each frame patch with `all`), clip 2 keeps everything;
      full:    as partial, but every frame of clip 1 is masked."""
    if kind == "none":
        return None
    frames, pf = spec["input"][0], spec["frame_patch_size"]
    m = torch.ones(BATCH, frames, dtype=torch.bool)
    m[0, :pf] = False
    if kind == "partial":
        m[1, min(pf, frames - 1)] = False
    else:
        m[1] = False
    return m


FAMILY = Family(
    name="vivit", model="vivit.ViViT", cases=VIVIT_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (BATCH, spec["channels"], *spec["input"]),
    init_seed=INIT_SEED, init={v: dict(INIT_KWARGS, variant=v) for v in VARIANTS},
    forwards=lambda spec: [(kind, {"mask": vivit_mask(spec, kind)}) for kind in MASK_KINDS])
