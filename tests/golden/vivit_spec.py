"""Recipe of the ViViT parity cases (reference vivit.py), shared by make_vivit_golden.py, which runs the UNMODIFIED
reference on them, and by the tests, which rebuild the same weights, inputs and frame masks from the seeds.  The weights
are not stored: the drop-in's constructor consumes the RNG exactly like the reference's (tests/test_vivit.py checks the
seeded-init digests), and vivit.pt keeps a digest of every rebuilt case so a drift in the recipe fails loudly instead of
comparing different models."""
import hashlib

import torch

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
# the seeded-init (unperturbed) comparison
INIT_SEED = 123
INIT_KWARGS = dict(image_size=(16, 24), image_patch_size=8, frames=8, frame_patch_size=2, channels=3, **BASE)


def case_kwargs(spec: dict) -> dict:
    return dict(image_size=spec["image_size"], image_patch_size=spec["image_patch_size"], frames=spec["frames"],
                frame_patch_size=spec["frame_patch_size"], channels=spec["channels"], pool=spec["pool"],
                variant=spec["variant"], use_flash_attn=spec["use_flash_attn"], **BASE)


def vivit_model(cls, spec: dict):
    """`cls` = the reference's ViViT (generator) or the drop-in's (tests): the same fp32 model from the same seeds.
    LayerNorm affine parameters are perturbed so they are exercised; every parameter is rounded to bf16-representable
    values, so a bf16 copy of the model holds the very same numbers."""
    torch.manual_seed(spec["seed"])
    model = cls(**case_kwargs(spec)).eval()
    g = torch.Generator().manual_seed(1000 + spec["seed"])
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1 and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 and n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        for t in model.parameters():
            t.copy_(t.bfloat16().float())
    return model


def vivit_input(spec: dict) -> torch.Tensor:
    """bf16 video [BATCH, channels, frames, height, width]."""
    g = torch.Generator().manual_seed(100 + spec["seed"])
    return torch.randn(BATCH, spec["channels"], *spec["input"], generator=g).bfloat16()


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


def weights_digest(model) -> str:
    """One sha256 over every state_dict entry (name, shape, dtype, bytes) in registration order."""
    h = hashlib.sha256()
    for k, v in model.state_dict().items():
        h.update(f"{k}{tuple(v.shape)}{v.dtype}".encode())
        h.update(v.detach().float().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def input_digest(x: torch.Tensor) -> str:
    return hashlib.sha256(x.float().contiguous().numpy().tobytes()).hexdigest()
