"""Recipe of the CaiT parity cases (reference cait.py), shared by make_cait_golden.py, which runs the UNMODIFIED
reference on them, and by the tests, which rebuild the same weights and inputs from the seeds.  The weights are not
stored: the drop-in's constructor consumes the RNG exactly like the reference's (tests/test_cait.py checks the
seeded-init digests), and cait.pt keeps a digest of every rebuilt case so a drift in the recipe fails loudly instead of
comparing different models."""
import hashlib
import random

import torch

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


def cait_model(cls, spec: dict):
    """`cls` = the reference's CaiT (generator) or the drop-in's (tests): the same fp32 model from the same seeds.
    LayerNorm affine parameters and the LayerScale vectors are perturbed so they are exercised, each layer's mixing
    matrices get `mix` times N(0, 1) noise, then every parameter is rounded to bf16-representable values, so a bf16 copy
    of the model holds the same numbers."""
    torch.manual_seed(spec["seed"])
    model = cls(**case_kwargs(spec)).eval()
    g = torch.Generator().manual_seed(1000 + spec["seed"])
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1 and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 and n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
            elif n.endswith(".scale"):                          # LayerScale [1, 1, dim]
                p.mul_(1 + 0.5 * torch.randn(p.shape, generator=g))
            elif n.endswith("mix_heads_pre_attn") or n.endswith("mix_heads_post_attn"):
                p.add_(spec["mix"] * torch.randn(p.shape, generator=g))
                if n.endswith("mix_heads_pre_attn") and spec.get("pre_sign", 1) < 0:
                    p.copy_(-p.abs())
        for t in model.parameters():
            t.copy_(t.bfloat16().float())
    return model


def seed_layer_dropout(spec: dict) -> None:
    """Seed the generators layer dropout draws from (torch's CPU generator, and `random` when every layer would be
    dropped) right before a forward, so that every run of the case keeps the same layers."""
    if "drop_seed" in spec:
        torch.manual_seed(spec["drop_seed"])
        random.seed(spec["drop_seed"])


def cait_input(spec: dict) -> torch.Tensor:
    """bf16 images [BATCH, 3, input, input]."""
    g = torch.Generator().manual_seed(100 + spec["seed"])
    return torch.randn(BATCH, 3, spec["input"], spec["input"], generator=g).bfloat16()


def weights_digest(model) -> str:
    """One sha256 over every state_dict entry (name, shape, dtype, bytes) in registration order."""
    h = hashlib.sha256()
    for k, v in model.state_dict().items():
        h.update(f"{k}{tuple(v.shape)}{v.dtype}".encode())
        h.update(v.detach().float().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def input_digest(x: torch.Tensor) -> str:
    return hashlib.sha256(x.float().contiguous().numpy().tobytes()).hexdigest()
