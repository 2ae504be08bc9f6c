"""Recipe of the vit_for_small_dataset parity cases (reference vit_for_small_dataset.py), shared by
make_vit_small_golden.py, which runs the UNMODIFIED reference on them, and by the tests, which rebuild the same weights
and inputs from the seeds.  The weights are not stored: the drop-in's constructor consumes the RNG exactly like the
reference's (tests/test_vit_small_dataset.py checks the seeded-init digests), and vit_small.pt keeps a digest of every
rebuilt case so a drift in the recipe fails loudly instead of comparing different models."""
import hashlib

import torch

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


def vit_small_model(cls, spec: dict):
    """`cls` = the reference's ViT (generator) or the drop-in's (tests): the same fp32 model from the same seeds.
    LayerNorm affine parameters are perturbed so they are exercised, and so is every layer's `temperature`, by a
    different amount per layer: its default is exactly log(dim_head ** -0.5), so a path that ignored it would match.
    Every parameter is then rounded to bf16-representable values, so a bf16 copy of the model holds the same numbers."""
    torch.manual_seed(spec["seed"])
    model = cls(**case_kwargs(spec)).eval()
    g = torch.Generator().manual_seed(1000 + spec["seed"])
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1 and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 and n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        for i, layer in enumerate(model.transformer.layers):
            layer[0].temperature.add_(0.3 * (i + 1) * (-1) ** i)
        for t in model.parameters():
            t.copy_(t.bfloat16().float())
    return model


def vit_small_input(spec: dict) -> torch.Tensor:
    """bf16 images [BATCH, channels, height, width]."""
    g = torch.Generator().manual_seed(100 + spec["seed"])
    return torch.randn(BATCH, spec["channels"], *spec["input"], generator=g).bfloat16()


def weights_digest(model) -> str:
    """One sha256 over every state_dict entry (name, shape, dtype, bytes) in registration order."""
    h = hashlib.sha256()
    for k, v in model.state_dict().items():
        h.update(f"{k}{tuple(v.shape)}{v.dtype}".encode())
        h.update(v.detach().float().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def input_digest(x: torch.Tensor) -> str:
    return hashlib.sha256(x.float().contiguous().numpy().tobytes()).hexdigest()
