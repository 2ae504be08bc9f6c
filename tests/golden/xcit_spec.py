"""Recipe of the XCiT parity cases (reference xcit.py), shared by make_xcit_golden.py, which runs the UNMODIFIED
reference on them, and by the tests, which rebuild the same weights and inputs from the seeds.  The weights are not
stored: the drop-in's constructor consumes the RNG exactly like the reference's (tests/test_xcit.py checks the
seeded-init digests), and xcit.pt keeps a digest of every rebuilt case so a drift in the recipe fails loudly instead of
comparing different models."""
import hashlib
import random

import torch

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


def xcit_model(cls, spec: dict):
    """`cls` = the reference's XCiT (generator) or the drop-in's (tests): the same fp32 model from the same seeds.
    LayerNorm and BatchNorm affine parameters, LayerScale vectors, temperatures and the BatchNorm running statistics are
    perturbed so they are exercised, then every parameter and floating-point buffer is rounded to bf16-representable
    values, so a bf16 copy of the model holds the same numbers."""
    torch.manual_seed(spec["seed"])
    model = cls(**case_kwargs(spec)).eval()
    g = torch.Generator().manual_seed(1000 + spec["seed"])
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1 and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 and n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
            elif n.endswith(".scale"):                          # LayerScale (dim,)
                p.mul_(1 + 0.5 * torch.randn(p.shape, generator=g))
            elif n.endswith("temperature"):
                p.add_(spec.get("tau", 0.0) + 0.3 * torch.randn(p.shape, generator=g))
        for n, b in model.named_buffers():
            if n.endswith("running_mean"):
                b.add_(0.2 * torch.randn(b.shape, generator=g))
            elif n.endswith("running_var"):
                b.mul_(0.5 + torch.rand(b.shape, generator=g))
        for t in list(model.parameters()) + [b for b in model.buffers() if b.is_floating_point()]:
            t.copy_(t.bfloat16().float())
    return model


def seed_layer_dropout(spec: dict) -> None:
    """Seed the generators layer dropout draws from (torch's CPU generator, and `random` when every layer would be
    dropped) right before a forward, so that every run of the case keeps the same layers."""
    if "drop_seed" in spec:
        torch.manual_seed(spec["drop_seed"])
        random.seed(spec["drop_seed"])


def xcit_input(spec: dict) -> torch.Tensor:
    """bf16 images [BATCH, 3, height, width]."""
    g = torch.Generator().manual_seed(100 + spec["seed"])
    return torch.randn(BATCH, 3, *spec["input"], generator=g).bfloat16()


def weights_digest(model) -> str:
    """One sha256 over every state_dict entry (name, shape, dtype, bytes) in registration order."""
    h = hashlib.sha256()
    for k, v in model.state_dict().items():
        h.update(f"{k}{tuple(v.shape)}{v.dtype}".encode())
        h.update(v.detach().float().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def input_digest(x: torch.Tensor) -> str:
    return hashlib.sha256(x.float().contiguous().numpy().tobytes()).hexdigest()
