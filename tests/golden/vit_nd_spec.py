"""Recipe of the N-dimensional ViT parity cases (reference vit_nd.py / vit_nd_rotary.py), shared by
make_vit_nd_golden.py, which runs the UNMODIFIED reference on them, and by the tests, which rebuild the same weights and
inputs from the seeds.  The weights are not stored: the drop-ins' constructors consume the RNG exactly like the
reference's (tests/test_vit_nd.py checks the seeded-init digests), and vit_nd.pt keeps a digest of every rebuilt case
so a drift in the recipe fails loudly instead of comparing different models."""
import hashlib

import torch

# every case: ViT dims below; `shape` is the input without (batch, channels)
BASE = dict(num_classes=7, dim=64, depth=2, heads=2, dim_head=32, mlp_dim=96)
BATCH = 3
VIT_ND_CASES = {
    "nd_r1_cls": dict(kind="vit_nd", seed=21, ndim=1, shape=(64,), patch=8, channels=3, pool="cls"),
    "nd_r2_mean": dict(kind="vit_nd", seed=22, ndim=2, shape=(16, 24), patch=(4, 8), channels=3, pool="mean"),
    "nd_r2_cls": dict(kind="vit_nd", seed=23, ndim=2, shape=(16, 24), patch=(4, 8), channels=3, pool="cls"),
    "nd_r3_cls": dict(kind="vit_nd", seed=24, ndim=3, shape=(4, 16, 16), patch=(2, 8, 4), channels=2, pool="cls"),
    "nd_r4_mean": dict(kind="vit_nd", seed=25, ndim=4, shape=(4, 4, 8, 8), patch=(2, 2, 4, 4), channels=1,
                       pool="mean"),
    "rot_r1": dict(kind="vit_nd_rotary", seed=31, ndim=1, shape=(64,), patch=8, channels=3),
    "rot_r2": dict(kind="vit_nd_rotary", seed=32, ndim=2, shape=(16, 24), patch=(4, 8), channels=3),
    "rot_r3": dict(kind="vit_nd_rotary", seed=33, ndim=3, shape=(4, 16, 16), patch=(2, 8, 4), channels=2),
    "rot_r4": dict(kind="vit_nd_rotary", seed=34, ndim=4, shape=(4, 4, 8, 8), patch=(2, 2, 4, 4), channels=1),
}
# the seeded-init (unperturbed) comparison of both classes
INIT_SEED = 123
INIT_KWARGS = dict(ndim=3, input_shape=(4, 16, 16), patch_size=(2, 8, 4), channels=2, **BASE)


def case_kwargs(spec: dict) -> dict:
    kw = dict(ndim=spec["ndim"], input_shape=spec["shape"], patch_size=spec["patch"], channels=spec["channels"], **BASE)
    if "pool" in spec:
        kw["pool"] = spec["pool"]
    return kw


def vit_nd_model(cls, spec: dict):
    """`cls` = the reference's ViTND (generator) or the drop-in's (tests): the same fp32 model from the same seeds.
    LayerNorm affine parameters are perturbed so they are exercised; every parameter AND buffer (the rotary `freqs`)
    is rounded to bf16-representable values, so a bf16 copy of the model holds the very same numbers."""
    torch.manual_seed(spec["seed"])
    model = cls(**case_kwargs(spec)).eval()
    g = torch.Generator().manual_seed(1000 + spec["seed"])
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1 and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 and n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        for t in list(model.parameters()) + list(model.buffers()):
            t.copy_(t.bfloat16().float())
    return model


def vit_nd_input(spec: dict) -> torch.Tensor:
    """bf16 input [BATCH, channels, *shape]."""
    g = torch.Generator().manual_seed(100 + spec["seed"])
    return torch.randn(BATCH, spec["channels"], *spec["shape"], generator=g).bfloat16()


def weights_digest(model) -> str:
    """One sha256 over every state_dict entry (name, shape, dtype, bytes) in registration order."""
    h = hashlib.sha256()
    for k, v in model.state_dict().items():
        h.update(f"{k}{tuple(v.shape)}{v.dtype}".encode())
        h.update(v.detach().float().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def input_digest(x: torch.Tensor) -> str:
    return hashlib.sha256(x.float().contiguous().numpy().tobytes()).hexdigest()
