"""Recipe of the CrossViT parity cases (reference cross_vit.py), shared by make_cross_vit_golden.py, which runs the
UNMODIFIED reference on them, and by the tests, which rebuild the same weights and inputs from the seeds.  The weights
are not stored: the drop-in's constructor consumes the RNG exactly like the reference's (tests/test_cross_vit.py checks
the seeded-init digests), and cross_vit.pt keeps a digest of every rebuilt case so a drift in the recipe fails loudly
instead of comparing different models."""
import hashlib

import torch

BASE = dict(num_classes=7, sm_dim=32, lg_dim=64, sm_patch_size=4, lg_patch_size=8, sm_enc_depth=1, sm_enc_heads=2,
            sm_enc_mlp_dim=64, sm_enc_dim_head=32, lg_enc_depth=2, lg_enc_heads=2, lg_enc_mlp_dim=96,
            lg_enc_dim_head=32, cross_attn_depth=2, cross_attn_heads=2, cross_attn_dim_head=32, depth=2,
            dropout=0., emb_dropout=0., channels=3)
BATCH = 3
# constructor keywords on top of BASE; `input` = side of the square image fed to it
CROSS_VIT_CASES = {
    # different widths: both ProjectInOut projections are Linears; 65 + 17 tokens
    "widths_32_64": dict(seed=71, image_size=32, input=32),
    # equal widths: both projections are Identity
    "equal_widths": dict(seed=72, image_size=32, input=32, sm_dim=48, lg_dim=48),
    # 24 x 24 sm patches + cls = 577 tokens (key-block attention); lg 16 x 16 patches (TMA patch path)
    "long_577": dict(seed=73, image_size=96, input=96, lg_patch_size=16, depth=1),
    # 16 x 16 sm patches with 3 channels: the TMA patch path on the sm stream
    "p16_c3": dict(seed=74, image_size=64, input=64, sm_patch_size=16, lg_patch_size=32),
    # a different head width in each attention
    "mixed_heads": dict(seed=75, image_size=32, input=32, sm_enc_dim_head=80, lg_enc_dim_head=128,
                        cross_attn_dim_head=32),
    "dh64": dict(seed=76, image_size=32, input=32, sm_enc_dim_head=64, lg_enc_dim_head=64, cross_attn_dim_head=64),
    "c1": dict(seed=77, image_size=32, input=32, channels=1),
    # an image smaller than the constructed one: the first n + 1 rows of each positional table
    "smaller_input": dict(seed=78, image_size=48, input=32),
    "depth1": dict(seed=79, image_size=32, input=32, depth=1, cross_attn_depth=1, lg_enc_depth=1),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 123
INIT_KWARGS = dict(image_size=32, **BASE)


def case_kwargs(spec: dict) -> dict:
    kw = dict(BASE)
    kw.update({k: v for k, v in spec.items() if k not in ("seed", "input")})
    return kw


def cross_vit_model(cls, spec: dict):
    """`cls` = the reference's CrossViT (generator) or the drop-in's (tests): the same fp32 model from the same seeds.
    LayerNorm affine parameters are perturbed so they are exercised, then every parameter is rounded to
    bf16-representable values, so a bf16 copy of the model holds the same numbers."""
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


def cross_vit_input(spec: dict) -> torch.Tensor:
    """bf16 images [BATCH, channels, input, input]."""
    g = torch.Generator().manual_seed(100 + spec["seed"])
    c = spec.get("channels", BASE["channels"])
    return torch.randn(BATCH, c, spec["input"], spec["input"], generator=g).bfloat16()


def weights_digest(model) -> str:
    """One sha256 over every state_dict entry (name, shape, dtype, bytes) in registration order."""
    h = hashlib.sha256()
    for k, v in model.state_dict().items():
        h.update(f"{k}{tuple(v.shape)}{v.dtype}".encode())
        h.update(v.detach().float().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def input_digest(x: torch.Tensor) -> str:
    return hashlib.sha256(x.float().contiguous().numpy().tobytes()).hexdigest()
