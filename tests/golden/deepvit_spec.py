"""Recipe of the DeepViT parity cases (reference deepvit.py), shared by make_deepvit_golden.py, which runs the
UNMODIFIED reference on them, and by the tests, which rebuild the same weights and inputs from the seeds.  The weights
are not stored: the drop-in's constructor consumes the RNG exactly like the reference's (tests/test_deepvit.py checks
the seeded-init digests), and deepvit.pt keeps a digest of every rebuilt case so a drift in the recipe fails loudly
instead of comparing different models."""
import hashlib

import torch

BASE = dict(num_classes=7, dim=64, depth=2, heads=4, mlp_dim=96, dim_head=32, pool='cls', channels=3, dropout=0.,
            emb_dropout=0.)
BATCH = 2
# constructor keywords on top of BASE; `input` = side of the square image fed to it; `mix` = scale of the noise added
# to every layer's re-attention matrix (0: the reference's own N(0, 1) init)
DEEPVIT_CASES = {
    # the README config (256 / 32, dim 1024, depth 6, 16 x 64 heads): 65 tokens, reference init of the mixing
    "readme": dict(seed=81, image_size=256, patch_size=32, dim=1024, depth=6, heads=16, mlp_dim=2048, dim_head=64,
                   input=256, mix=0.0),
    "dh32_n65": dict(seed=82, image_size=32, patch_size=4, input=32, mix=0.5),
    # CaiT's head width, three 16-wide slabs; 197 tokens
    "dh48_n197": dict(seed=83, image_size=56, patch_size=4, heads=6, dim_head=48, input=56, mix=0.5),
    "dh80_mean": dict(seed=84, image_size=32, patch_size=8, heads=3, dim_head=80, input=32, pool='mean', mix=0.5),
    "dh128": dict(seed=85, image_size=32, patch_size=8, heads=2, dim_head=128, input=32, mix=0.5),
    # 576 patches + cls: 37 key blocks, two CTAs of output heads
    "n577_h8": dict(seed=86, image_size=96, patch_size=4, heads=8, dim_head=32, input=96, mix=0.5),
    # 224 / 16: 197 tokens, mean pool, 16 heads
    "p16_h16_mean": dict(seed=87, image_size=224, patch_size=16, heads=16, dim_head=32, dim=96, input=224,
                         pool='mean', mix=0.5),
    # one head: the LayerNorm over a single head yields its beta
    "heads1": dict(seed=88, image_size=32, patch_size=4, heads=1, dim_head=64, input=32, mix=0.5),
    # an image smaller than the constructed one: the first n + 1 rows of the positional table
    "smaller_input": dict(seed=89, image_size=64, patch_size=8, input=32, mix=0.5),
    "depth1_c1": dict(seed=90, image_size=32, patch_size=4, depth=1, channels=1, input=32, mix=0.5),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 123
INIT_KWARGS = dict(image_size=32, patch_size=8, **{k: v for k, v in BASE.items()})


def case_kwargs(spec: dict) -> dict:
    kw = dict(BASE)
    kw.update({k: v for k, v in spec.items() if k not in ("seed", "input", "mix")})
    return kw


def deepvit_model(cls, spec: dict):
    """`cls` = the reference's DeepViT (generator) or the drop-in's (tests): the same fp32 model from the same seeds.
    LayerNorm affine parameters (the one over heads included) are perturbed so they are exercised, each layer's
    re-attention matrix gets `mix` times N(0, 1) noise, then every parameter is rounded to bf16-representable values,
    so a bf16 copy of the model holds the same numbers."""
    torch.manual_seed(spec["seed"])
    model = cls(**case_kwargs(spec)).eval()
    g = torch.Generator().manual_seed(1000 + spec["seed"])
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1 and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 and n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
            elif n.endswith("reattn_weights"):
                p.add_(spec["mix"] * torch.randn(p.shape, generator=g))
        for t in model.parameters():
            t.copy_(t.bfloat16().float())
    return model


def deepvit_input(spec: dict) -> torch.Tensor:
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
