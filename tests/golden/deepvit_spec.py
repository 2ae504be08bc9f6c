"""DeepViT parity cases (reference deepvit.py), on the shared recipe of parity.py.  Its own rule: each layer's
re-attention matrix gets `mix` times N(0, 1) noise (the LayerNorm over the heads is perturbed by the shared rule)."""
import torch

from parity import Family

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


def extra(n, p, g, spec) -> None:
    if n.endswith("reattn_weights"):
        p.add_(spec["mix"] * torch.randn(p.shape, generator=g))


FAMILY = Family(
    name="deepvit", model="deepvit.DeepViT", cases=DEEPVIT_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (BATCH, spec.get("channels", BASE["channels"]), spec["input"], spec["input"]),
    init_seed=INIT_SEED, init={pool: dict(INIT_KWARGS, pool=pool) for pool in ("cls", "mean")}, extra=extra)
