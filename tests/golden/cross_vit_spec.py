"""CrossViT parity cases (reference cross_vit.py), on the shared recipe of parity.py."""
from parity import Family

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


FAMILY = Family(
    name="cross_vit", model="cross_vit.CrossViT", cases=CROSS_VIT_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (BATCH, spec.get("channels", BASE["channels"]), spec["input"], spec["input"]),
    init_seed=INIT_SEED, init={"widths": INIT_KWARGS, "equal": dict(INIT_KWARGS, lg_dim=INIT_KWARGS["sm_dim"])})
