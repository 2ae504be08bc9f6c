"""T2T-ViT parity cases (reference t2t.py), on the shared recipe of parity.py."""
from parity import Family, load

BASE = dict(num_classes=7, dim=64, depth=1, heads=2, mlp_dim=96, dim_head=32, pool='cls', channels=3, dropout=0.,
            emb_dropout=0.)
BATCH = 2
# constructor keywords on top of BASE; `input` = (height, width) of the image fed to it; `kind` = "vit_transformer":
# transformer= is given a vit.Transformer of the package under test.  The comments give every soft split's token map
# and width (-> the attention path: the key-block kernel at dp <= 160, the wide kernel above).
README = dict(image_size=224, num_classes=1000, dim=512, depth=5, heads=8, mlp_dim=512, dim_head=64,
              input=(224, 224))
T2T_CASES = {
    # 56 x 56 (147 wide, dp 160) -> 28 x 28 (1323, dp 1344) -> 14 x 14 (11907, the final Linear)
    "readme": dict(README, seed=401),
    # 8 x 8 (147) -> 4 x 4 (1323) -> 2 x 2 (11907); mean pooling over the cls row and the tokens
    "pool_mean": dict(seed=402, image_size=32, pool='mean', input=(32, 32)),
    # one channel: 8 x 8 (49, dp 64) -> 4 x 4 (441, dp 448) -> 2 x 2 (3969)
    "channels1": dict(seed=403, image_size=32, channels=1, input=(32, 32)),
    # two soft splits: 8 x 8 (147) -> 4 x 4 (1323, the final Linear only)
    "two_stage": dict(seed=404, image_size=32, t2t_layers=((7, 4), (3, 2)), input=(32, 32)),
    # 3 x 3 windows throughout: 8 x 8 (27, dp 32) -> 4 x 4 (243, dp 256) -> 2 x 2 (2187)
    "k3_small": dict(seed=405, image_size=16, t2t_layers=((3, 2), (3, 2), (3, 2)), input=(16, 16)),
    # an image smaller than the constructed one: the first n + 1 rows of the positional table; 8 x 8 -> 4 x 4 -> 2 x 2
    "smaller_input": dict(seed=406, image_size=64, input=(32, 32)),
    # a 4 x 16 first map: the reference reads its 64 tokens as 8 x 8 (int(sqrt(n))), then 4 x 4 -> 2 x 2
    "isqrt_4x16": dict(seed=407, image_size=64, input=(16, 64)),
    # main encoder heads 80 wide
    "dh80": dict(seed=408, image_size=32, dim=160, heads=2, dim_head=80, mlp_dim=160, input=(32, 32)),
    # transformer= a vit.Transformer(64, 2, 2, 32, 128) of the package under test
    "dropin_transformer": dict(seed=409, image_size=32, kind="vit_transformer", input=(32, 32)),
    # 66 x 66 (27) -> 33 x 33 (243 wide over 1089 tokens: past the wide kernel's 1024) -> 17 x 17 (2187): PyTorch graph
    "past_wide_cap": dict(seed=410, image_size=132, t2t_layers=((3, 2), (3, 2), (3, 2)), input=(132, 132)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 421
INIT_KWARGS = dict(image_size=32, **BASE)

_SPEC_KEYS = ("seed", "input", "kind")


def case_kwargs(spec: dict) -> dict:
    kw = dict(BASE)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def make(package: str, spec: dict):
    cls = load(package, "t2t.T2TViT")
    if spec.get("kind") != "vit_transformer":
        return cls
    transformer = load(package, "vit.Transformer")

    def build(**kw):
        kw.pop("depth"), kw.pop("heads"), kw.pop("mlp_dim"), kw.pop("dim_head")
        return cls(transformer=transformer(kw["dim"], 2, 2, 32, 128), **kw)
    return build


FAMILY = Family(
    name="t2t", model="t2t.T2TViT", cases=T2T_CASES, case_kwargs=case_kwargs, make=make,
    input_shape=lambda spec: (BATCH, case_kwargs(spec)["channels"], *spec["input"]),
    init_seed=INIT_SEED, init={None: INIT_KWARGS})
