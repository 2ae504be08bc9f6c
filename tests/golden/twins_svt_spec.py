"""Twins-SVT parity cases (reference twins_svt.py), on the shared recipe of parity.py."""
import torch

from parity import Family

# every stage runs 8 heads of 64 whatever its width (the reference never passes heads / dim_head down)
BASE = dict(num_classes=7, s1_emb_dim=16, s2_emb_dim=24, s3_emb_dim=32, s4_emb_dim=40, s1_depth=1, s2_depth=1,
            s3_depth=1, s4_depth=1, dropout=0.)
BATCH = 2
# constructor keywords on top of BASE (`default`: on top of nothing but num_classes); `input` = (height, width) of the
# image, `batch` its batch size.  The comments give per stage the token grid, the window and the number of keys.
TWINS_CASES = {
    # the default config at 224 x 224: 56 x 56 (7 x 7 windows, 8 x 8 = 64 keys) -> 28 x 28 (16 keys) -> 14 x 14
    # (4 keys) -> 7 x 7 (1 key: every output is that value row); depths 1, 1, 5, 4
    "default": dict(seed=401, input=(224, 224), default=True, num_classes=10),
    # full 64-row window tiles: 16 x 16 (window 8, k 4: 16 keys) -> 8 x 8 (window 8, k 8: 1 key) -> 4 x 4 (window 4,
    # k 2: 4 keys) -> 2 x 2 (k 2: 1 key)
    "window8": dict(seed=402, input=(32, 32), s1_patch_size=2, s1_local_patch_size=8, s1_global_k=4,
                    s2_local_patch_size=8, s2_global_k=8, s3_local_patch_size=4, s3_global_k=2, s4_global_k=2),
    # a non-square image, packed windows, a k that does not divide the grid, k 1, stage depths > 1, a 5 x 5 PEG:
    # 32 x 16 (window 4, k 3: 10 x 5 = 50 keys, the last 2 rows and 1 column feed no key) -> 16 x 8 (window 2, k 2:
    # 32 keys) -> 8 x 4 (window 1, k 1: 32 keys == queries) -> 4 x 2 (k 1: 8 keys)
    "nonsquare_packed": dict(seed=403, input=(64, 32), s1_patch_size=2, s1_local_patch_size=4, s1_global_k=3,
                             s2_local_patch_size=2, s2_global_k=2, s2_depth=2, s3_local_patch_size=1, s3_global_k=1,
                             s4_global_k=1, s4_depth=2, peg_kernel_size=5),
    # more than 128 keys, windows that do not fill a tile, a 7 x 7 PEG: 24 x 24 (window 6, k 2: 144 keys) -> 12 x 12
    # (window 3, k 1: 144 keys) -> 6 x 6 (window 2, k 3: 4 keys) -> 3 x 3 (k 3: 1 key)
    "keys_144": dict(seed=404, input=(48, 48), s1_patch_size=2, s1_local_patch_size=6, s1_global_k=2,
                     s2_local_patch_size=3, s2_global_k=1, s3_local_patch_size=2, s3_global_k=3, s4_global_k=3,
                     peg_kernel_size=7),
    # more than 512 keys (they stream through shared memory), batch 1, a 1 x 1 PEG, an s4_patch_size of 1:
    # 28 x 28 (window 7, k 1: 784 keys == queries) -> 14 x 14 (window 7, k 2: 49 keys) -> 7 x 7 (window 7, k 7: 1 key)
    # -> 7 x 7 (k 7: 1 key)
    "keys_784_batch1": dict(seed=405, input=(56, 56), batch=1, s1_patch_size=2, s1_global_k=1, s2_global_k=2,
                            s4_patch_size=1, peg_kernel_size=1),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 421
INIT_KWARGS = dict(BASE, s1_patch_size=2, s3_depth=2, s4_depth=2)

_SPEC_KEYS = ("seed", "input", "batch", "default")


def case_kwargs(spec: dict) -> dict:
    kw = {} if spec.get("default") else dict(BASE)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def perturb_norms(name: str, p: torch.Tensor, g: torch.Generator, spec: dict) -> None:
    """The LayerNorm affines are 4-D `g` / `b`, which the shared 1-D weight / bias rules skip."""
    if name.endswith(".g"):
        p.add_(0.1 * torch.randn(p.shape, generator=g))
    elif name.endswith(".b"):
        p.add_(0.05 * torch.randn(p.shape, generator=g))


FAMILY = Family(
    name="twins_svt", model="twins_svt.TwinsSVT", cases=TWINS_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (spec.get("batch", BATCH), 3, *spec["input"]),
    init_seed=INIT_SEED, init={None: INIT_KWARGS}, extra=perturb_norms)
