"""N-dimensional ViT parity cases (reference vit_nd.py / vit_nd_rotary.py), on the shared recipe of parity.py.  A case's
`kind` picks the module; the fixture stores both classes' signatures and seeded-init digests by kind.  Its own rules:
the rotary `freqs` buffer is rounded to bf16 like the parameters, and the rotary model's return_embed output for the
first sample is stored too."""
from parity import Family, load, round_buffers, signature

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


KINDS = ("vit_nd", "vit_nd_rotary")


def embed(model, x, spec) -> dict:
    rotary = spec["kind"] == "vit_nd_rotary"
    return {"embed0_fp32": model(x.float(), return_embed=True)[:1].clone() if rotary else None}


FAMILY = Family(
    name="vit_nd", model="vit_nd.ViTND", cases=VIT_ND_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (BATCH, spec["channels"], *spec["shape"]),
    init_seed=INIT_SEED, init={kind: INIT_KWARGS for kind in KINDS},
    make=lambda package, spec: load(package, f"{spec['kind']}.ViTND"),
    signatures=lambda package: {"signature": {k: signature(load(package, f"{k}.ViTND")) for k in KINDS}},
    after=lambda model, g, spec: round_buffers(model), embed=embed)
