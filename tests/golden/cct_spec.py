"""CCT parity cases (reference cct.py), on the shared recipe of parity.py.  A case with a `preset` builds that cct_*
function instead of CCT; the fixture also stores the presets' and _cct's signatures and each case's sequence_length."""
from parity import Family, load, signature

BASE = dict(embedding_dim=64, n_input_channels=3, num_layers=2, num_heads=1, mlp_ratio=2, num_classes=7,
            dropout_rate=0., attention_dropout=0.1, stochastic_depth_rate=0.1)
BATCH = 2
# constructor keywords on top of BASE (`preset` names a cct_* function called instead of CCT); `input` = (height,
# width) of the image fed to it.  The comments give the conv output and token grid.
CCT_CASES = {
    # the CIFAR shape: k3 s1 p1, 32 x 32 -> pool to 16 x 16 (256 tokens), sine table
    "cifar_k3": dict(seed=401, img_size=32, kernel_size=3, stride=1, padding=1, input=(32, 32)),
    # the README's two-layer tokenizer, k7 s2 p3, on a non-square image: 40 x 72 -> 20 x 36 -> 10 x 18 -> 5 x 9 -> 3 x 5
    "two_layers_k7_nonsquare": dict(seed=402, img_size=(40, 72), n_conv_layers=2, kernel_size=7, stride=2, padding=3,
                                    num_heads=2, input=(40, 72)),
    # a learnable table
    "learnable": dict(seed=403, img_size=24, kernel_size=3, stride=1, padding=1, positional_embedding="learnable",
                      input=(24, 24)),
    # no table, an image larger than the constructed one (more tokens than sequence_length runs without a table)
    "none_longer": dict(seed=404, img_size=16, kernel_size=3, stride=1, padding=1, positional_embedding="none",
                        input=(20, 24)),
    # MaxPool2d(2, 2, 0): 30 x 30 -> 15 x 15 tokens
    "pool_2_2_0": dict(seed=405, img_size=30, kernel_size=3, stride=1, padding=1, pooling_kernel_size=2,
                       pooling_stride=2, pooling_padding=0, input=(30, 30)),
    # k5 s3 p2 with four channels and three conv layers: 48 -> 16 -> 8 -> 3 -> 2 -> 1 -> 1
    "three_layers_k5_s3": dict(seed=406, img_size=48, n_conv_layers=3, kernel_size=5, stride=3, padding=2,
                               n_input_channels=4, input=(48, 48)),
    # dim_head 32 and 128
    "dh32": dict(seed=407, img_size=16, kernel_size=3, stride=1, padding=1, embedding_dim=64, num_heads=2,
                 input=(16, 16)),
    "dh128": dict(seed=408, img_size=16, kernel_size=3, stride=1, padding=1, embedding_dim=128, num_heads=1,
                  input=(16, 16)),
    # the cct_2 preset (its stride and padding default from kernel_size 3), 32 x 32
    "preset_cct_2": dict(seed=409, preset="cct_2", img_size=32, num_classes=10, input=(32, 32)),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 421
INIT_KWARGS = dict(BASE, img_size=32, kernel_size=3, stride=1, padding=1, n_conv_layers=2, num_heads=2)
PRESETS = ("cct_2", "cct_4", "cct_6", "cct_7", "cct_8", "cct_14", "cct_16")

_SPEC_KEYS = ("seed", "input", "preset")


def case_kwargs(spec: dict) -> dict:
    if "preset" in spec:
        return {k: v for k, v in spec.items() if k not in _SPEC_KEYS}
    kw = dict(BASE)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def signatures(package: str) -> dict:
    return {"signature": signature(load(package, "cct.CCT")),
            "presets": {p: signature(load(package, f"cct.{p}")) for p in PRESETS},
            "cct_defaults": signature(load(package, "cct._cct"))}


FAMILY = Family(
    name="cct", model="cct.CCT", cases=CCT_CASES, case_kwargs=case_kwargs,
    input_shape=lambda spec: (BATCH, case_kwargs(spec).get("n_input_channels", 3), *spec["input"]),
    init_seed=INIT_SEED, init={None: INIT_KWARGS},
    make=lambda package, spec: load(package, "cct." + spec.get("preset", "CCT")),
    signatures=signatures,
    stored=lambda model, spec: {"sequence_length": model.classifier.sequence_length})
