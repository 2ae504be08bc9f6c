"""Recipe of the CCT parity cases (reference cct.py), shared by make_cct_golden.py, which runs the UNMODIFIED reference
on them, and by the tests, which rebuild the same weights and inputs from the seeds.  The weights are not stored: the
drop-in's constructor consumes the RNG exactly like the reference's (tests/test_cct.py checks the seeded-init digest),
and cct.pt keeps a digest of every rebuilt case so a drift in the recipe fails loudly instead of comparing different
models."""
import hashlib

import torch

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


def input_channels(spec: dict) -> int:
    return case_kwargs(spec).get("n_input_channels", 3)


def cct_model(module, spec: dict):
    """`module` = the reference's vit_pytorch.cct (generator) or vit_pytorch_b200.cct (tests): the same fp32 model from
    the same seeds.  LayerNorm affine parameters and every bias are perturbed so they are exercised, then every
    parameter is rounded to a bf16-representable value, so a bf16 copy of the model holds the same numbers."""
    torch.manual_seed(spec["seed"])
    ctor = getattr(module, spec["preset"]) if "preset" in spec else module.CCT
    model = ctor(**case_kwargs(spec)).eval()
    g = torch.Generator().manual_seed(1000 + spec["seed"])
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1 and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 and n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        for p in model.parameters():
            p.copy_(p.bfloat16().float())
    return model


def cct_input(spec: dict) -> torch.Tensor:
    """bf16 images [BATCH, channels, height, width]."""
    g = torch.Generator().manual_seed(100 + spec["seed"])
    return torch.randn(BATCH, input_channels(spec), *spec["input"], generator=g).bfloat16()


def weights_digest(model) -> str:
    """One sha256 over every state_dict entry (name, shape, dtype, bytes) in registration order."""
    h = hashlib.sha256()
    for k, v in model.state_dict().items():
        h.update(f"{k}{tuple(v.shape)}{v.dtype}".encode())
        h.update(v.detach().float().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def input_digest(x: torch.Tensor) -> str:
    return hashlib.sha256(x.float().contiguous().numpy().tobytes()).hexdigest()
