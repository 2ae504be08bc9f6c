"""Generate tests/golden/vivit.pt from the UNMODIFIED reference (lucidrains/vit-pytorch 1.23.6, a checkout of which
VIT_REFERENCE points at), on CPU:

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_vivit_golden.py

Stored, for vit_pytorch.vivit.ViViT: the constructor signature, the seeded-init state_dict digests of both variants,
and per case of vivit_spec.py (both variants x both pools x use_flash_attn True / False, a clip shorter and smaller than
the constructed size, one frame per patch with 16 x 16 patches) the digests of the rebuilt bf16-representable weights
and input, and the reference's fp32 logits without a mask, with a partial frame mask and with a mask that hides every
frame of one clip.
No weights: the tests rebuild them from the seeds with the same recipe.
"""
from __future__ import annotations

import hashlib
import importlib
import inspect
import os
import sys

import torch

REF = os.environ["VIT_REFERENCE"]
sys.path.insert(0, REF)
sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from vivit_spec import (INIT_KWARGS, INIT_SEED, MASK_KINDS, VIVIT_CASES, input_digest, vivit_input,  # noqa: E402
                        vivit_mask, vivit_model, weights_digest)


def state_digest(sd) -> dict:
    """sha256 of every tensor's bytes (as make_golden.state_digest / conftest.state_digest)."""
    return {k: (tuple(v.shape), str(v.dtype), hashlib.sha256(v.detach().contiguous().cpu().numpy().tobytes()).hexdigest())
            for k, v in sd.items()}


def signature(cls) -> list:
    return [(k, repr(v.default)) for k, v in inspect.signature(cls.__init__).parameters.items() if k != "self"]


def main() -> None:
    m = importlib.import_module("vit_pytorch.vivit")
    out = {"signature": signature(m.ViViT), "init": {}, "cases": {},
           "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
    for variant in ("factorized_encoder", "factorized_self_attention"):
        torch.manual_seed(INIT_SEED)
        out["init"][variant] = state_digest(m.ViViT(variant=variant, **INIT_KWARGS).state_dict())
    for name, spec in VIVIT_CASES.items():
        model = vivit_model(m.ViViT, spec)
        x = vivit_input(spec)
        logits = {}
        with torch.inference_mode():
            for kind in MASK_KINDS:
                logits[kind] = model(x.float(), mask=vivit_mask(spec, kind)).clone()
        out["cases"][name] = {"spec": spec, "weights": weights_digest(model), "input": input_digest(x),
                              "logits_fp32": logits}
        print(f"{name}: |max| {logits['none'].abs().max():.4f}, full - partial mask on clip 1: "
              f"{(logits['full'][1] - logits['partial'][1]).abs().max():.4f}")
    path = os.path.join(HERE, "vivit.pt")
    torch.save(out, path)
    print(f"vivit: {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    main()
