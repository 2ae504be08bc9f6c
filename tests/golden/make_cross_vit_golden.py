"""Generate tests/golden/cross_vit.pt from the UNMODIFIED reference (lucidrains/vit-pytorch 1.23.6, a checkout of
which VIT_REFERENCE points at), on CPU:

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_cross_vit_golden.py

Stored, for vit_pytorch.cross_vit.CrossViT: the constructor signature, the seeded-init state_dict digests (different
and equal widths), and per case of cross_vit_spec.py the digests of the rebuilt bf16-representable weights and input
and the reference's fp32 logits.  No weights: the tests rebuild them from the seeds with the same recipe.
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

from cross_vit_spec import (CROSS_VIT_CASES, INIT_KWARGS, INIT_SEED, cross_vit_input, cross_vit_model,  # noqa: E402
                            input_digest, weights_digest)


def state_digest(sd) -> dict:
    """sha256 of every tensor's bytes (as make_golden.state_digest / conftest.state_digest)."""
    return {k: (tuple(v.shape), str(v.dtype), hashlib.sha256(v.detach().contiguous().cpu().numpy().tobytes()).hexdigest())
            for k, v in sd.items()}


def signature(cls) -> list:
    return [(k, repr(v.default)) for k, v in inspect.signature(cls.__init__).parameters.items() if k != "self"]


def main() -> None:
    m = importlib.import_module("vit_pytorch.cross_vit")
    out = {"signature": signature(m.CrossViT), "init": {}, "cases": {},
           "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
    for name, kw in (("widths", {}), ("equal", dict(lg_dim=INIT_KWARGS["sm_dim"]))):
        torch.manual_seed(INIT_SEED)
        out["init"][name] = state_digest(m.CrossViT(**{**INIT_KWARGS, **kw}).state_dict())
    for name, spec in CROSS_VIT_CASES.items():
        model = cross_vit_model(m.CrossViT, spec)
        x = cross_vit_input(spec)
        with torch.inference_mode():
            logits = model(x.float()).clone()
        out["cases"][name] = {"spec": spec, "weights": weights_digest(model), "input": input_digest(x),
                              "logits_fp32": logits}
        print(f"{name}: |max| {logits.abs().max():.4f}")
    path = os.path.join(HERE, "cross_vit.pt")
    torch.save(out, path)
    print(f"cross_vit: {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    main()
