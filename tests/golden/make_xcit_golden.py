"""Generate tests/golden/xcit.pt from the UNMODIFIED reference (lucidrains/vit-pytorch 1.23.6, a checkout of which
VIT_REFERENCE points at), on CPU:

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_xcit_golden.py

Stored, for vit_pytorch.xcit.XCiT: the constructor signature, the seeded-init state_dict digest (depth 20, so the
LayerScale init takes its 0.1 and 1e-6 branches, BatchNorm buffers included), and per case of xcit_spec.py the digests of the rebuilt
bf16-representable weights and input and the reference's fp32 logits.  No weights: the tests rebuild them from the
seeds with the same recipe.
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

from xcit_spec import (XCIT_CASES, INIT_KWARGS, INIT_SEED, xcit_input, xcit_model, input_digest,  # noqa: E402
                       seed_layer_dropout, weights_digest)


def state_digest(sd) -> dict:
    """sha256 of every tensor's bytes (as make_golden.state_digest / conftest.state_digest)."""
    return {k: (tuple(v.shape), str(v.dtype), hashlib.sha256(v.detach().contiguous().cpu().numpy().tobytes()).hexdigest())
            for k, v in sd.items()}


def signature(cls) -> list:
    return [(k, repr(v.default)) for k, v in inspect.signature(cls.__init__).parameters.items() if k != "self"]


def main() -> None:
    m = importlib.import_module("vit_pytorch.xcit")
    torch.manual_seed(INIT_SEED)
    out = {"signature": signature(m.XCiT), "init": state_digest(m.XCiT(**INIT_KWARGS).state_dict()), "cases": {},
           "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
    for name, spec in XCIT_CASES.items():
        model = xcit_model(m.XCiT, spec)
        x = xcit_input(spec)
        seed_layer_dropout(spec)
        with torch.inference_mode():
            logits = model(x.float()).clone()
        out["cases"][name] = {"spec": spec, "weights": weights_digest(model), "input": input_digest(x),
                              "logits_fp32": logits}
        print(f"{name}: |max| {logits.abs().max():.4f}")
    path = os.path.join(HERE, "xcit.pt")
    torch.save(out, path)
    print(f"xcit: {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    main()
