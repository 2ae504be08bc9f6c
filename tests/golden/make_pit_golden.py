"""Generate tests/golden/pit.pt from the UNMODIFIED reference (lucidrains/vit-pytorch 1.23.6, a checkout of which
VIT_REFERENCE points at), on CPU:

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_pit_golden.py

Stored, for vit_pytorch.pit.PiT: the constructor signature, the seeded-init state_dict digest, and per case of
pit_spec.py the digests of the rebuilt bf16-representable weights and input and the reference's fp32 logits.  No
weights: the tests rebuild them from the seeds with the same recipe.
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

from pit_spec import INIT_KWARGS, INIT_SEED, PIT_CASES, input_digest, pit_input, pit_model, weights_digest  # noqa: E402


def state_digest(sd) -> dict:
    """sha256 of every tensor's bytes (as make_golden.state_digest / conftest.state_digest)."""
    return {k: (tuple(v.shape), str(v.dtype), hashlib.sha256(v.detach().contiguous().cpu().numpy().tobytes()).hexdigest())
            for k, v in sd.items()}


def signature(cls) -> list:
    return [(k, repr(v.default)) for k, v in inspect.signature(cls.__init__).parameters.items() if k != "self"]


def main() -> None:
    m = importlib.import_module("vit_pytorch.pit")
    torch.manual_seed(INIT_SEED)
    out = {"signature": signature(m.PiT), "init": state_digest(m.PiT(**INIT_KWARGS).state_dict()), "cases": {},
           "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
    for name, spec in PIT_CASES.items():
        model = pit_model(m.PiT, spec)
        x = pit_input(spec)
        with torch.inference_mode():
            logits = model(x.float()).clone()
        out["cases"][name] = {"spec": spec, "weights": weights_digest(model), "input": input_digest(x),
                              "logits_fp32": logits}
        print(f"{name}: |max| {logits.abs().max():.4f}")
    path = os.path.join(HERE, "pit.pt")
    torch.save(out, path)
    print(f"pit: {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    main()
