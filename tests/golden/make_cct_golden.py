"""Generate tests/golden/cct.pt from the UNMODIFIED reference (lucidrains/vit-pytorch 1.23.6, a checkout of which
VIT_REFERENCE points at), on CPU:

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_cct_golden.py

Stored, for vit_pytorch.cct: the signatures of CCT and of the cct_* presets, the seeded-init state_dict digest, and
per case of cct_spec.py the digests of the rebuilt bf16-representable weights and input and the reference's fp32
logits.  No weights: the tests rebuild them from the seeds with the same recipe.
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

from cct_spec import CCT_CASES, INIT_KWARGS, INIT_SEED, PRESETS, cct_input, cct_model, input_digest, weights_digest  # noqa: E402,E501


def state_digest(sd) -> dict:
    """sha256 of every tensor's bytes (as make_golden.state_digest / conftest.state_digest)."""
    return {k: (tuple(v.shape), str(v.dtype), hashlib.sha256(v.detach().contiguous().cpu().numpy().tobytes()).hexdigest())
            for k, v in sd.items()}


def signature(fn) -> list:
    """(name, repr(default)) of every parameter: of cls.__init__ for a class, of the function itself otherwise."""
    target = fn.__init__ if inspect.isclass(fn) else fn
    return [(k, repr(v.default)) for k, v in inspect.signature(target).parameters.items() if k != "self"]


def main() -> None:
    m = importlib.import_module("vit_pytorch.cct")
    torch.manual_seed(INIT_SEED)
    out = {"signature": signature(m.CCT), "presets": {p: signature(getattr(m, p)) for p in PRESETS},
           "cct_defaults": signature(m._cct),
           "init": state_digest(m.CCT(**INIT_KWARGS).state_dict()), "cases": {},
           "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
    for name, spec in CCT_CASES.items():
        model = cct_model(m, spec)
        x = cct_input(spec)
        with torch.inference_mode():
            logits = model(x.float()).clone()
        out["cases"][name] = {"spec": spec, "weights": weights_digest(model), "input": input_digest(x),
                              "sequence_length": model.classifier.sequence_length, "logits_fp32": logits}
        print(f"{name}: n {model.classifier.sequence_length} |max| {logits.abs().max():.4f}")
    path = os.path.join(HERE, "cct.pt")
    torch.save(out, path)
    print(f"cct: {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    main()
