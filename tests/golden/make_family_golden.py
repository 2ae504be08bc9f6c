"""Generate the drop-in families' fixtures tests/golden/<family>.pt from the UNMODIFIED reference
(lucidrains/vit-pytorch 1.23.6, a checkout of which VIT_REFERENCE points at), on CPU; every family of
parity.FAMILY_NAMES, or those named:

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_family_golden.py [family ...]

Stored per family: the constructor signature (and the family's other signature fields), the seeded-init state_dict
digest of each init variant, and per case of <family>_spec.py the case spec, the digests of the rebuilt
bf16-representable weights and input, and the reference's outputs (fp32 logits, plus the family's extra fields).  No
weights: the tests rebuild them from the seeds with the same recipe (parity.py).
"""
from __future__ import annotations

import os
import sys

import torch

REF = os.environ["VIT_REFERENCE"]
sys.path.insert(0, REF)
sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from parity import FAMILY_NAMES, REFERENCE, families, input_digest, state_digest, weights_digest  # noqa: E402


def generate(f) -> dict:
    init = {v: state_digest(f.init_state(REFERENCE, v)) for v in f.init}
    out = {**f.signature_fields(REFERENCE), "init": init[None] if list(init) == [None] else init, "cases": {},
           "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
    for name, spec in f.cases.items():
        model = f.build(spec, REFERENCE)
        x = f.input(spec)
        with torch.inference_mode():
            stored = f.outputs(model, x, spec)
        out["cases"][name] = {"spec": spec, "weights": weights_digest(model), "input": input_digest(x), **stored}
        print(f"{f.name} {name}: done")
    return out


def main(names) -> None:
    fams = families()
    for name in names or FAMILY_NAMES:
        path = os.path.join(HERE, f"{name}.pt")
        torch.save(generate(fams[name]), path)
        print(f"{name}: {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    main(sys.argv[1:])
