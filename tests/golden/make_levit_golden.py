"""Generate tests/golden/levit.pt from the UNMODIFIED reference (a checkout of which VIT_REFERENCE points at), on CPU,
with make_family_golden.generate on the family record of levit_spec.py, plus the distill-head case (levit_spec.DISTILL,
whose model returns (out, distill)) under the key "distill":

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_levit_golden.py
"""
from __future__ import annotations

import os

import torch

import make_family_golden as G          # puts the reference checkout and this directory on sys.path
from levit_spec import DISTILL, FAMILY
from parity import REFERENCE, input_digest, weights_digest


def distill_case(package: str = REFERENCE) -> dict:
    model = FAMILY.build(DISTILL, package)
    x = FAMILY.input(DISTILL)
    with torch.inference_mode():
        out, distill = model(x.float())
    return {"spec": DISTILL, "weights": weights_digest(model), "input": input_digest(x), "out_fp32": out.clone(),
            "distill_fp32": distill.clone()}


if __name__ == "__main__":
    path = os.path.join(G.HERE, f"{FAMILY.name}.pt")
    fixture = G.generate(FAMILY)
    fixture["distill"] = distill_case()
    torch.save(fixture, path)
    print(f"{FAMILY.name}: {os.path.getsize(path) / 1e3:.1f} kB")
