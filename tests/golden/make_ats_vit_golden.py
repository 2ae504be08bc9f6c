"""Generate tests/golden/ats_vit.pt from the UNMODIFIED reference (a checkout of which VIT_REFERENCE points at), on CPU,
with make_family_golden.generate on the family record of ats_vit_spec.py (which also records every case's uniforms,
token ids, padded lengths and Gumbel-max margin):

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_ats_vit_golden.py
"""
from __future__ import annotations

import os

import torch

import make_family_golden as G          # puts the reference checkout and this directory on sys.path
from ats_vit_spec import FAMILY, MARGIN

if __name__ == "__main__":
    path = os.path.join(G.HERE, f"{FAMILY.name}.pt")
    data = G.generate(FAMILY)
    for name, case in data["cases"].items():
        assert case["margin"] >= MARGIN, f"{name}: Gumbel-max margin {case['margin']} < {MARGIN}: re-seed the case"
    torch.save(data, path)
    print(f"{FAMILY.name}: {os.path.getsize(path) / 1e3:.1f} kB")
