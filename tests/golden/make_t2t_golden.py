"""Generate tests/golden/t2t.pt from the UNMODIFIED reference (a checkout of which VIT_REFERENCE points at), on CPU,
with make_family_golden.generate on the family record of t2t_spec.py:

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_t2t_golden.py
"""
from __future__ import annotations

import os

import torch

import make_family_golden as G          # puts the reference checkout and this directory on sys.path
from t2t_spec import FAMILY

if __name__ == "__main__":
    path = os.path.join(G.HERE, f"{FAMILY.name}.pt")
    torch.save(G.generate(FAMILY), path)
    print(f"{FAMILY.name}: {os.path.getsize(path) / 1e3:.1f} kB")
