"""Generate tests/golden/vit_nd.pt from the UNMODIFIED reference (lucidrains/vit-pytorch 1.23.6, a checkout of which
VIT_REFERENCE points at), on CPU:

    VIT_REFERENCE=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_vit_nd_golden.py

Stored, for vit_pytorch.vit_nd.ViTND and vit_pytorch.vit_nd_rotary.ViTND: the constructor signatures, the seeded-init
state_dict digests, and per case of vit_nd_spec.py (ranks 1 to 4, both pools of vit_nd) the digests of the rebuilt
bf16-representable weights and input, the reference's fp32 logits and, for the rotary model, its return_embed output
for the first sample.
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

from vit_nd_spec import (INIT_KWARGS, INIT_SEED, VIT_ND_CASES, input_digest, vit_nd_input, vit_nd_model,  # noqa: E402
                         weights_digest)


def state_digest(sd) -> dict:
    """sha256 of every tensor's bytes (as make_golden.state_digest / conftest.state_digest)."""
    return {k: (tuple(v.shape), str(v.dtype), hashlib.sha256(v.detach().contiguous().cpu().numpy().tobytes()).hexdigest())
            for k, v in sd.items()}


def signature(cls) -> list:
    return [(k, repr(v.default)) for k, v in inspect.signature(cls.__init__).parameters.items() if k != "self"]


def main() -> None:
    mods = {k: importlib.import_module("vit_pytorch." + k) for k in ("vit_nd", "vit_nd_rotary")}
    out = {"signature": {}, "init": {}, "cases": {},
           "versions": {"torch": str(torch.__version__), "reference": "vit-pytorch 1.23.6"}}
    for kind, m in mods.items():
        out["signature"][kind] = signature(m.ViTND)
        torch.manual_seed(INIT_SEED)
        out["init"][kind] = state_digest(m.ViTND(**INIT_KWARGS).state_dict())
    for name, spec in VIT_ND_CASES.items():
        model = vit_nd_model(mods[spec["kind"]].ViTND, spec)
        x = vit_nd_input(spec)
        with torch.inference_mode():
            logits = model(x.float())
            embed = model(x.float(), return_embed=True) if spec["kind"] == "vit_nd_rotary" else None
        out["cases"][name] = {"spec": spec, "weights": weights_digest(model), "input": input_digest(x),
                              "logits_fp32": logits.clone(),
                              "embed0_fp32": None if embed is None else embed[:1].clone()}
        print(f"{name}: logits {tuple(logits.shape)} |max| {logits.abs().max():.4f}")
    path = os.path.join(HERE, "vit_nd.pt")
    torch.save(out, path)
    print(f"vit_nd: {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    main()
