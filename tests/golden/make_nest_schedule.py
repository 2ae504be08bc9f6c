"""Generate tests/golden/nest_schedule.json: the launch sequence of the whole fused NesT forward (the patch embedding,
every level's entry and encoder layers, the Aggregate convolutions between levels, the head), per LayerNorm mode and
host loop, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_nest_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder, as
make_sep_vit_schedule.py uses it.  A tensor is stored as the input image (`img`), as a buffer of a level's engine
workspace (`level<i>.ws.<name>`), as a prepared weight (its key -- `model.*` from the model's own weights,
`level<i>.*` from the level transformer's engine, `head.*` -- and a digest of its bytes), or as the k-th intermediate
buffer the forward allocated (`tmp<k>`).  Every level attends over blocks of 196 tokens with heads 32 wide, the
lengths the persistent attention kernel runs.
"""
from __future__ import annotations

import os
import sys
from typing import Dict, List

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_engine_schedule as S  # noqa: E402
from make_pit_schedule import Recorder  # noqa: E402

from vit_pytorch_b200 import _lib  # noqa: E402

FIXTURE = os.path.join(HERE, "nest_schedule.json")
# entry points of the forward that make_engine_schedule.ENTRY_POINTS does not list
EXTRA_ENTRY_POINTS = ("patchify_ln", "nest_level_entry", "nest_im2col", "mean_pool")

# a 112 x 112 image, patch 2 -> maps 56 x 56 (4 x 4 blocks), 28 x 28 (2 x 2), 14 x 14: 196-token blocks at widths
# 32, 64 and 128 with 1, 2 and 4 heads of 32; the last level has two layers
KWARGS = dict(image_size=112, patch_size=2, dim=32, heads=1, num_hierarchies=3, block_repeats=(1, 1, 2), num_classes=5)
INPUT = (2, 3, 112, 112)
RUNS = [("fold", "c"), ("fold", "python"), ("exact", "c"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.nest import NesT
    torch.manual_seed(seed)
    m = NesT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {f"model.{k}": v for k, v in m.prepared().items()}
        for i, (tr, _) in enumerate(m.layers):
            out.update({f"level{i}.{k}": v for k, v in tr.engine().prepared().items()})
        p = m.__dict__.get("_head_engine")
        if p is not None and isinstance(getattr(p, "prep", p).t, (dict, tuple)):
            t = getattr(p, "prep", p).t
            out.update({f"head.{k}": v for k, v in (t.items() if isinstance(t, dict) else enumerate(t))})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"level{i}.ws.{k}", v) for i, (tr, _) in enumerate(model.layers)
                                 for k, v in tr.engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"nest three levels | {ln_mode} | {host_loop}"


def generate() -> Dict[str, List[dict]]:
    return {run_name(m, h): record(m, h) for m, h in RUNS}


if __name__ == "__main__":
    if not _lib.LIB_PATH.exists():
        from vit_pytorch_b200 import build as _build
        _build.build()
    text = S.dumps(generate())
    with open(FIXTURE, "w") as f:
        f.write(text)
    print(f"wrote {FIXTURE} ({len(text)} bytes)")
