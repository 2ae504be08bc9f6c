"""Generate tests/golden/regionvit_schedule.json: the launch sequence of the whole fused RegionViT forward (the
3-conv local tokenizer, the region patches, the shared downsampling convolutions, the PEGs, every stage's R2L layers,
the head), per LayerNorm mode and host loop, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_regionvit_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder, as
make_mobile_vit_schedule.py uses it.  A tensor is stored as the input image (`img`), as a buffer of a stage's engine
workspace (`stage<i>.ws.<name>`), as a prepared weight (its key -- `model.*` from the model's convolutions,
`stage<i>.*` from the stage transformer's engine, `head.*` -- and a digest of its bytes), or as the k-th intermediate
buffer the forward allocated (`tmp<k>`).  The region-to-local layers never take the one-call C layer loop, so both
host loops record the same sequence.
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

FIXTURE = os.path.join(HERE, "regionvit_schedule.json")
# entry points of the forward that make_engine_schedule.ENTRY_POINTS does not list
EXTRA_ENTRY_POINTS = ("conv_im2col_nchw", "conv_im2col_nhwc", "peg", "patchify_nd", "head_layernorm_gelu",
                      "attention_region_local", "mean_pool")

# a 112 x 56 image -> local / region maps 28 x 14 / 4 x 2, 14 x 7 / 2 x 1, 7 x 4 / 1 x 1, 4 x 2 / 1 x 1: windows
# 7 x 7, 7 x 7, 7 x 4 and 4 x 2; the second stage has two layers
KWARGS = dict(num_classes=5, dim=(32, 32, 64, 64), depth=(1, 2, 1, 1), tokenize_local_3_conv=True, use_peg=True)
INPUT = (2, 3, 112, 56)
RUNS = [("fold", "c"), ("fold", "python"), ("exact", "c"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.regionvit import RegionViT
    torch.manual_seed(seed)
    m = RegionViT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {f"model.{k}": v for k, v in m.prepared().items()}
        for i, (_, _, tr) in enumerate(m.layers):
            out.update({f"stage{i}.{k}": v for k, v in tr.engine().prepared().items()})
        for name in ("_head_engine", "_head_norm"):
            p = m.__dict__.get(name)
            if p is not None and isinstance(getattr(p, "prep", p).t, (dict, tuple)):
                t = getattr(p, "prep", p).t
                out.update({f"head.{name}.{k}": v for k, v in (t.items() if isinstance(t, dict) else enumerate(t))})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"stage{i}.ws.{k}", v) for i, (_, _, tr) in enumerate(model.layers)
                                 for k, v in tr.engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"regionvit 112 x 56 | {ln_mode} | {host_loop}"


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
