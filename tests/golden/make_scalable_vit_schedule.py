"""Generate tests/golden/scalable_vit_schedule.json: the launch sequence of the whole fused ScalableViT forward (the
patch convolution, every stage's encoder layers and PEG, the Downsample convolutions between stages, the head), per
LayerNorm mode and host loop, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_scalable_vit_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder, as
make_sep_vit_schedule.py uses it.  A tensor is stored as the input image (`img`), as a buffer of a stage's engine
workspace (`stage<i>.ws.<name>`), as a prepared weight (its key -- `model.*` from the model's own weights,
`stage<i>.*` from the stage transformer's engine, `head.*` -- and a digest of its bytes), or as the k-th intermediate
buffer the forward allocated (`tmp<k>`).  Stage 1 is the README's: a 64 x 64 map whose IWSA attends over 64 x 64
windows with heads 32 wide and whose SSA attends over 8 x 8 keys with dim_key 40, run at 48, and value heads 32 wide.
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

FIXTURE = os.path.join(HERE, "scalable_vit_schedule.json")
# entry points of the forward that make_engine_schedule.ENTRY_POINTS does not list
EXTRA_ENTRY_POINTS = ("conv_im2col_nchw", "conv_im2col_nhwc", "attention_kv_ex", "attention_iwsa", "peg",
                      "mean_pool")

# a 256 x 256 image -> maps 64 x 64 and 32 x 32; stage 1 as the README's (2 heads, ssa_dim_key 40, reduction 8,
# whole-map windows), stage 2 with 4 heads, reduction 4, 16 x 16 windows and two layers
KWARGS = dict(num_classes=5, dim=64, heads=(2, 4), depth=(1, 2), ssa_dim_key=40, reduction_factor=(8, 4),
              window_size=(64, 16))
INPUT = (2, 3, 256, 256)
RUNS = [("fold", "c"), ("fold", "python"), ("exact", "c"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.scalable_vit import ScalableViT
    torch.manual_seed(seed)
    m = ScalableViT(**KWARGS).eval()
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
            out.update({f"stage{i}.{k}": v for k, v in tr.engine().prepared().items()})
            out.update({f"stage{i}.peg.{k}": v for k, v in tr.peg_weights().items()})
        p = m.__dict__.get("_head_engine")
        if p is not None and isinstance(getattr(p, "prep", p).t, (dict, tuple)):
            t = getattr(p, "prep", p).t
            out.update({f"head.{k}": v for k, v in (t.items() if isinstance(t, dict) else enumerate(t))})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"stage{i}.ws.{k}", v) for i, (tr, _) in enumerate(model.layers)
                                 for k, v in tr.engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"scalable_vit two stages | {ln_mode} | {host_loop}"


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
