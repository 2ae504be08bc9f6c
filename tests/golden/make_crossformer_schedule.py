"""Generate tests/golden/crossformer_schedule.json: the launch sequence of the whole fused CrossFormer forward (the
stage-1 cross-scale embedding kernel, the later stages' per-scale im2col + GEMMs into the stream's column slices, every
stage's short- and long-distance window attention and feed-forward layers, the head), per LayerNorm mode, recorded on
CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_crossformer_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder, as make_cvt_schedule.py
uses it.  A tensor is stored as the input image (`img`), as a buffer of a stage's engine workspace
(`stage<i>.ws.<name>`), as a prepared weight (its key -- `embed<i>.*` from the stage's embedding, `stage<i>.*` from
the stage's engine, `head.*` -- and a digest of its bytes), or as the k-th intermediate buffer the forward allocated
(`tmp<k>`).
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

FIXTURE = os.path.join(HERE, "crossformer_schedule.json")
# entry points of the forward that make_engine_schedule.ENTRY_POINTS does not list
EXTRA_ENTRY_POINTS = ("cross_embed_nchw", "conv_im2col_nhwc", "attention_window_relpos", "mean_pool")

# a 64 x 64 image -> stage 1 16 x 16 (stem kernels 4 / 8, widths 16 / 16) -> 8 x 8 -> 4 x 4 -> 2 x 2, widths 32 / 32 /
# 48 / 64 (1, 1, 1 and 2 heads of 32), local windows 2, global 2 / 2 / 1 / 2, depth 1 per stage
KWARGS = dict(num_classes=5, dim=(32, 32, 48, 64), depth=(1, 1, 1, 1), global_window_size=(2, 2, 1, 2),
              local_window_size=2, cross_embed_kernel_sizes=((4, 8), (2, 4), (2, 4), (2, 4)))
INPUT = (2, 3, 64, 64)
RUNS = [("fold", "python"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.crossformer import CrossFormer
    torch.manual_seed(seed)
    m = CrossFormer(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {}
        for i, (cel, t) in enumerate(m.layers):
            out.update({f"embed{i}.{k}": v for k, v in m._embed_weights(i, cel).items()})
            out.update({f"stage{i}.{k}": v for k, v in t.engine().prepared().items()})
        p = m.__dict__.get("_head_engine")
        if p is not None and isinstance(p.prep.t, dict):
            out.update({f"head.{k}": v for k, v in p.prep.t.items()})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"stage{i}.ws.{k}", v) for i, (_, t) in enumerate(model.layers)
                                 for k, v in t.engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"crossformer four stages | {ln_mode} | {host_loop}"


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
