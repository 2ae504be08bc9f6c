"""Generate tests/golden/levit_schedule.json: the launch sequence of the whole fused LeViT forward (the four-convolution
stem, every Transformer layer's five launches, the head), per LayerNorm setting, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_levit_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder: every _lib entry point
the forward reaches is replaced by a recorder and torch.cuda.current_stream is stubbed, so LeViT.forward_fused runs on
CPU tensors and nothing computes.  A tensor is stored as the input image (`img`), as a prepared weight (its key in
LeViT.prepared() and a digest of its bytes), or as the k-th intermediate buffer the forward allocated (`tmp<k>`).
LeViT has no LayerNorm, so both settings of B200VIT_LN_MODE record the same sequence.
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

FIXTURE = os.path.join(HERE, "levit_schedule.json")
# entry points of the forward that make_engine_schedule.ENTRY_POINTS does not list
EXTRA_ENTRY_POINTS = ("conv_im2col_nchw", "conv_im2col_nhwc", "attention_posbias", "gemm_hardswish", "mean_pool",
                      "cast_f32_bf16")

# 7 -> 4 -> 2 (an odd grid; the downsampling layers take 49 -> 16 and 16 -> 4 queries), a distill head
KWARGS = dict(image_size=112, num_classes=5, dim=(32, 48, 64), depth=(1, 2, 1), heads=(2, 3, 4), mlp_mult=2,
              dim_key=16, dim_value=32, num_distill_classes=3)
INPUT = (2, 3, 112, 112)
RUNS = [("fold", "python"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.levit import LeViT
    torch.manual_seed(seed)
    m = LeViT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)
    with S.recording(model, lambda: [("img", img)], ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"levit three stages | {ln_mode} | {host_loop}"


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
