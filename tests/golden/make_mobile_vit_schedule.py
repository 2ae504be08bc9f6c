"""Generate tests/golden/mobile_vit_schedule.json: the launch sequence of the whole fused MobileViT forward (conv1,
the MV2Blocks, every MobileViT block's local convolutions, its transformer layers over strided patch groups and its
fusion, the head), per LayerNorm mode and host loop, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_mobile_vit_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder, as
make_crossformer_schedule.py uses it.  A tensor is stored as the input image (`img`), as a buffer of a block's engine
workspace (`block<i>.ws.<name>`), as a prepared weight (its key -- `model.*` from the model's convolutions,
`block<i>.*` from the block transformer's engine, `head.*` -- and a digest of its bytes), or as the k-th intermediate
buffer the forward allocated (`tmp<k>`).  The patch-group layers never take the one-call C layer loop, so both host
loops record the same sequence.
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

FIXTURE = os.path.join(HERE, "mobile_vit_schedule.json")
# entry points of the forward that make_engine_schedule.ENTRY_POINTS does not list
EXTRA_ENTRY_POINTS = ("gemm_act", "conv_im2col_nchw", "conv_im2col_nhwc", "mbconv_dwconv_ex", "attention_groups", "mean_pool")

# a 64 x 64 image -> conv1 32 x 32 -> stem 16 x 16 -> blocks 8 x 8, 4 x 4, 2 x 2 (groups of 16, 4, 1 tokens); stem.0
# adds its input (channels[0] == channels[1]), expansion 2, depth 1 per block
KWARGS = dict(image_size=(64, 64), dims=(32, 40, 48), channels=[16, 16, 24, 24, 32, 32, 40, 40, 48, 48, 96],
              num_classes=5, expansion=2, depths=(1, 1, 1))
INPUT = (2, 3, 64, 64)
RUNS = [("fold", "c"), ("fold", "python"), ("exact", "c"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.mobile_vit import MobileViT
    torch.manual_seed(seed)
    m = MobileViT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {f"model.{k}": v for k, v in m.prepared().items()}
        for i, (_, blk) in enumerate(m.trunk):
            out.update({f"block{i}.{k}": v for k, v in blk.transformer.engine().prepared().items()})
        p = m.__dict__.get("_head_engine")
        if p is not None and isinstance(p.prep.t, dict):
            out.update({f"head.{k}": v for k, v in p.prep.t.items()})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"block{i}.ws.{k}", v) for i, (_, blk) in enumerate(model.trunk)
                                 for k, v in blk.transformer.engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"mobile_vit three blocks | {ln_mode} | {host_loop}"


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
