"""Generate tests/golden/cvt_schedule.json: the launch sequence of the whole fused CvT forward (each stage's
convolutional embedding and channel LayerNorm, its layers' convolutional projections, attention and feed-forward
blocks, the head), per LayerNorm mode, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_cvt_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder: every _lib entry point
the forward reaches is replaced by a recorder and torch.cuda.current_stream is stubbed, so CvT.forward_fused runs on
CPU tensors and nothing computes.  A tensor is stored as the input image (`img`), as a buffer of a stage's engine
workspace (`stage<i>.ws.<name>`), as a prepared weight (its key -- `embed<i>.*` from the stage's embedding,
`stage<i>.*` from the stage's engine, `head.*` -- and a digest of its bytes), or as the k-th intermediate buffer the
forward allocated (`tmp<k>`).
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

FIXTURE = os.path.join(HERE, "cvt_schedule.json")
# entry points of the forward that make_engine_schedule.ENTRY_POINTS does not list
EXTRA_ENTRY_POINTS = ("conv_im2col_nchw", "conv_im2col_nhwc", "embed_tokens", "conv_proj_dw", "attention_kv",
                      "mean_pool")

# a 24 x 20 image -> stage 1 6 x 5 (k 3, kv stride 2: 3 x 3 keys) -> stage 2 3 x 3 (depth 2, k 5, kv stride 1: 3 x 3)
# -> stage 3 2 x 2 (k 1, kv stride 2: 1 x 1), widths 16 / 32 / 48, 2 heads of 64, mlp_mult 2
KWARGS = dict(num_classes=5, s1_emb_dim=16, s1_heads=2, s1_mlp_mult=2, s2_emb_dim=32, s2_heads=2, s2_depth=2,
              s2_proj_kernel=5, s2_kv_proj_stride=1, s2_mlp_mult=2, s3_emb_dim=48, s3_heads=2, s3_depth=1,
              s3_proj_kernel=1, s3_mlp_mult=2)
INPUT = (2, 3, 24, 20)
RUNS = [("fold", "python"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.cvt import CvT
    torch.manual_seed(seed)
    m = CvT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {}
        for i, stage in enumerate(m.layers):
            out.update({f"embed{i}.{k}": v for k, v in m._embed_weights(i, stage).items()})
            out.update({f"stage{i}.{k}": v for k, v in stage[2].engine().prepared().items()})
        p = m.__dict__.get("_head_engine")
        if p is not None and isinstance(p.prep.t, dict):
            out.update({f"head.{k}": v for k, v in p.prep.t.items()})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"stage{i}.ws.{k}", v) for i, s in enumerate(model.layers)
                                 for k, v in s[2].engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"cvt three stages | {ln_mode} | {host_loop}"


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
