"""Generate tests/golden/max_vit_schedule.json: the launch sequence of the whole fused MaxViT forward (the stem, every
block's MBConv with squeeze-excitation, block and grid attention with their feed-forward blocks, the head), per
LayerNorm mode, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_max_vit_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder: every _lib entry point
the forward reaches is replaced by a recorder and torch.cuda.current_stream is stubbed, so MaxViT.forward_fused runs
on CPU tensors and nothing computes.  A tensor is stored as the input image (`img`), as a buffer of a block's engine
workspace (`block<i>.ws.<name>`; the blocks of a stage share one), as a prepared weight (its key -- `mbconv.*` from
MaxViT.prepared(), `block<i>.*` from the block's engine, `head.*` -- and a digest of its bytes), or as the k-th
intermediate buffer the forward allocated (`tmp<k>`).
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

FIXTURE = os.path.join(HERE, "max_vit_schedule.json")
# entry points of the forward that make_engine_schedule.ENTRY_POINTS does not list
EXTRA_ENTRY_POINTS = ("conv_im2col_nchw", "conv_im2col_nhwc", "mbconv_dwconv", "se_pool", "gemm_silu", "gemm_sigmoid",
                      "se_scale", "attention_window_relpos", "mean_pool")

# a 32 x 16 image -> stem 16 x 8 -> stage 1 8 x 4 (two blocks: the second adds its MBConv into the stream) -> stage 2
# 4 x 2, window 2, widths 32 and 64, hidden widths 64 and 128, squeeze widths 32 and 64
KWARGS = dict(num_classes=5, dim=32, depth=(2, 1), dim_head=32, dim_conv_stem=8, window_size=2,
              mbconv_expansion_rate=2, mbconv_shrinkage_rate=0.5)
INPUT = (2, 3, 32, 16)
RUNS = [("fold", "python"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.max_vit import MaxViT
    torch.manual_seed(seed)
    m = MaxViT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {f"mbconv.{k}": v for k, v in m.prepared().items()}
        for i, e in enumerate(m._encoders()):
            out.update({f"block{i}.{k}": v for k, v in e.engine().prepared().items()})
        for name in ("_head_norm", "_head_engine"):
            p = m.__dict__.get(name)
            t = None if p is None else (p.prep.t if name == "_head_engine" else p.t)
            if isinstance(t, dict):
                out.update({f"head.{k}": v for k, v in t.items()})
            elif isinstance(t, tuple):
                out.update({f"head.ln.{j}": v for j, v in enumerate(t)})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"block{i}.ws.{k}", v) for i, e in enumerate(model._encoders())
                                 for k, v in e.engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"max_vit two stages | {ln_mode} | {host_loop}"


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
