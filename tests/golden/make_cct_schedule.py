"""Generate tests/golden/cct_schedule.json: the launch sequence of the whole fused CCT forward (two tokenizer blocks,
token assembly, two post-norm encoder layers, sequence pooling, classifier), per LayerNorm mode and host loop, recorded
on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_cct_schedule.py

The recording machinery is make_engine_schedule.recording, with make_pit_schedule.py's Recorder: every _lib entry
point the forward reaches is replaced by a recorder and torch.cuda.current_stream is stubbed, so CCT.forward_fused
runs on CPU tensors and nothing computes.  A tensor is stored as the input image (`img`), as a buffer of the
classifier's workspace (`ws.<name>`), as a prepared weight (its key -- `conv<i>`, `seq.*`, `enc.*`, `head.*` -- and a
digest of its bytes), or as the k-th intermediate buffer the forward allocated (`tmp<k>`), with byte offset, shape and
stride.
"""
from __future__ import annotations

import os
import sys
from typing import Dict, List

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_engine_schedule as S  # noqa: E402
import make_pit_schedule as PS  # noqa: E402

from vit_pytorch_b200 import _lib  # noqa: E402

FIXTURE = os.path.join(HERE, "cct_schedule.json")
# entry points of the forward that TransformerEngine.run_blocks does not reach
EXTRA_ENTRY_POINTS = ("conv_im2col_nchw", "conv_im2col_nhwc", "relu_maxpool", "embed_tokens", "seq_pool")

# 20 x 12 image, k3 s1 p1: 20 x 12 conv -> 10 x 6 pool -> 10 x 6 conv (64 -> 32 channels) -> 5 x 3 pool: 15 tokens
KWARGS = dict(img_size=(20, 12), embedding_dim=32, n_conv_layers=2, kernel_size=3, stride=1, padding=1, num_layers=2,
              num_heads=1, mlp_ratio=2, num_classes=5)
INPUT = (2, 3, 20, 12)
RUNS = PS.RUNS


def build(seed: int = 0):
    from vit_pytorch_b200.cct import CCT
    torch.manual_seed(seed)
    m = CCT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {f"conv{i}": m._conv_weights(i, blk[0]) for i, blk in enumerate(m.tokenizer.conv_layers)}
        out.update({f"seq.{k}": v for k, v in m._pool_weights().items() if isinstance(v, torch.Tensor)})
        out.update({f"enc.{k}": v for k, v in m.classifier.engine().prepared().items()})
        he = m.__dict__.get("_head_engine")
        if he is not None and isinstance(he.prep.t, dict):
            out.update({f"head.{k}": v for k, v in he.prep.t.items()})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"ws.{k}", v) for k, v in model.classifier.engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, PS.Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"cct two conv blocks | {ln_mode} | {host_loop}"


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
