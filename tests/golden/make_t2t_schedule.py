"""Generate tests/golden/t2t_schedule.json: the launch sequence of the whole fused T2T-ViT forward (three soft splits --
a narrow one on the key-block attention and a wide one on b200vit_attention_wide -- the final Linear, the cls row and
positions, the main encoder and the head), per LayerNorm mode and host loop, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_t2t_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder: every _lib entry point the
forward reaches is replaced by a recorder and torch.cuda.current_stream is stubbed, so T2TViT.forward_fused runs on CPU
tensors and nothing computes.  A tensor is stored as the input image (`img`), as a buffer of the main encoder's
workspace (`main.ws.<name>`), as a prepared weight (its key -- `split<i>.*`, `embed.*`, `main.*`, `head.*` -- and a
digest of its bytes), or as the k-th intermediate buffer the forward allocated (`tmp<k>`), with byte offset, shape and
stride, so the fixture pins which buffer every call reads and writes.
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

FIXTURE = os.path.join(HERE, "t2t_schedule.json")
# entry points of the forward that TransformerEngine.run_blocks does not reach
EXTRA_ENTRY_POINTS = ("t2t_unfold_image", "t2t_unfold_tokens", "attention_wide", "embed_tokens", "mean_pool")

# soft splits 8 x 8 (27 wide: the key-block attention at dp 32) -> 4 x 4 (243 wide: the wide attention at dp 256) ->
# 2 x 2 (2187, the final Linear); main encoder dim 32, one layer, 1 x 32 heads
KWARGS = dict(image_size=16, num_classes=5, dim=32, depth=1, heads=1, dim_head=32, mlp_dim=64,
              t2t_layers=((3, 2), (3, 2), (3, 2)))
INPUT = (2, 3, 16, 16)
RUNS = [("fold", "c"), ("fold", "python"), ("exact", "c"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.t2t import T2TViT
    torch.manual_seed(seed)
    m = T2TViT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


def _flat(prefix: str, t: dict) -> Dict[str, torch.Tensor]:
    out = {}
    for k, v in t.items():
        if isinstance(v, torch.Tensor):
            out[f"{prefix}.{k}"] = v
        elif isinstance(v, tuple):
            out.update({f"{prefix}.{k}.{j}": e for j, e in enumerate(v) if isinstance(e, torch.Tensor)})
    return out


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {}
        for i, t in enumerate(m.soft_splits()):
            if t is not None:
                out.update(_flat(f"split{i}", m._split_weights(i, t)))
        out.update(_flat("embed", m._embed_weights()))
        out.update({f"main.{k}": v for k, v in m.transformer.engine().prepared().items()})
        he = m.__dict__.get("_head_engine")
        if he is not None and isinstance(he.prep.t, dict):
            out.update({f"head.{k}": v for k, v in he.prep.t.items()})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"main.ws.{k}", v) for k, v in model.transformer.engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, PS.Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"t2t three soft splits | {ln_mode} | {host_loop}"


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
