"""Generate tests/golden/twins_svt_schedule.json: the launch sequence of the whole fused Twins-SVT forward (four stages
of patch embedding, Transformer, PEG, Transformer, then the head), per LayerNorm mode, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_twins_svt_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder: every _lib entry point
the forward reaches is replaced by a recorder and torch.cuda.current_stream is stubbed, so TwinsSVT.forward_fused runs
on CPU tensors and nothing computes.  A tensor is stored as the input image (`img`), as a buffer of a stage's
workspace (`stage<i>.ws.<name>`; both Transformers of a stage share it), as a prepared weight (its key --
`merge<i>.*`, `peg<i>.*`, `stage<i>.t<1|2>.*`, `head.*` -- and a digest of its bytes), or as the k-th intermediate
buffer the forward allocated (`tmp<k>`).
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

FIXTURE = os.path.join(HERE, "twins_svt_schedule.json")
# entry points of the forward that make_engine_schedule.ENTRY_POINTS does not list
EXTRA_ENTRY_POINTS = ("patchify_ln", "embed_tokens", "merge_patches_ln", "peg", "attention_window", "attention_kv",
                      "conv_im2col_nhwc", "mean_pool")

# 16 x 8 (window 4, k 3: 5 x 2 keys) -> 8 x 4 (window 2, k 2) -> 4 x 2 (window 1, k 1: no im2col) -> 2 x 1 (k 1)
KWARGS = dict(num_classes=5, s1_emb_dim=16, s1_patch_size=2, s1_local_patch_size=4, s1_global_k=3, s1_depth=1,
              s2_emb_dim=24, s2_patch_size=2, s2_local_patch_size=2, s2_global_k=2, s2_depth=2,
              s3_emb_dim=32, s3_patch_size=2, s3_local_patch_size=1, s3_global_k=1, s3_depth=1,
              s4_emb_dim=40, s4_patch_size=2, s4_global_k=1, s4_depth=1, peg_kernel_size=3)
INPUT = (2, 3, 32, 16)
RUNS = [("fold", "python"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.twins_svt import TwinsSVT
    torch.manual_seed(seed)
    m = TwinsSVT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {}
        for i, (pe, t1, peg, t2) in enumerate(m.stages()):
            out.update({f"merge{i}.{k}": v for k, v in m._merge_weights(i, pe).items()})
            out.update({f"peg{i}.{k}": v for k, v in m._peg_weights(i, peg).items()})
            for j, t in ((1, t1), (2, t2)):
                out.update({f"stage{i}.t{j}.{k}": v for k, v in t.engine().prepared().items()})
        p = m.__dict__.get("_head_engine")
        if p is not None and isinstance(p.prep.t, dict):
            out.update({f"head.{k}": v for k, v in p.prep.t.items()})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"stage{i}.ws.{k}", v) for i, s in enumerate(model.stages())
                                 for k, v in s[1].engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"twins_svt four stages | {ln_mode} | {host_loop}"


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
