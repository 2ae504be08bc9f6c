"""Generate tests/golden/ats_vit_schedule.json: the launch sequence of the whole fused Adaptive Token Sampling ViT
forward -- patch embedding and token assembly, a plain layer, a layer that may sample (LN1 + QKV, select, gather,
attention of the kept queries, out-projection, feed-forward), a later layer that cannot sample (attention with the
queries read in place), the head -- per LayerNorm mode and host loop, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_ats_vit_schedule.py

The recording machinery is make_engine_schedule.recording with make_pit_schedule's Recorder: every _lib entry point the
forward reaches is replaced by a recorder and torch.cuda.current_stream is stubbed, so ViT.forward_fused runs on CPU
tensors and nothing computes.  A tensor is stored as the input image (`img`), as a buffer of the encoder's workspace
(`ws.<name>`), of the sampling layers' scratch (`scratch.<name>`) or of the starting lengths and ids (`start.<name>`),
as a prepared weight (its key -- `main.*`, `patch.*`, `head.*`, `head_norm.*` -- and a digest of its bytes), or as the
k-th intermediate buffer the forward allocated (`tmp<k>`: the stream, the uniforms, the pooled rows, the logits), with
byte offset, shape and stride, so the fixture pins which buffer, which rows and which statistics slot every call
reads and writes.
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

FIXTURE = os.path.join(HERE, "ats_vit_schedule.json")
# entry points of the forward that TransformerEngine.run_blocks does not reach
EXTRA_ENTRY_POINTS = ("patchify_ln", "embed_tokens", "ats_select", "ats_gather", "attention_kv_lens")

# 4 x 4 patches + cls = 17 rows per image: layer 0 (K = 16) cannot sample and runs through run_blocks; layer 1 (K = 8)
# may sample, 17 -> 9 rows; layer 2 (K = 8) cannot sample any more, 9 rows with the queries in place
KWARGS = dict(image_size=32, patch_size=8, num_classes=5, dim=32, depth=3, max_tokens_per_depth=(16, 8, 8), heads=1,
              dim_head=32, mlp_dim=64)
INPUT = (2, 3, 32, 32)
RUNS = [("fold", "c"), ("fold", "python"), ("exact", "c")]


def build(seed: int = 0):
    from vit_pytorch_b200.ats_vit import ViT
    torch.manual_seed(seed)
    m = ViT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {f"main.{k}": v for k, v in m.transformer.engine().prepared().items()}
        pe = m.__dict__.get("_patch_engine")
        if pe is not None and isinstance(pe.prep.t, dict):
            out.update({f"patch.{k}": v for k, v in pe.prep.t.items()})
        he = m.__dict__.get("_head_engine")
        if he is not None and isinstance(he.prep.t, dict):
            out.update({f"head.{k}": v for k, v in he.prep.t.items()})
        hn = m.__dict__.get("_head_norm")
        if hn is not None and hn.t is not None:
            out.update({f"head_norm.{j}": v for j, v in enumerate(hn.t)})
        return out


def record(ln_mode: str, host_loop: str) -> List[dict]:
    import vit_pytorch_b200.ats_vit as A
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        out = [("img", img)] + [(f"ws.{k}", v) for k, v in model.transformer.engine().slot.t.items()]
        for key, v in model._cu.items():
            if isinstance(v, dict):
                out += [(f"scratch.{k}", e) for k, e in v.items() if isinstance(e, torch.Tensor)]
                out += [(f"scratch.{k}{j}", e) for k, e in v.items() if isinstance(e, list) for j, e in enumerate(e)]
            else:
                out += [("start.lens", v[0]), ("start.ids", v[1])]
        return out
    saved = A.draw_uniform
    A.draw_uniform = lambda shape, device, dtype, layer: torch.zeros(shape, device=device, dtype=dtype)
    try:
        with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, PS.Recorder) as rec:
            model.forward_fused(img)
    finally:
        A.draw_uniform = saved
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"ats_vit plain, sampling and padded layers | {ln_mode} | {host_loop}"


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
