"""Generate tests/golden/pit_schedule.json: the launch sequence of the whole fused PiT forward (patch embedding, three
stages, two stage transitions, head), per LayerNorm mode and host loop, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_pit_schedule.py

The recording machinery is make_engine_schedule.recording, with this file's Recorder: every _lib entry point the
forward reaches is replaced by a recorder and torch.cuda.current_stream is stubbed, so PiT.forward_fused runs on CPU
tensors and nothing computes.  A tensor is stored as the input image (`img`), as a buffer of a stage's workspace
(`stage<i>.ws.<name>`), as a prepared weight (its key -- `patch.*`, `pool<i>.*`, `stage<i>.*`, `head.*` -- and a
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

from vit_pytorch_b200 import _lib  # noqa: E402

FIXTURE = os.path.join(HERE, "pit_schedule.json")
# entry points of the forward that TransformerEngine.run_blocks does not reach
EXTRA_ENTRY_POINTS = ("unfold_patches", "pit_pool", "embed_tokens")

# three stages: a 7 x 7 unfold grid (49 patches + cls) -> 4 x 4 -> 2 x 2; stage dims 16, 32, 64
KWARGS = dict(image_size=16, patch_size=4, num_classes=5, dim=16, depth=(1, 2, 1), heads=(1, 2, 2), mlp_dim=32,
              dim_head=32)
INPUT = (2, 3, 16, 16)
RUNS = [("fold", "c"), ("fold", "python"), ("exact", "python")]


def build(seed: int = 0):
    from vit_pytorch_b200.pit import PiT
    torch.manual_seed(seed)
    m = PiT(**KWARGS).eval()
    S.quantize_(m, seed)
    return m


class _Weights:
    """Every prepared weight of the model under one key space, for the recorder's weight look-up."""

    def __init__(self, model) -> None:
        self.model = model

    def prepared(self) -> Dict[str, torch.Tensor]:
        m = self.model
        out = {f"patch.{k}": v for k, v in m._patch_weights().items()}
        for i, pool in enumerate(m.pools()):
            out.update({f"pool{i}.{k}": v for k, v in m._pool_weights(i, pool).items()})
        for i, t in enumerate(m.stages()):
            out.update({f"stage{i}.{k}": v for k, v in t.engine().prepared().items()})
        for name in ("_head_norm", "_head_engine"):
            p = m.__dict__.get(name)
            t = None if p is None else (p.prep.t if name == "_head_engine" else p.t)
            if isinstance(t, dict):
                out.update({f"head.{k}": v for k, v in t.items()})
            elif isinstance(t, tuple):
                out.update({f"head.ln.{j}": v for j, v in enumerate(t)})
        return out


class Recorder(S.Recorder):
    """make_engine_schedule's Recorder, with every tensor that is neither an owner's nor a prepared weight named by
    the order in which the forward first passed its storage to the library (kept alive so no address is reused)."""

    def __init__(self, eng, owners) -> None:
        super().__init__(eng, owners)
        self.tmp: Dict[int, int] = {}
        self.alive: List[torch.Tensor] = []

    def tensor(self, t: torch.Tensor) -> dict:
        enc = super().tensor(t)
        if "role" in enc or enc["key"] is not None:
            return enc
        base = t.untyped_storage().data_ptr()
        if base not in self.tmp:
            self.tmp[base] = len(self.tmp)
            self.alive.append(t)
        return {"role": f"tmp{self.tmp[base]}", "offset": t.data_ptr() - base, "dtype": str(t.dtype).replace("torch.", ""),
                "shape": list(t.shape), "stride": list(t.stride())}


def record(ln_mode: str, host_loop: str) -> List[dict]:
    model = build()
    img = torch.zeros(*INPUT, dtype=torch.bfloat16)

    def owners():
        return [("img", img)] + [(f"stage{i}.ws.{k}", v) for i, t in enumerate(model.stages())
                                 for k, v in t.engine().slot.t.items()]
    with S.recording(_Weights(model), owners, ln_mode, host_loop, EXTRA_ENTRY_POINTS, Recorder) as rec:
        model.forward_fused(img)
    return rec.calls


def run_name(ln_mode: str, host_loop: str) -> str:
    return f"pit three stages | {ln_mode} | {host_loop}"


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
