"""Throughput of the fused LeViT (vit_pytorch_b200.levit) on one GPU.

    python scripts/bench_levit.py [--steps 10] [--warmup 3] [--batch 256]

Prints one JSON line: the README configuration (dim 256 / 384 / 512, depth 4, heads 4 / 6 / 8, mlp_mult 2, dim_key 32,
dim_value 64) at 224 x 224 in bf16 -- grids 14 x 14, 7 x 7 and 4 x 4, downsampling attention 196 -> 49 and 49 -> 16
queries.  Fused images/s with eager launches and with the whole forward replayed through GraphedForward, the module's
own eager bf16 graph on the same GPU, the largest logit differences, ms per step, launches and the share of every
library kernel (per-call CUDA events in a separate profiled step), with the card's name and power limit read in the
same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_vit_small_dataset import card, kernel_breakdown, timed  # noqa: E402
from vit_pytorch_b200 import _lib  # noqa: E402
from vit_pytorch_b200.graph import GraphedForward  # noqa: E402
from vit_pytorch_b200.levit import LeViT  # noqa: E402

IMAGE = 224
README = dict(image_size=224, num_classes=1000, stages=3, dim=(256, 384, 512), depth=4, heads=(4, 6, 8), mlp_mult=2,
              dropout=0.1)


def run(args, dev, info: dict) -> dict:
    B = args.batch
    torch.manual_seed(1)
    x = torch.randn(B, 3, IMAGE, IMAGE, device=dev).bfloat16()
    torch.manual_seed(0)
    model = LeViT(**README).eval().to(dev, torch.bfloat16)
    with torch.inference_mode():
        reason = model.fused_reason(x)
    assert reason is None, reason
    call = lambda: model(x)                       # noqa: E731
    ms = timed(call, args.steps, args.warmup)
    with torch.inference_mode():
        out = call().float().clone()
        _lib.reset_launch_count()
        call()
        torch.cuda.synchronize()
        launches = _lib.launch_count()
    fwd = GraphedForward(model, x)
    ms_graph = timed(lambda: fwd(x), args.steps, args.warmup)
    graph_diff = (fwd(x).float() - out).abs().max().item()
    os.environ["B200VIT_DISABLE_FUSED"] = "1"     # the module's own PyTorch graph, every submodule included
    try:
        ms_eager = timed(call, max(3, args.steps // 2), 2)
        with torch.inference_mode():
            diff = (model(x).float() - out).abs().max().item()
    finally:
        del os.environ["B200VIT_DISABLE_FUSED"]
    return {"workload": "levit_readme", "model": "vit_pytorch_b200.levit.LeViT", "batch": B,
            "input": [3, IMAGE, IMAGE], "grids": [14, 7, 4], "config": {k: v for k, v in README.items()},
            "fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
            "fused_graph_images_per_s": round(B / ms_graph * 1e3, 2), "fused_graph_ms_per_step": round(ms_graph, 3),
            "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 2), "eager_bf16_ms_per_step": round(ms_eager, 3),
            "speedup_vs_eager": round(ms_eager / ms, 3), "graph_speedup_vs_eager": round(ms_eager / ms_graph, 3),
            "max_abs_logit_diff_fused_vs_eager": diff, "max_abs_logit_diff_graph_vs_launches": graph_diff,
            "launches_per_step": launches, "kernels": kernel_breakdown(call), "steps": args.steps, "gpu": info}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_levit.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    print(json.dumps(run(args, dev, card())), flush=True)


if __name__ == "__main__":
    main()
