"""Throughput of the fused CvT (vit_pytorch_b200.cvt) on one GPU.

    python scripts/bench_cvt.py [--steps 10] [--warmup 3] [--batch 64]

Prints one JSON line: the README CvT (emb_dim 64 / 192 / 384, depth 1 / 2 / 10, heads 1 / 3 / 4, 3 x 3 projections,
key / value stride 2) at 224 x 224 in bf16 -- maps 56 x 56, 28 x 28 and 14 x 14 with 784, 196 and 49 keys.  Fused
images/s with eager launches and with the whole forward replayed through GraphedForward, the module's own eager bf16
graph on the same GPU, the largest logit differences, ms per step, launches and the share of every library kernel
(per-call CUDA events in a separate profiled step; conv_proj_dw is the depthwise projection kernel), with the card's
name and power limit read in the same run.  Writes nothing.
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
from vit_pytorch_b200.cvt import CvT  # noqa: E402
from vit_pytorch_b200.graph import GraphedForward  # noqa: E402

IMAGE = 224
README = dict(num_classes=1000, s1_emb_dim=64, s1_emb_kernel=7, s1_emb_stride=4, s1_proj_kernel=3,
              s1_kv_proj_stride=2, s1_heads=1, s1_depth=1, s1_mlp_mult=4, s2_emb_dim=192, s2_emb_kernel=3,
              s2_emb_stride=2, s2_proj_kernel=3, s2_kv_proj_stride=2, s2_heads=3, s2_depth=2, s2_mlp_mult=4,
              s3_emb_dim=384, s3_emb_kernel=3, s3_emb_stride=2, s3_proj_kernel=3, s3_kv_proj_stride=2, s3_heads=4,
              s3_depth=10, s3_mlp_mult=4, dropout=0.)


def run(args, dev, info: dict) -> dict:
    B = args.batch
    torch.manual_seed(1)
    x = torch.randn(B, 3, IMAGE, IMAGE, device=dev).bfloat16()
    torch.manual_seed(0)
    model = CvT(**README).eval().to(dev, torch.bfloat16)
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
    return {"workload": "cvt_readme", "model": "vit_pytorch_b200.cvt.CvT", "batch": B, "input": [3, IMAGE, IMAGE],
            "maps": [56, 28, 14], "keys": [784, 196, 49], "config": dict(README),
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
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cvt.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    print(json.dumps(run(args, dev, card())), flush=True)


if __name__ == "__main__":
    main()
