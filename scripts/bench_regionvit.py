"""Throughput of the fused RegionViT (vit_pytorch_b200.regionvit) on one GPU.

    python scripts/bench_regionvit.py [--steps 10] [--warmup 3] [--batch 64]

Prints one JSON line: the README RegionViT (dim 64 / 128 / 256 / 512, depth 2 / 2 / 8 / 2, window 7, one-conv local
tokenizer, no PEG) at 224 x 224 in bf16 -- local maps 56, 28, 14 and 7 over region maps 8, 4, 2 and 1, 7 x 7 windows
throughout.  Fused images/s with eager launches and with the whole forward replayed through GraphedForward, the
module's own eager bf16 graph on the same GPU, the largest logit difference, ms per step, launches and the share of
every library kernel (per-call CUDA events in a separate profiled step).  For every attention_region_local launch of
that step: its time, the bytes it must move and that rate as a share of 3.35 TB/s (the H100 SXM's HBM3 bandwidth).
The card's name and power limit are read in the same run.  Writes nothing.
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
from vit_pytorch_b200.regionvit import RegionViT  # noqa: E402

IMAGE = 224
README = dict(dim=(64, 128, 256, 512), depth=(2, 2, 8, 2), window_size=7, num_classes=1000,
              tokenize_local_3_conv=False, use_peg=False)
HBM_BYTES_PER_S = 3.35e12
NEW_KERNELS = ("attention_region_local",)


def new_kernels(call) -> list:
    """Per launch of the new kernels in one profiled step: shape, time, bytes and the share of HBM bandwidth."""
    with torch.inference_mode():
        call()
        torch.cuda.synchronize()
        _lib.profile_start()
        call()
        rec = _lib.profile_stop()
    out = []
    for name, meta, ms in rec:
        if name not in NEW_KERNELS:
            continue
        gbs = meta["bytes"] / (ms * 1e-3) / 1e9
        out.append({"kernel": name, **{k: v for k, v in meta.items() if k != "bytes"}, "us": round(ms * 1e3, 2),
                    "bytes": meta["bytes"], "GB_per_s": round(gbs, 1),
                    "share_of_3.35TBps": round(gbs * 1e9 / HBM_BYTES_PER_S, 3)})
    return out


def run(args, dev, info: dict) -> dict:
    B = args.batch
    torch.manual_seed(1)
    x = torch.randn(B, 3, IMAGE, IMAGE, device=dev).bfloat16()
    torch.manual_seed(0)
    model = RegionViT(**README).eval().to(dev, torch.bfloat16)
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
    del fwd
    os.environ["B200VIT_DISABLE_FUSED"] = "1"     # the module's own PyTorch graph, every submodule included
    try:
        ms_eager = timed(call, max(3, args.steps // 2), 2)
        with torch.inference_mode():
            diff = (model(x).float() - out).abs().max().item()
    finally:
        del os.environ["B200VIT_DISABLE_FUSED"]
    return {"workload": "regionvit_readme_224", "model": "vit_pytorch_b200.regionvit.RegionViT", "batch": B,
            "input": [3, IMAGE, IMAGE], "stage_maps": [list(m) for m in model.stage_maps(IMAGE, IMAGE)],
            "config": {**README, "dim": list(README["dim"]), "depth": list(README["depth"])},
            "fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
            "fused_graph_images_per_s": round(B / ms_graph * 1e3, 2), "fused_graph_ms_per_step": round(ms_graph, 3),
            "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 2), "eager_bf16_ms_per_step": round(ms_eager, 3),
            "speedup_vs_eager": round(ms_eager / ms, 3), "graph_speedup_vs_eager": round(ms_eager / ms_graph, 3),
            "max_abs_logit_diff_fused_vs_eager": diff, "max_abs_logit_diff_graph_vs_launches": graph_diff,
            "launches_per_step": launches, "kernels": kernel_breakdown(call), "new_kernels": new_kernels(call),
            "steps": args.steps, "gpu": info}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_regionvit.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    print(json.dumps(run(args, dev, card())), flush=True)


if __name__ == "__main__":
    main()
