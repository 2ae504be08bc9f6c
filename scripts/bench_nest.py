"""Throughput of the fused NesT (vit_pytorch_b200.nest) on one GPU.

    python scripts/bench_nest.py [--workload readme|hier4] [--steps 10] [--warmup 3] [--batch 64]

Prints one JSON line for one workload at 224 x 224 in bf16:
  * readme: the README NesT-T (dim 96, heads 3, num_hierarchies 3, block_repeats (2, 2, 8)): maps 56, 28 and 14 in
    4 x 4, 2 x 2 and 1 blocks, every level attending over 196-token blocks (the persistent attention kernel's range);
  * hier4: the same with num_hierarchies 4 and block_repeats (2, 2, 2, 8): maps 56, 28, 14 and 7 in 8 x 8, 4 x 4,
    2 x 2 and 1 blocks of 7 x 7 = 49 tokens, which fill 49 of the attention kernel's 128 query rows -- its
    `attention` share is the number that decides whether short blocks should be packed into 64-row tiles.
Fused images/s with eager launches and with the whole forward replayed through GraphedForward, the module's own eager
bf16 graph on the same GPU, the largest logit difference, ms per step, launches and the share of every library kernel
(per-call CUDA events in a separate profiled step).  For every nest_level_entry and nest_im2col launch of that step:
its time, the bytes it must move and that rate as a share of 3.35 TB/s (the H100 SXM's HBM3 bandwidth).  The card's
name and power limit are read in the same run.  Writes nothing.
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
from vit_pytorch_b200.nest import NesT  # noqa: E402

IMAGE = 224
README = dict(image_size=IMAGE, patch_size=4, dim=96, heads=3, num_hierarchies=3, block_repeats=(2, 2, 8),
              num_classes=1000)
WORKLOADS = {
    "readme": (README, [(56, 4), (28, 2), (14, 1)]),
    "hier4": (dict(README, num_hierarchies=4, block_repeats=(2, 2, 2, 8)), [(56, 8), (28, 4), (14, 2), (7, 1)]),
}
HBM_BYTES_PER_S = 3.35e12
NEW_KERNELS = ("nest_level_entry", "nest_im2col")


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
    config, levels = WORKLOADS[args.workload]
    model = NesT(**config).eval().to(dev, torch.bfloat16)
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
    return {"workload": f"nest_{args.workload}_224", "model": "vit_pytorch_b200.nest.NesT", "batch": B,
            "input": [3, IMAGE, IMAGE],
            "levels": [{"map": m, "blocks": f"{nb} x {nb}", "tokens_per_block": (m // nb) ** 2} for m, nb in levels],
            "config": {**config, "block_repeats": list(config["block_repeats"])},
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
    ap.add_argument("--workload", choices=sorted(WORKLOADS), default="readme")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nest.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    print(json.dumps(run(args, dev, card())), flush=True)


if __name__ == "__main__":
    main()
