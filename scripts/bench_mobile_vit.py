"""Throughput of the fused MobileViT (vit_pytorch_b200.mobile_vit) on one GPU.

    python scripts/bench_mobile_vit.py [--steps 10] [--warmup 3] [--batch 256]

Prints one JSON line: the README mbvit_xs (dims 96 / 120 / 144, channels 16 32 48 48 64 64 80 80 96 96 384, expansion
4, patch 2 x 2, depths 2 / 4 / 3) at 256 x 256 in bf16 -- MobileViT block maps 32 x 32, 16 x 16 and 8 x 8, groups of
256, 64 and 16 tokens.  Fused images/s with eager launches and with the whole forward replayed through GraphedForward,
the module's own eager bf16 graph on the same GPU, the largest logit differences, ms per step, launches and the share
of every library kernel (per-call CUDA events in a separate profiled step); for every attention_groups launch its time
and the exponential floor: n^2 exponentials per (group, head) at 16 per SM per clock, over the SM count and the SM
clock read in the same run.  The card's name and power limit are read in the same run.  Writes nothing.
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
from vit_pytorch_b200.mobile_vit import MobileViT  # noqa: E402

IMAGE = 256
README = dict(image_size=(256, 256), dims=[96, 120, 144], channels=[16, 32, 48, 48, 64, 64, 80, 80, 96, 96, 384],
              num_classes=1000)
EX2_PER_SM_PER_CLOCK = 16          # MUFU throughput of an sm_90 SM (CUDA C++ Programming Guide, arithmetic throughput)


def sm_clock_mhz() -> float:
    """The SM clock the card runs at now, from nvidia-smi (0 if it cannot be read)."""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                               # noqa: BLE001
        return 0.0


def group_attention(call, dev) -> list:
    """Per attention_groups launch of one profiled step: its shape, time and the exponential floor."""
    with torch.inference_mode():
        call()
        torch.cuda.synchronize()
        _lib.profile_start()
        call()
        clock = sm_clock_mhz()
        rec = _lib.profile_stop()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    out = []
    for name, meta, ms in rec:
        if name != "attention_groups":
            continue
        floor_us = meta["exps"] / (EX2_PER_SM_PER_CLOCK * sms * clock * 1e6) * 1e6 if clock else None
        out.append({"map": [meta["h"], meta["w"]], "tokens_per_group": meta["n"], "us": round(ms * 1e3, 2),
                    "exps": meta["exps"], "sm_clock_mhz": clock,
                    "ex2_floor_us": None if floor_us is None else round(floor_us, 2),
                    "share_of_floor": None if floor_us is None else round(floor_us / (ms * 1e3), 3)})
    return out


def run(args, dev, info: dict) -> dict:
    B = args.batch
    torch.manual_seed(1)
    x = torch.randn(B, 3, IMAGE, IMAGE, device=dev).bfloat16()
    torch.manual_seed(0)
    model = MobileViT(**README).eval().to(dev, torch.bfloat16)
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
    return {"workload": "mobile_vit_readme_xs", "model": "vit_pytorch_b200.mobile_vit.MobileViT", "batch": B,
            "input": [3, IMAGE, IMAGE], "block_maps": [32, 16, 8], "config": README,
            "fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
            "fused_graph_images_per_s": round(B / ms_graph * 1e3, 2), "fused_graph_ms_per_step": round(ms_graph, 3),
            "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 2), "eager_bf16_ms_per_step": round(ms_eager, 3),
            "speedup_vs_eager": round(ms_eager / ms, 3), "graph_speedup_vs_eager": round(ms_eager / ms_graph, 3),
            "max_abs_logit_diff_fused_vs_eager": diff, "max_abs_logit_diff_graph_vs_launches": graph_diff,
            "launches_per_step": launches, "kernels": kernel_breakdown(call),
            "attention_groups": group_attention(call, dev), "steps": args.steps, "gpu": info}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mobile_vit.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    print(json.dumps(run(args, dev, card())), flush=True)


if __name__ == "__main__":
    main()
