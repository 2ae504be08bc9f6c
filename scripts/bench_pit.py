"""Throughput of the fused PiT (vit_pytorch_b200.pit) on one GPU.

    python scripts/bench_pit.py [--steps 10] [--warmup 3] [--only NAME] [--torch-profile]

Prints one JSON line per workload, batch 256 each:
  readme   the reference README's configuration: 224 x 224 / 14 (a 31 x 31 unfold grid, 962 tokens in stage 1), dim 256,
           depth (3, 3, 3), 16 x 64 heads, mlp 2048
  pit_b    PiT-B-like: 224 x 224 / 14, dim 256, depth (3, 6, 4), heads (4, 8, 16) x 64, mlp 1024
  pit_ti   PiT-Ti-like: 224 x 224 / 14, dim 64, depth (2, 6, 4), heads (2, 4, 8) x 32, mlp 256
Each line: fused images/s, the module's own eager bf16 graph on the same GPU, their largest logit difference, ms per
step, launches and share of every library kernel (per-call CUDA events in a separate profiled step), with the card's
name and power limit read in the same run.  --torch-profile runs instead one torch.profiler step per workload (a
separate run, since tracing slows the host) and splits the step's CUDA time between the unfold, the pool, attention and
the GEMMs.  Writes nothing.
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
from vit_pytorch_b200.pit import PiT  # noqa: E402

WORKLOADS = {
    "readme": dict(batch=256, kw=dict(image_size=224, patch_size=14, num_classes=1000, dim=256, depth=(3, 3, 3),
                                      heads=16, mlp_dim=2048, dropout=0.1, emb_dropout=0.1)),
    "pit_b": dict(batch=256, kw=dict(image_size=224, patch_size=14, num_classes=1000, dim=256, depth=(3, 6, 4),
                                     heads=(4, 8, 16), dim_head=64, mlp_dim=1024)),
    "pit_ti": dict(batch=256, kw=dict(image_size=224, patch_size=14, num_classes=1000, dim=64, depth=(2, 6, 4),
                                      heads=(2, 4, 8), dim_head=32, mlp_dim=256)),
}


def patches(kw: dict) -> int:
    p = kw["patch_size"]
    return ((kw["image_size"] - p) // (p // 2) + 1) ** 2


def _model_and_input(spec: dict, dev):
    B, kw = spec["batch"], spec["kw"]
    torch.manual_seed(1)
    x = torch.randn(B, 3, kw["image_size"], kw["image_size"], device=dev).bfloat16()
    torch.manual_seed(0)
    return PiT(**kw).eval().to(dev, torch.bfloat16), x


def torch_profile(name: str, spec: dict, dev, info: dict) -> dict:
    """One profiled fused step (after a warm-up step): CUDA time per kernel family."""
    model, x = _model_and_input(spec, dev)
    with torch.inference_mode():
        model(x)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            model(x)
            torch.cuda.synchronize()
    split = {"unfold": 0.0, "pit_pool": 0.0, "attention": 0.0, "gemm": 0.0}
    total = 0.0
    for e in prof.key_averages():
        t = e.device_time_total
        total += t
        if "unfold_kernel" in e.key:
            split["unfold"] += t
        elif "pit_pool_kernel" in e.key:
            split["pit_pool"] += t
        elif "attn" in e.key or "attention" in e.key:
            split["attention"] += t
        elif "gemm" in e.key:
            split["gemm"] += t
    del model
    torch.cuda.empty_cache()
    return {"workload": name, "batch": spec["batch"], "patches": patches(spec["kw"]), "cuda_ms": round(total / 1e3, 3),
            **{f"{k}_ms": round(v / 1e3, 3) for k, v in split.items()},
            **{f"{k}_share": round(v / total, 4) if total else None for k, v in split.items()}, "gpu": info}


def run(name: str, spec: dict, args, dev, info: dict) -> dict:
    B, kw = spec["batch"], spec["kw"]
    model, x = _model_and_input(spec, dev)
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
    os.environ["B200VIT_DISABLE_FUSED"] = "1"     # the module's own PyTorch graph, every submodule included
    try:
        ms_eager = timed(call, max(3, args.steps // 2), 2)
        with torch.inference_mode():
            diff = (model(x).float() - out).abs().max().item()
    finally:
        del os.environ["B200VIT_DISABLE_FUSED"]
    res = {"workload": name, "model": "vit_pytorch_b200.pit.PiT", "batch": B,
           "input": [3, kw["image_size"], kw["image_size"]], "patches": patches(kw),
           "fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
           "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 2), "eager_bf16_ms_per_step": round(ms_eager, 3),
           "speedup_vs_eager": round(ms_eager / ms, 3), "max_abs_logit_diff_fused_vs_eager": diff,
           "launches_per_step": launches, "kernels": kernel_breakdown(call), "steps": args.steps, "gpu": info}
    del model
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=sorted(WORKLOADS), default=None)
    ap.add_argument("--torch-profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pit.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    info = card()
    for name, spec in WORKLOADS.items():
        if args.only in (None, name):
            res = torch_profile(name, spec, dev, info) if args.torch_profile else run(name, spec, args, dev, info)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
