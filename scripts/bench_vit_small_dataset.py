"""Throughput of the fused ViT for small datasets (vit_pytorch_b200.vit_for_small_dataset) on one GPU.

    python scripts/bench_vit_small_dataset.py [--steps 10] [--warmup 3] [--only NAME]

Prints one JSON line per workload:
  readme   the reference README's configuration: 256 x 256, patch 16, dim 1024, depth 6, heads 16, mlp 2048,
           batch 256 (N = 257)
  cifar    32 x 32, patch 4, dim 512, depth 6, heads 8, mlp 512, batch 1024 (N = 65)
  long     224 x 224, patch 8, dim 384, depth 6, heads 6, mlp 1536, batch 64 (N = 785: the key-block attention)
Each line: fused images/s, the module's own eager bf16 graph on the same GPU, their largest logit difference, ms per
step, launches and share of every library kernel (per-call CUDA events in a separate profiled step), and beside it
vit_pytorch_b200.ViT at the same dims -- what the 5x-wider shifted-patch GEMM and the self mask cost over plain ViT --
with the card's name and power limit read in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from vit_pytorch_b200 import ViT as PlainViT, _lib  # noqa: E402
from vit_pytorch_b200.vit_for_small_dataset import ViT  # noqa: E402

WORKLOADS = {
    "readme": dict(batch=256, size=256, kw=dict(image_size=256, patch_size=16, num_classes=1000, dim=1024, depth=6,
                                                heads=16, mlp_dim=2048)),
    "cifar": dict(batch=1024, size=32, kw=dict(image_size=32, patch_size=4, num_classes=10, dim=512, depth=6, heads=8,
                                               mlp_dim=512)),
    "long": dict(batch=64, size=224, kw=dict(image_size=224, patch_size=8, num_classes=1000, dim=384, depth=6, heads=6,
                                             mlp_dim=1536)),
}


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception as e:  # noqa: BLE001  (reported, not fatal)
        out["power_limit_w"] = f"unavailable: {type(e).__name__}"
    return out


def timed(fn, steps: int, warmup: int) -> float:
    """ms per call, CUDA events around `steps` calls after `warmup` calls."""
    with torch.inference_mode():
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def kernel_breakdown(fn) -> dict:
    """One profiled step: per library kernel name, ms per step, launches, GB/s and TFLOP/s (from the shapes)."""
    with torch.inference_mode():
        _lib.profile_start()
        fn()
        rec = _lib.profile_stop()
    agg: dict = {}
    for name, meta, ms in rec:
        a = agg.setdefault(name, {"ms_per_step": 0.0, "launches": 0, "bytes": 0.0, "flops": 0.0})
        a["ms_per_step"] += ms
        a["launches"] += 1
        a["bytes"] += float(meta.get("bytes", 0.0))
        a["flops"] += float(meta.get("flops", 0.0))
    total = sum(a["ms_per_step"] for a in agg.values())
    out = {}
    for name, a in sorted(agg.items(), key=lambda kv: -kv[1]["ms_per_step"]):
        e = {"ms_per_step": round(a["ms_per_step"], 4), "launches": a["launches"],
             "share_of_profiled_step": round(a["ms_per_step"] / total, 4)}
        if a["bytes"]:
            e["GB_per_step"] = round(a["bytes"] / 1e9, 3)
            e["GB_per_s"] = round(a["bytes"] / (a["ms_per_step"] / 1e3) / 1e9, 1)
        if a["flops"]:
            e["TFLOP_per_s"] = round(a["flops"] / (a["ms_per_step"] / 1e3) / 1e12, 1)
        out[name] = e
    return out


def measure(model, x, args) -> dict:
    with torch.inference_mode():
        reason = model.fused_reason(x)
    assert reason is None, reason
    fused = lambda: model(x)                      # noqa: E731
    ms = timed(fused, args.steps, args.warmup)
    with torch.inference_mode():
        out = model(x).float()
        _lib.reset_launch_count()
        model(x)
        torch.cuda.synchronize()
        launches = _lib.launch_count()
    # the module's own PyTorch graph, every submodule included (the Transformer would otherwise dispatch fused)
    os.environ["B200VIT_DISABLE_FUSED"] = "1"
    try:
        ms_eager = timed(fused, max(3, args.steps // 2), 2)
        with torch.inference_mode():
            diff = (model(x).float() - out).abs().max().item()
    finally:
        del os.environ["B200VIT_DISABLE_FUSED"]
    B = x.shape[0]
    return {"fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
            "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 2), "eager_bf16_ms_per_step": round(ms_eager, 3),
            "speedup_vs_eager": round(ms_eager / ms, 3), "max_abs_logit_diff_fused_vs_eager": diff,
            "launches_per_step": launches, "kernels": kernel_breakdown(fused)}


def run(name: str, spec: dict, args, dev, info: dict) -> dict:
    B, S = spec["batch"], spec["size"]
    torch.manual_seed(1)
    x = torch.randn(B, 3, S, S, device=dev).bfloat16()
    torch.manual_seed(0)
    model = ViT(**spec["kw"]).eval().to(dev, torch.bfloat16)
    small = measure(model, x, args)
    del model
    torch.cuda.empty_cache()
    torch.manual_seed(0)
    plain = PlainViT(**spec["kw"]).eval().to(dev, torch.bfloat16)
    base = measure(plain, x, args)
    del plain
    torch.cuda.empty_cache()
    n = (S // spec["kw"]["patch_size"]) ** 2 + 1
    return {"workload": name, "model": "vit_pytorch_b200.vit_for_small_dataset.ViT", "batch": B,
            "input": [3, S, S], "tokens": n, **small,
            "plain_vit": {"model": "vit_pytorch_b200.ViT", **base},
            "fused_time_vs_plain_vit": round(small["fused_ms_per_step"] / base["fused_ms_per_step"], 3),
            "steps": args.steps, "gpu": info}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=sorted(WORKLOADS), default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vit_small_dataset.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    info = card()
    for name, spec in WORKLOADS.items():
        if args.only in (None, name):
            print(json.dumps(run(name, spec, args, dev, info)), flush=True)


if __name__ == "__main__":
    main()
