"""Throughput of the fused N-dimensional ViTs (vit_pytorch_b200.vit_nd / vit_nd_rotary) on one GPU.

    python scripts/bench_vit_nd.py [--steps 10] [--warmup 3] [--only NAME]

Prints one JSON line per workload:
  rot_2d   rotary ViTND, rank 2: 224 x 224, patch 16, ViT-B dims, batch 512 -- next to vit_pytorch_b200.ViT ViT-B/16
           at the same batch (the cost of the rotary pass against the learned-table model)
  rot_3d   rotary ViTND, rank 3: video 16 x 224 x 224, patch 2 x 16 x 16, ViT-B dims, batch 32 (N = 1568: the
           key-block attention path)
  nd_1d    ViTND, rank 1: 3 x 4096 signal, patch 16, ViT-B dims, batch 256
Each line: fused images/s, the module's own eager bf16 graph on the same GPU, their largest logit difference, ms per
step and GB/s of rope_qk and patchify_nd (library per-call CUDA events in a separate profiled step; bytes from the
shapes, see _lib), the card's name and power limit read in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from vit_pytorch_b200 import ViT, _lib  # noqa: E402
from vit_pytorch_b200.vit_nd import ViTND  # noqa: E402
from vit_pytorch_b200.vit_nd_rotary import ViTND as RotaryViTND  # noqa: E402

VIT_B = dict(dim=768, depth=12, heads=12, mlp_dim=3072, num_classes=1000)
WORKLOADS = {
    "rot_2d": dict(cls=RotaryViTND, batch=512, kw=dict(ndim=2, input_shape=224, patch_size=16, **VIT_B),
                   shape=(3, 224, 224), twin_vit=True),
    "rot_3d": dict(cls=RotaryViTND, batch=32, kw=dict(ndim=3, input_shape=(16, 224, 224), patch_size=(2, 16, 16),
                                                      **VIT_B), shape=(3, 16, 224, 224)),
    "nd_1d": dict(cls=ViTND, batch=256, kw=dict(ndim=1, input_shape=4096, patch_size=16, **VIT_B),
                  shape=(3, 4096)),
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
    """One profiled step: per library kernel name, ms per step, launches and GB/s (bytes from the shapes)."""
    with torch.inference_mode():
        _lib.profile_start()
        fn()
        rec = _lib.profile_stop()
    agg: dict = {}
    for name, meta, ms in rec:
        a = agg.setdefault(name, {"ms_per_step": 0.0, "launches": 0, "bytes": 0.0})
        a["ms_per_step"] += ms
        a["launches"] += 1
        a["bytes"] += float(meta.get("bytes", 0.0))
    total = sum(a["ms_per_step"] for a in agg.values())
    out = {}
    for name in ("rope_qk", "patchify_nd"):
        if name in agg:
            a = agg[name]
            out[name] = {"ms_per_step": round(a["ms_per_step"], 4), "launches": a["launches"],
                         "GB_per_step": round(a["bytes"] / 1e9, 3),
                         "GB_per_s": round(a["bytes"] / (a["ms_per_step"] / 1e3) / 1e9, 1),
                         "share_of_profiled_step": round(a["ms_per_step"] / total, 4)}
    return out


def run(name: str, spec: dict, args, dev, info: dict) -> dict:
    torch.manual_seed(0)
    model = spec["cls"](**spec["kw"]).eval().to(dev, torch.bfloat16)
    B = spec["batch"]
    torch.manual_seed(1)
    x = torch.randn(B, *spec["shape"], device=dev).bfloat16()
    with torch.inference_mode():
        reason = model.fused_reason(x)
    assert reason is None, reason
    fused = lambda: model(x)                      # noqa: E731
    ms = timed(fused, args.steps, args.warmup)
    with torch.inference_mode():
        out = model(x).float()
    # the module's own PyTorch graph, every submodule included (the Transformer would otherwise dispatch fused)
    os.environ["B200VIT_DISABLE_FUSED"] = "1"
    try:
        ms_eager = timed(fused, max(3, args.steps // 2), 2)
        with torch.inference_mode():
            diff = (model(x).float() - out).abs().max().item()
    finally:
        del os.environ["B200VIT_DISABLE_FUSED"]
    line = {"workload": name, "model": f"{spec['cls'].__module__}.ViTND", "batch": B, "input": list(spec["shape"]),
            "tokens": model._nd_engine.tokens(x)[1], "fused_images_per_s": round(B / ms * 1e3, 1),
            "fused_ms_per_step": round(ms, 3), "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 1),
            "eager_bf16_ms_per_step": round(ms_eager, 3), "speedup_vs_eager": round(ms_eager / ms, 3),
            "max_abs_logit_diff_fused_vs_eager": diff, "kernels": kernel_breakdown(fused),
            "steps": args.steps, "gpu": info}
    del model
    if spec.get("twin_vit"):
        torch.manual_seed(0)
        vit = ViT(image_size=224, patch_size=16, **VIT_B).eval().to(dev, torch.bfloat16)
        ms_vit = timed(lambda: vit(x), args.steps, args.warmup)
        line["vit_b16_same_batch"] = {"fused_images_per_s": round(B / ms_vit * 1e3, 1),
                                      "fused_ms_per_step": round(ms_vit, 3)}
        del vit
    torch.cuda.empty_cache()
    return line


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=sorted(WORKLOADS), default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vit_nd.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    info = card()
    for name, spec in WORKLOADS.items():
        if args.only in (None, name):
            print(json.dumps(run(name, spec, args, dev, info)), flush=True)


if __name__ == "__main__":
    main()
