"""Throughput of the fused DeepViT (vit_pytorch_b200.deepvit) on one GPU.

    python scripts/bench_deepvit.py [--steps 10] [--warmup 3] [--only NAME]

Prints one JSON line per workload:
  readme   the reference README's configuration: 256 x 256, patch 32, dim 1024, depth 6, 16 x 64 heads, mlp 2048,
           batch 256 (N = 65)
  p16      the same model at 224 x 224 with patch 16 (N = 197), batch 256
  dh48     224 x 224 / 16, dim 384, depth 24, 8 x 48 heads, mlp 1536 (CaiT-S24's encoder shape), batch 256
  latency  the readme configuration at batch 8, replayed through graph.GraphedForward, against the eager bf16 graph
--torch-profile runs instead one torch.profiler step per workload (a separate run, since tracing slows the host) and
prints the head-mixing kernel's share of the step's CUDA time.
Each line: fused images/s, the module's own eager bf16 graph on the same GPU, their largest logit difference, ms per
step, launches and share of every library kernel (per-call CUDA events in a separate profiled step), with the card's
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
from vit_pytorch_b200.deepvit import DeepViT  # noqa: E402
from vit_pytorch_b200.graph import GraphedForward  # noqa: E402

README = dict(image_size=256, patch_size=32, num_classes=1000, dim=1024, depth=6, heads=16, mlp_dim=2048, dropout=0.1,
              emb_dropout=0.1)
WORKLOADS = {
    "readme": dict(batch=256, kw=README),
    "p16": dict(batch=256, kw=dict(README, image_size=224, patch_size=16)),
    "dh48": dict(batch=256, kw=dict(image_size=224, patch_size=16, num_classes=1000, dim=384, depth=24, heads=8,
                                    dim_head=48, mlp_dim=1536)),
    "latency": dict(batch=8, kw=README, graphed=True),
}


def tokens(kw: dict) -> int:
    return (kw["image_size"] // kw["patch_size"]) ** 2 + 1


def qk_recompute(kw: dict) -> int:
    """How many times the head-mixing kernel computes QK^T relative to plain attention: 3 ceil(H / 2G), G output heads
    per warpgroup (hm_group in csrc/headmix.cu)."""
    H, dh = kw["heads"], kw.get("dim_head", 64)
    hc = 4 if H <= 4 else 8 if (H <= 8 or dh == 128) else 16
    if hc == 4:
        G = 2
    elif hc == 8:
        G = 4 if dh <= 64 else 1 if dh == 128 else 2
    else:
        G = 4 if dh <= 32 else 2 if dh <= 64 else 1
    return 3 * -(-H // (2 * G))


def torch_profile(name: str, spec: dict, dev, info: dict) -> dict:
    """One profiled fused step (after a warm-up step): the share of CUDA time spent in the head-mixing kernel."""
    B, kw = spec["batch"], spec["kw"]
    torch.manual_seed(1)
    x = torch.randn(B, 3, kw["image_size"], kw["image_size"], device=dev).bfloat16()
    torch.manual_seed(0)
    model = DeepViT(**kw).eval().to(dev, torch.bfloat16)
    fused = GraphedForward(model, x) if spec.get("graphed") else None
    with torch.inference_mode():
        step = (lambda: fused(x)) if fused is not None else (lambda: model(x))
        step()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
    total = mix = 0.0
    for e in prof.key_averages():
        t = e.device_time_total
        total += t
        if "attention_headmix" in e.key:
            mix += t
    del fused, model
    torch.cuda.empty_cache()
    return {"workload": name, "batch": B, "tokens": tokens(kw), "cuda_graph": spec.get("graphed", False),
            "headmix_ms": round(mix / 1e3, 3), "cuda_ms": round(total / 1e3, 3),
            "headmix_share_of_cuda_time": round(mix / total, 4) if total else None,
            "qk_recompute_vs_plain_attention": qk_recompute(kw), "gpu": info}


def run(name: str, spec: dict, args, dev, info: dict) -> dict:
    B, kw = spec["batch"], spec["kw"]
    torch.manual_seed(1)
    x = torch.randn(B, 3, kw["image_size"], kw["image_size"], device=dev).bfloat16()
    torch.manual_seed(0)
    model = DeepViT(**kw).eval().to(dev, torch.bfloat16)
    with torch.inference_mode():
        reason = model.fused_reason(x)
    assert reason is None, reason
    call = lambda: model(x)                       # noqa: E731
    fused = GraphedForward(model, x) if spec.get("graphed") else None
    step = (lambda: fused(x)) if fused is not None else call
    ms = timed(step, args.steps, args.warmup)
    with torch.inference_mode():
        out = step().float().clone()
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
    res = {"workload": name, "model": "vit_pytorch_b200.deepvit.DeepViT", "batch": B,
           "input": [3, kw["image_size"], kw["image_size"]], "tokens": tokens(kw),
           "cuda_graph": fused is not None,
           "fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
           "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 2), "eager_bf16_ms_per_step": round(ms_eager, 3),
           "speedup_vs_eager": round(ms_eager / ms, 3), "max_abs_logit_diff_fused_vs_eager": diff,
           "qk_recompute_vs_plain_attention": qk_recompute(kw), "launches_per_step": launches,
           "kernels": kernel_breakdown(call), "steps": args.steps, "gpu": info}
    del fused, model
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
        raise SystemExit("bench_deepvit.py measures the GPU path and needs a CUDA device")
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
