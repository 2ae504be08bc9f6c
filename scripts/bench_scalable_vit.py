"""Throughput of the fused ScalableViT (vit_pytorch_b200.scalable_vit) on one GPU.

    python scripts/bench_scalable_vit.py [--steps 10] [--warmup 3] [--batch 64]

Prints one JSON line: the README ScalableViT-S (dim 64, heads 2 / 4 / 8 / 16, depth 2 / 2 / 20 / 2, ssa_dim_key
40 / 40 / 40 / 32, reduction 8 / 4 / 2 / 1, window 64 / 32 / None / None) at 256 x 256 in bf16 -- stage maps 64, 32,
16 and 8, every IWSA window the whole map.  Fused images/s with eager launches and replayed through GraphedForward,
the module's own eager bf16 graph on the same GPU, the largest logit difference, ms per step, launches and the share
of every library kernel (per-call CUDA events in a separate profiled step).  For every attention_iwsa and
attention_kv_ex launch of that step: its time, FLOPs from the shapes, TFLOP/s and their share of 989 TFLOP/s (the
H100 SXM's dense BF16 figure), and its bytes.  The yardstick: attention_iwsa on the stage-1 whole-map shape
(4096 tokens, 2 heads of 32) alternated in the same process with b200vit_attention_kv over the same qkv (q the first
I columns, k | v the rest, Nq = Nk = 4096), which does the same arithmetic but the LIM add; medians of three rounds.
The card's name and power limit are read in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_vit_small_dataset import card, kernel_breakdown, timed  # noqa: E402
from vit_pytorch_b200 import _lib  # noqa: E402
from vit_pytorch_b200.graph import GraphedForward  # noqa: E402
from vit_pytorch_b200.scalable_vit import ScalableViT  # noqa: E402

IMAGE = 256
README = dict(num_classes=1000, dim=64, heads=(2, 4, 8, 16), depth=(2, 2, 20, 2), ssa_dim_key=(40, 40, 40, 32),
              reduction_factor=(8, 4, 2, 1), window_size=(64, 32, None, None))
BF16_FLOPS = 989e12
NEW_KERNELS = ("attention_iwsa", "attention_kv_ex")


def new_kernels(call) -> list:
    """Per launch of the new kernels in one profiled step: shape, time, FLOPs, TFLOP/s, share of peak, bytes."""
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
        tfs = meta["flops"] / (ms * 1e-3) / 1e12
        out.append({"kernel": name, **{k: v for k, v in meta.items() if k not in ("bytes", "flops")},
                    "us": round(ms * 1e3, 2), "flops": meta["flops"], "TFLOP_per_s": round(tfs, 1),
                    "share_of_989TFLOPs": round(tfs * 1e12 / BF16_FLOPS, 3), "bytes": meta["bytes"]})
    return out


def yardstick(B: int, dev) -> dict:
    """attention_iwsa on the stage-1 whole-map shape against attention_kv over the same qkv, alternated."""
    gh = gw = IMAGE // 4
    H, d = 2, 32
    N, I = gh * gw, H * d
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = torch.randn(B * N, 3 * I, device=dev, generator=g).bfloat16()
    lim = torch.randn(B * N, I, device=dev, generator=g).bfloat16()
    o1, o2 = torch.empty(B * N, I, device=dev, dtype=torch.bfloat16), torch.empty(B * N, I, device=dev,
                                                                                 dtype=torch.bfloat16)
    iwsa = lambda: _lib.attention_iwsa(qkv, lim, o1, B, gh, gw, gh, gw, H, d, d, d ** -0.5)       # noqa: E731
    kv = lambda: _lib.attention_kv(qkv[:, :I], qkv[:, I:], o2, B, N, N, H, d, d ** -0.5)          # noqa: E731
    rounds = {"attention_iwsa": [], "attention_kv": []}
    for _ in range(3):
        for name, f in (("attention_iwsa", iwsa), ("attention_kv", kv)):
            rounds[name].append(timed(f, 20, 3))
    med = {k: statistics.median(v) for k, v in rounds.items()}
    flops = 4.0 * B * H * N * N * d
    return {"shape": {"B": B, "map": [gh, gw], "H": H, "dk": d, "dv": d},
            **{f"{k}_ms": round(v, 4) for k, v in med.items()},
            **{f"{k}_TFLOP_per_s": round(flops / (v * 1e-3) / 1e12, 1) for k, v in med.items()},
            "iwsa_over_kv_time": round(med["attention_iwsa"] / med["attention_kv"], 3),
            "rounds_ms": {k: [round(x, 4) for x in v] for k, v in rounds.items()}}


def run(args, dev, info: dict) -> dict:
    B = args.batch
    torch.manual_seed(1)
    x = torch.randn(B, 3, IMAGE, IMAGE, device=dev).bfloat16()
    torch.manual_seed(0)
    model = ScalableViT(**README).eval().to(dev, torch.bfloat16)
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
    return {"workload": "scalable_vit_s_readme_256", "model": "vit_pytorch_b200.scalable_vit.ScalableViT", "batch": B,
            "input": [3, IMAGE, IMAGE], "stage_maps": [64, 32, 16, 8],
            "config": {k: list(v) if isinstance(v, tuple) else v for k, v in README.items()},
            "fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
            "fused_graph_images_per_s": round(B / ms_graph * 1e3, 2), "fused_graph_ms_per_step": round(ms_graph, 3),
            "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 2), "eager_bf16_ms_per_step": round(ms_eager, 3),
            "speedup_vs_eager": round(ms_eager / ms, 3), "graph_speedup_vs_eager": round(ms_eager / ms_graph, 3),
            "max_abs_logit_diff_fused_vs_eager": diff, "max_abs_logit_diff_graph_vs_launches": graph_diff,
            "launches_per_step": launches, "kernels": kernel_breakdown(call), "new_kernels": new_kernels(call),
            "yardstick": yardstick(B, dev), "steps": args.steps, "gpu": info}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_scalable_vit.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    print(json.dumps(run(args, dev, card())), flush=True)


if __name__ == "__main__":
    main()
