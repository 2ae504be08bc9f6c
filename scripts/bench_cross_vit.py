"""Throughput of the fused CrossViT (vit_pytorch_b200.cross_vit) on one GPU.

    python scripts/bench_cross_vit.py [--steps 10] [--warmup 3] [--only NAME]

Prints one JSON line per workload:
  readme   the reference README's configuration: 256 x 256, sm patch 16 / lg patch 64, sm_dim 192 / lg_dim 384,
           depth 4, cross_attn_depth 2, 8 heads, mlp 2048, batch 256 (N = 257 / 17)
  small    CrossViT-S-like: 240 x 240, sm patch 12 / lg patch 16 (N = 401 / 226), sm 192 with 6 x 32 heads, lg 384 with
           6 x 64 heads, mlp ratio 3, lg_enc_depth 4, depth 3, cross_attn_depth 1, batch 256
  long     the readme configuration with sm patch 8 (N = 1025: the key-block attention), batch 64
  latency  the readme configuration at batch 8, replayed through graph.GraphedForward, against the eager bf16 graph
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
from vit_pytorch_b200.cross_vit import CrossViT  # noqa: E402
from vit_pytorch_b200.graph import GraphedForward  # noqa: E402

README = dict(image_size=256, num_classes=1000, depth=4, sm_dim=192, sm_patch_size=16, sm_enc_depth=2,
              sm_enc_heads=8, sm_enc_mlp_dim=2048, lg_dim=384, lg_patch_size=64, lg_enc_depth=3, lg_enc_heads=8,
              lg_enc_mlp_dim=2048, cross_attn_depth=2, cross_attn_heads=8, dropout=0.1, emb_dropout=0.1)
WORKLOADS = {
    "readme": dict(batch=256, kw=README),
    "small": dict(batch=256, kw=dict(image_size=240, num_classes=1000, depth=3, sm_dim=192, sm_patch_size=12,
                                     sm_enc_depth=1, sm_enc_heads=6, sm_enc_dim_head=32, sm_enc_mlp_dim=576,
                                     lg_dim=384, lg_patch_size=16, lg_enc_depth=4, lg_enc_heads=6, lg_enc_dim_head=64,
                                     lg_enc_mlp_dim=1152, cross_attn_depth=1, cross_attn_heads=6,
                                     cross_attn_dim_head=64, dropout=0., emb_dropout=0.)),
    "long": dict(batch=64, kw=dict(README, sm_patch_size=8)),
    "latency": dict(batch=8, kw=README, graphed=True),
}


def tokens(kw: dict) -> list:
    s = kw["image_size"]
    return [(s // kw["sm_patch_size"]) ** 2 + 1, (s // kw["lg_patch_size"]) ** 2 + 1]


def run(name: str, spec: dict, args, dev, info: dict) -> dict:
    B, kw = spec["batch"], spec["kw"]
    torch.manual_seed(1)
    x = torch.randn(B, 3, kw["image_size"], kw["image_size"], device=dev).bfloat16()
    torch.manual_seed(0)
    model = CrossViT(**kw).eval().to(dev, torch.bfloat16)
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
    res = {"workload": name, "model": "vit_pytorch_b200.cross_vit.CrossViT", "batch": B,
           "input": [3, kw["image_size"], kw["image_size"]], "tokens_sm_lg": tokens(kw),
           "cuda_graph": fused is not None,
           "fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
           "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 2), "eager_bf16_ms_per_step": round(ms_eager, 3),
           "speedup_vs_eager": round(ms_eager / ms, 3), "max_abs_logit_diff_fused_vs_eager": diff,
           "launches_per_step": launches, "kernels": kernel_breakdown(call), "steps": args.steps, "gpu": info}
    del fused, model
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=sorted(WORKLOADS), default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cross_vit.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    info = card()
    for name, spec in WORKLOADS.items():
        if args.only in (None, name):
            print(json.dumps(run(name, spec, args, dev, info)), flush=True)


if __name__ == "__main__":
    main()
