"""Throughput of the fused CCT (vit_pytorch_b200.cct) on one GPU.

    python scripts/bench_cct.py [--steps 10] [--warmup 3] [--only NAME]

Prints one JSON line per workload:
  readme   the reference README's CCT(...): 224 x 448, two conv blocks k7 s2 p3 (3 -> 64 -> 384), 392 tokens, dim 384,
           14 layers, 6 heads, mlp ratio 3, learnable table; batch 256
  cct_14   the README's cct_14: 224 x 224, one conv block k7 s2 p3, 3136 tokens, dim 384; batch 256
  cifar    cct_7(img_size=32, kernel_size=3, n_conv_layers=1): 256 tokens, dim 256, 7 layers, 4 heads; batch 1024
Each line: fused images/s, the module's own eager bf16 graph on the same GPU, their largest logit difference, ms per
step, launches, and the share of the profiled step (per-call CUDA events) taken by each kernel family -- the tokenizer
(im2col, conv GEMMs, ReLU max-pool), token assembly, attention, the encoder GEMMs and LayerNorms, sequence pooling, the
classifier -- with the card's name and power limit read in the same run.  Writes nothing.
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
from vit_pytorch_b200.cct import CCT, cct_7, cct_14  # noqa: E402

WORKLOADS = {
    "readme": dict(batch=256, size=(224, 448), make=CCT,
                   kw=dict(img_size=(224, 448), embedding_dim=384, n_conv_layers=2, kernel_size=7, stride=2, padding=3,
                           pooling_kernel_size=3, pooling_stride=2, pooling_padding=1, num_layers=14, num_heads=6,
                           mlp_ratio=3., num_classes=1000, positional_embedding='learnable')),
    "cct_14": dict(batch=256, size=(224, 224), make=cct_14,
                   kw=dict(img_size=224, n_conv_layers=1, kernel_size=7, stride=2, padding=3, pooling_kernel_size=3,
                           pooling_stride=2, pooling_padding=1, num_classes=1000, positional_embedding='learnable')),
    "cifar": dict(batch=1024, size=(32, 32), make=cct_7,
                  kw=dict(img_size=32, kernel_size=3, n_conv_layers=1, num_classes=10)),
}


def families(fn) -> dict:
    """One profiled step split by kernel family: ms per step and share of the profiled step.  The tokenizer's GEMMs are
    the ones before embed_tokens."""
    with torch.inference_mode():
        _lib.profile_start()
        fn()
        rec = _lib.profile_stop()
    out = {k: 0.0 for k in ("tokenizer", "embed_tokens", "attention", "encoder_gemm_ln", "seq_pool", "classifier")}
    seen_embed = False
    for i, (name, _, ms) in enumerate(rec):
        if name in ("conv_im2col", "relu_maxpool") or (name == "gemm" and not seen_embed):
            out["tokenizer"] += ms
        elif name == "embed_tokens":
            seen_embed = True
            out["embed_tokens"] += ms
        elif name.startswith("attention"):
            out["attention"] += ms
        elif name == "seq_pool":
            out["seq_pool"] += ms
        elif name == "gemm" and i == len(rec) - 1:
            out["classifier"] += ms
        else:
            out["encoder_gemm_ln"] += ms
    total = sum(out.values())
    return {k: {"ms_per_step": round(v, 4), "share": round(v / total, 4) if total else None} for k, v in out.items()}


def run(name: str, spec: dict, args, dev, info: dict) -> dict:
    B, (H, W) = spec["batch"], spec["size"]
    torch.manual_seed(1)
    x = torch.randn(B, 3, H, W, device=dev).bfloat16()
    torch.manual_seed(0)
    model = spec["make"](**spec["kw"]).eval().to(dev, torch.bfloat16)
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
    res = {"workload": name, "model": "vit_pytorch_b200.cct", "batch": B, "input": [3, H, W],
           "tokens": model.classifier.sequence_length,
           "fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
           "eager_bf16_images_per_s": round(B / ms_eager * 1e3, 2), "eager_bf16_ms_per_step": round(ms_eager, 3),
           "speedup_vs_eager": round(ms_eager / ms, 3), "max_abs_logit_diff_fused_vs_eager": diff,
           "launches_per_step": launches, "families": families(call), "kernels": kernel_breakdown(call),
           "steps": args.steps, "gpu": info}
    del model
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=sorted(WORKLOADS), default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cct.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    info = card()
    for name, spec in WORKLOADS.items():
        if args.only in (None, name):
            print(json.dumps(run(name, spec, args, dev, info)), flush=True)


if __name__ == "__main__":
    main()
