"""Throughput of the fused T2T-ViT (vit_pytorch_b200.t2t) on one GPU, against the same module's PyTorch graph in bf16.

    python scripts/bench_t2t.py [--batches 64 256] [--steps 5] [--rounds 3]

The reference README's configuration: 224 x 224, t2t_layers ((7, 4), (3, 2), (3, 2)) (soft splits 147 wide over 3136
tokens and 1323 wide over 784, then Linear(11907, 512)), dim 512, depth 5, 8 heads, mlp 512.  Per batch size, every
shape warmed up first, then `rounds` rounds that each time the fused forward and the PyTorch graph (alternating),
`steps` calls each; the medians are reported.  Then one profiled fused step per soft split: every launch of its layer
with its time, and the achieved TFLOP/s of its attention and GEMMs from FLOP counts computed here from the shapes; the
final Linear; and the time and bandwidth of every soft-split unfold.  The card's name and power limit are read in the
same run.  One JSON line per batch size; writes nothing.
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

from bench_vit_small_dataset import card, timed  # noqa: E402
from vit_pytorch_b200 import _lib  # noqa: E402
from vit_pytorch_b200.t2t import T2TViT, round8, soft_split_layer  # noqa: E402

README = dict(image_size=224, num_classes=1000, dim=512, depth=5, heads=8, mlp_dim=512)


def layer_flops(B: int, n: int, w: int, dp: int) -> dict:
    """FLOPs of one soft-split layer's launches, from the shapes (the GEMMs at their true K = w)."""
    M = B * n
    return {"qkv": 2.0 * M * 3 * dp * w, "attention": 4.0 * B * n * n * dp, "out": 2.0 * M * round8(w) * w,
            "fc1": 2.0 * M * round8(w) * w, "fc2": 2.0 * M * round8(w) * w}


def stage_profile(model: T2TViT, B: int, dev) -> list:
    """Per soft split: every launch of its layer on a random stream of its shape, timed with CUDA events."""
    geo = model.stage_geometry(224, 224)
    out, width = [], 3
    for i, ((k, _), t, (_, _, oh, ow)) in enumerate(zip(model.t2t_layers, model.soft_splits(), geo)):
        w, n = width * k * k, oh * ow
        width = w
        if t is None:
            continue
        wts = model._split_weights(i, t)
        x = torch.zeros(B * n, round8(w), device=dev)
        x[:, :w] = torch.randn(B * n, w, device=dev)
        vl = model._varlen(B, n, dev)
        with torch.inference_mode():
            soft_split_layer(wts, x.clone(), B, n, vl)          # warm-up
            torch.cuda.synchronize()
            _lib.profile_start()
            soft_split_layer(wts, x, B, n, vl)
            rec = _lib.profile_stop()
        fl = layer_flops(B, n, w, wts["dp"])
        launches, gemms = [], ["qkv", "out", "fc1", "fc2"] if wts["dp"] <= 160 else ["qkv", "fc1", "fc2"]
        for name, meta, ms in rec:
            e = {"kernel": name, "ms": round(ms, 4)}
            if name.startswith("attention"):
                e["TFLOP_per_s"] = round(fl["attention"] / (ms / 1e3) / 1e12, 1)
            elif name == "gemm":
                g = gemms.pop(0)
                e["gemm"] = g
                e["TFLOP_per_s"] = round(fl[g] / (ms / 1e3) / 1e12, 1)
            launches.append(e)
        out.append({"stage": i, "tokens": n, "width": w, "dp": wts["dp"], "ms": round(sum(r[2] for r in rec), 3),
                    "launches": launches})
    return out


def run(B: int, args, dev, info: dict) -> dict:
    torch.manual_seed(0)
    model = T2TViT(**README).eval().to(dev, torch.bfloat16)
    torch.manual_seed(1)
    x = torch.randn(B, 3, 224, 224, device=dev).bfloat16()
    with torch.inference_mode():
        assert model.fused_reason(x) is None, model.fused_reason(x)
    call = lambda: model(x)                       # noqa: E731

    def eager():
        os.environ["B200VIT_DISABLE_FUSED"] = "1"
        try:
            return timed(call, args.steps, 1)
        finally:
            del os.environ["B200VIT_DISABLE_FUSED"]

    timed(call, 1, 2)                             # warm every shape of both paths
    eager()
    fused_ms, eager_ms = [], []
    for _ in range(args.rounds):
        fused_ms.append(timed(call, args.steps, 1))
        eager_ms.append(eager())
    with torch.inference_mode():
        out = call().float()
        os.environ["B200VIT_DISABLE_FUSED"] = "1"
        try:
            diff = (call().float() - out).abs().max().item()
        finally:
            del os.environ["B200VIT_DISABLE_FUSED"]
        _lib.reset_launch_count()
        call()
        torch.cuda.synchronize()
        launches = _lib.launch_count()
    f, e = statistics.median(fused_ms), statistics.median(eager_ms)
    with torch.inference_mode():                  # the soft-split unfolds of one profiled fused step
        call()
        torch.cuda.synchronize()
        _lib.profile_start()
        call()
        unfolds = [{"ms": round(ms, 4), "GB_per_s": round(meta["bytes"] / (ms / 1e3) / 1e9, 1)}
                   for name, meta, ms in _lib.profile_stop() if name == "t2t_unfold"]
    # the final Linear(11907, 512) over B * 196 rows
    lin = model.to_patch_embedding[-1]
    a = torch.randn(B * 196, round8(lin.in_features), device=dev).bfloat16()
    y = torch.empty(B * 196, lin.out_features, device=dev)
    wts = model._embed_weights()
    lin_ms = timed(lambda: _lib.gemm(a, wts["w"], out_f32=y, bias=wts["b"], k=lin.in_features), args.steps, 2)
    lin_flops = 2.0 * B * 196 * lin.out_features * lin.in_features
    res = {"workload": "t2t_readme", "model": "vit_pytorch_b200.t2t.T2TViT", "batch": B, "input": [3, 224, 224],
           "fused_images_per_s": round(B / f * 1e3, 2), "fused_ms_per_step": round(f, 3),
           "eager_bf16_images_per_s": round(B / e * 1e3, 2), "eager_bf16_ms_per_step": round(e, 3),
           "speedup_vs_eager": round(e / f, 3), "rounds_fused_ms": [round(v, 3) for v in fused_ms],
           "rounds_eager_ms": [round(v, 3) for v in eager_ms], "max_abs_logit_diff_fused_vs_eager": diff,
           "launches_per_step": launches, "unfolds": unfolds, "soft_splits": stage_profile(model, B, dev),
           "final_linear": {"ms": round(lin_ms, 4), "TFLOP_per_s": round(lin_flops / (lin_ms / 1e3) / 1e12, 1)},
           "steps": args.steps, "rounds": args.rounds, "gpu": info}
    del model
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_t2t.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    info = card()
    for B in args.batches:
        print(json.dumps(run(B, args, dev, info)), flush=True)


if __name__ == "__main__":
    main()
