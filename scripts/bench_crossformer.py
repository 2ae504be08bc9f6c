"""Throughput of the fused CrossFormer (vit_pytorch_b200.crossformer) on one GPU.

    python scripts/bench_crossformer.py [--steps 10] [--warmup 3] [--batch 64]

Prints one JSON line: the README CrossFormer (dim 64 / 128 / 256 / 512, depth 2 / 2 / 8 / 2, global windows 8 / 4 /
2 / 1, local window 7, stem kernels 4 / 8 / 16 / 32 at stride 4) at 224 x 224 in bf16 -- maps 56 x 56, 28 x 28,
14 x 14 and 7 x 7.  Fused images/s with eager launches and with the whole forward replayed through GraphedForward, the
module's own fp32 eager graph on the same GPU (its bf16 graph raises, as the reference's does), the largest logit
differences, ms per step, launches, the share of every library kernel and of every window attention launch by stage map,
window and partition (per-call CUDA events in a separate profiled step), and the stage-1 cross-scale embedding kernel
against the four cuDNN bf16 convolutions + torch.cat on the same input, with the card's name and power limit read in
the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_vit_small_dataset import card, kernel_breakdown, timed  # noqa: E402
from vit_pytorch_b200 import _lib  # noqa: E402
from vit_pytorch_b200.crossformer import CrossFormer, embed_weights  # noqa: E402
from vit_pytorch_b200.graph import GraphedForward  # noqa: E402

IMAGE = 224
README = dict(num_classes=1000, dim=(64, 128, 256, 512), depth=(2, 2, 8, 2), global_window_size=(8, 4, 2, 1),
              local_window_size=7)


def window_breakdown(fn) -> list:
    """One profiled step: per (map, window, partition) of attention_window_relpos, ms per step and launches."""
    with torch.inference_mode():
        _lib.profile_start()
        fn()
        rec = _lib.profile_stop()
    agg: dict = {}
    for name, meta, ms in rec:
        if name != "attention_window_relpos":
            continue
        key = (meta["h"], meta["w"], meta["window"], "grid" if meta["grid"] else "block", meta["H"])
        a = agg.setdefault(key, [0.0, 0])
        a[0] += ms
        a[1] += 1
    return [{"map": f"{k[0]}x{k[1]}", "window": k[2], "partition": k[3], "heads": k[4],
             "windows_per_launch": meta_windows(k), "ms": round(v[0], 4), "launches": v[1],
             "us_per_launch": round(v[0] / v[1] * 1e3, 2)} for k, v in sorted(agg.items(), reverse=True)]


def meta_windows(k) -> int:
    return (k[0] // k[2]) * (k[1] // k[2])


def embed_vs_cudnn(model, x, steps: int, warmup: int) -> dict:
    """The stage-1 cross-scale embedding kernel against the cuDNN bf16 convolutions + torch.cat (NCHW out), both timed
    with CUDA events on the same input."""
    cel = model.layers[0][0]
    m = embed_weights(cel, True)
    ks = [c.kernel_size[0] for c in cel.convs]
    widths = [c.out_channels for c in cel.convs]
    s = cel.convs[0].stride[0]
    B = x.shape[0]
    h = w = _lib.conv_out_size(IMAGE, ks[0], s, (ks[0] - s) // 2)
    out = torch.empty(B * h * w, sum(widths), device=x.device)
    ms_kernel = timed(lambda: _lib.cross_embed_nchw(x, m["w"], m["b"], out, ks, widths, s), steps, warmup)
    ms_cudnn = timed(lambda: torch.cat([F.conv2d(x, c.weight, c.bias, stride=s, padding=(c.kernel_size[0] - s) // 2)
                                        for c in cel.convs], dim=1), steps, warmup)
    with torch.inference_mode():
        want = torch.cat([F.conv2d(x, c.weight, c.bias, stride=s, padding=(c.kernel_size[0] - s) // 2)
                          for c in cel.convs], dim=1).float().permute(0, 2, 3, 1).reshape(-1, sum(widths))
        _lib.cross_embed_nchw(x, m["w"], m["b"], out, ks, widths, s)
    flops = 2.0 * B * h * w * sum(n * x.shape[1] * k * k for k, n in zip(ks, widths))
    return {"cross_embed_nchw_ms": round(ms_kernel, 4), "cudnn_conv2d_x4_cat_ms": round(ms_cudnn, 4),
            "speedup_vs_cudnn": round(ms_cudnn / ms_kernel, 3),
            "cross_embed_nchw_tflops": round(flops / ms_kernel / 1e9, 2),
            "max_abs_diff_vs_cudnn": (out - want).abs().max().item()}


def run(args, dev, info: dict) -> dict:
    B = args.batch
    torch.manual_seed(1)
    x = torch.randn(B, 3, IMAGE, IMAGE, device=dev).bfloat16()
    torch.manual_seed(0)
    model = CrossFormer(**README).eval().to(dev, torch.bfloat16)
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
    # the module's own PyTorch graph in fp32 (a bf16 copy raises in the dynamic position bias, as the reference)
    m32, x32 = model.float(), x.float()
    ms_eager = timed(lambda: m32(x32), max(3, args.steps // 2), 2)
    with torch.inference_mode():
        diff = (m32(x32) - out).abs().max().item()
    model.to(torch.bfloat16)
    embed = embed_vs_cudnn(model, x, args.steps * 5, args.warmup)
    return {"workload": "crossformer_readme", "model": "vit_pytorch_b200.crossformer.CrossFormer", "batch": B,
            "input": [3, IMAGE, IMAGE], "maps": [56, 28, 14, 7], "config": {k: v for k, v in README.items()},
            "fused_images_per_s": round(B / ms * 1e3, 2), "fused_ms_per_step": round(ms, 3),
            "fused_graph_images_per_s": round(B / ms_graph * 1e3, 2), "fused_graph_ms_per_step": round(ms_graph, 3),
            "eager_fp32_images_per_s": round(B / ms_eager * 1e3, 2), "eager_fp32_ms_per_step": round(ms_eager, 3),
            "speedup_vs_eager_fp32": round(ms_eager / ms, 3),
            "graph_speedup_vs_eager_fp32": round(ms_eager / ms_graph, 3),
            "max_abs_logit_diff_fused_vs_eager_fp32": diff, "max_abs_logit_diff_graph_vs_launches": graph_diff,
            "launches_per_step": launches, "kernels": kernel_breakdown(call), "window_attention": window_breakdown(call),
            "stem": embed, "steps": args.steps, "gpu": info}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_crossformer.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    print(json.dumps(run(args, dev, card())), flush=True)


if __name__ == "__main__":
    main()
