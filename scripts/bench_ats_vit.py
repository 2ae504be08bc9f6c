"""Throughput of the fused Adaptive Token Sampling ViT (vit_pytorch_b200.ats_vit) on one GPU, against the same module's
PyTorch graph in bf16.

    python scripts/bench_ats_vit.py [--batches 64 256] [--steps 5] [--rounds 3]

The reference README's configuration: 256 x 256, patch 16 (257 tokens), dim 1024, depth 6, 16 heads, mlp 2048,
max_tokens_per_depth (256, 128, 64, 32, 16, 8).  Per batch size, every shape warmed up first, then `rounds` rounds that
each time the fused forward and the PyTorch graph (alternating), `steps` calls each; the medians are reported.  The
same weights with no layer sampling (every K at 256) are timed the same way, fused, to show what sampling saves.  Then
one profiled fused step: per layer its row slot, the mean kept tokens per image (with and without the cls row), the
select kernel's and the attention's time, and every GEMM's achieved TFLOP/s from FLOP counts computed from the shapes;
the head's launches apart.  The card's name and
power limit are read in the same run.  One JSON line per batch size; writes nothing.
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
from vit_pytorch_b200.ats_vit import ViT, slot_plan  # noqa: E402

README = dict(image_size=256, patch_size=16, num_classes=1000, dim=1024, depth=6,
              max_tokens_per_depth=(256, 128, 64, 32, 16, 8), heads=16, mlp_dim=2048, dropout=0.1, emb_dropout=0.1)


def layer_profile(model: ViT, x: torch.Tensor) -> list:
    """One profiled fused step: its launches attributed to the layers in order (each layer opens with its QKV GEMM; the
    patch embedding before the first is left out) and the head's two launches (LayerNorm of the cls rows, the
    classifier GEMM) apart, plus the mean kept rows per image after every layer that may sample, with and without the
    cls row.  Returns (layers, head)."""
    kept = []
    real = _lib.ats_select

    def select(*a, **k):
        real(*a, **k)
        kept.append(a[5].clone())                        # lens_out: a ping-pong buffer a later layer overwrites
    with torch.inference_mode():
        model(x)
        torch.cuda.synchronize()
        _lib.ats_select = select
        try:
            _lib.profile_start()
            model(x)
            rec = _lib.profile_stop()
        finally:
            _lib.ats_select = real
    kept = [float(v.float().mean()) for v in kept]
    plan = slot_plan((x.shape[2] // 16) * (x.shape[3] // 16) + 1, model.max_tokens_per_depth)
    D = model.cls_token.shape[-1]
    head = [{"kernel": name, "ms": round(ms, 4)} for name, meta, ms in rec[-2:]]
    layers, cur = [], None
    for name, meta, ms in rec[:-2]:
        if name == "gemm" and meta.get("N") == 3 * D and meta.get("K") == D:
            cur = {"launches": []}
            layers.append(cur)
        if cur is None:
            continue
        e = {"kernel": name, "ms": round(ms, 4)}
        if name == "gemm":
            e["M"], e["N"], e["K"] = meta["M"], meta["N"], meta["K"]
            e["TFLOP_per_s"] = round(meta["flops"] / (ms / 1e3) / 1e12, 1)
        elif "flops" in meta:
            e["TFLOP_per_s"] = round(meta["flops"] / (ms / 1e3) / 1e12, 1)
        cur["launches"].append(e)
    it = iter(kept)
    for i, (L, (S_in, S_out, may)) in enumerate(zip(layers, plan)):
        L.update({"layer": i, "slot_in": S_in, "slot_out": S_out, "may_sample": may,
                  "ms": round(sum(e["ms"] for e in L["launches"]), 4),
                  "select_ms": sum(e["ms"] for e in L["launches"] if e["kernel"] == "ats_select") or None,
                  "attention_ms": sum(e["ms"] for e in L["launches"] if e["kernel"].startswith("attention"))})
        if may:
            rows = next(it)
            L["mean_kept_rows_per_image_with_cls"] = round(rows, 2)
            L["mean_kept_tokens_per_image"] = round(rows - 1, 2)
    return layers, head


def run(B: int, args, dev, info: dict) -> dict:
    torch.manual_seed(0)
    model = ViT(**README).eval().to(dev, torch.bfloat16)
    flat = ViT(**dict(README, max_tokens_per_depth=(256,) * 6)).eval().to(dev, torch.bfloat16)
    flat.load_state_dict(model.state_dict())
    torch.manual_seed(1)
    x = torch.randn(B, 3, 256, 256, device=dev).bfloat16()
    with torch.inference_mode():
        assert model.fused_reason(x) is None, model.fused_reason(x)
    call = lambda: model(x)                       # noqa: E731
    call_flat = lambda: flat(x)                   # noqa: E731

    def eager():
        os.environ["B200VIT_DISABLE_FUSED"] = "1"
        try:
            return timed(call, args.steps, 1)
        finally:
            del os.environ["B200VIT_DISABLE_FUSED"]

    timed(call, 1, 2)                             # warm every shape of every path
    timed(call_flat, 1, 2)
    eager()
    fused_ms, eager_ms, flat_ms = [], [], []
    for _ in range(args.rounds):
        fused_ms.append(timed(call, args.steps, 1))
        eager_ms.append(eager())
        flat_ms.append(timed(call_flat, args.steps, 1))
    with torch.inference_mode():
        _lib.reset_launch_count()
        call()
        torch.cuda.synchronize()
        launches = _lib.launch_count()
    f, e, fl = (statistics.median(v) for v in (fused_ms, eager_ms, flat_ms))
    layers, head = layer_profile(model, x)
    res = {"workload": "ats_vit_readme", "model": "vit_pytorch_b200.ats_vit.ViT", "batch": B, "input": [3, 256, 256],
           "fused_images_per_s": round(B / f * 1e3, 2), "fused_ms_per_step": round(f, 3),
           "eager_bf16_images_per_s": round(B / e * 1e3, 2), "eager_bf16_ms_per_step": round(e, 3),
           "speedup_vs_eager": round(e / f, 3),
           "fused_no_sampling_ms_per_step": round(fl, 3), "sampling_saves_vs_no_sampling": round(fl / f, 3),
           "rounds_fused_ms": [round(v, 3) for v in fused_ms], "rounds_eager_ms": [round(v, 3) for v in eager_ms],
           "rounds_no_sampling_ms": [round(v, 3) for v in flat_ms], "launches_per_step": launches,
           "layers": layers, "head": head,
           "steps": args.steps, "rounds": args.rounds, "gpu": info}
    del model, flat
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ats_vit.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _lib.device_ok(dev.index):
        raise SystemExit("libb200vit.so cannot run on this device: " + _lib.lib().b200vit_last_error().decode())
    info = card()
    for B in args.batches:
        print(json.dumps(run(B, args, dev, info)), flush=True)


if __name__ == "__main__":
    main()
