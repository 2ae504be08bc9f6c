"""Where the time of the four ViT-B/16 layer GEMMs goes: main loop against the fixed cost of each output tile.

    python scripts/bench_gemm_epilogue.py [--launches 50] [--warmup 5] [--m 100864] [--block-n 0 [1 2]]
                                          [--rounds 1] [--residual-only]

Times QKV, out-proj, FC1 and FC2 through _lib.gemm at M = 512 * 197 rows, with the flags and outputs that
b200vit_encoder_blocks_ex passes (LN-fold row sums over stats_parts(768) parts for QKV and FC1, an in-place fp32
residual with a bf16 copy and row statistics for out-proj and FC2).  Each GEMM also runs at 2x and 4x its K; a linear
fit of time against K splits a launch into the main loop (slope * K) and a fixed cost (intercept: the epilogue and
the pipeline fill of every tile).  Per-tile figures are per 128 x 256 block of output spread over the SMs, so that
builds with different tile widths compare directly.  CUDA events around --launches launches after --warmup.
--block-n sets the tile width (test hook 12: 0 = the library's choice, 1 = 128, 2 = 256); with several widths, each
of --rounds rounds times every width in turn, and the figures are medians over the rounds.  --residual-only times
out-proj and FC2 alone.  B200VIT_LIB selects the library.  Prints one JSON object with the card's name, power limit
and maximum SM clock.  Needs a GPU; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from vit_pytorch_b200 import _lib  # noqa: E402

D, HIDDEN, QKV = 768, 3072, 3 * 768


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(), "num_sms": torch.cuda.get_device_properties(0).multi_processor_count}
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        _, pl, clk = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        out.update(power_limit_w=float(pl), max_sm_clock_mhz=float(clk))
    except Exception as e:  # noqa: BLE001  (reported, not fatal)
        out["power_limit_w"] = f"unavailable: {type(e).__name__}"
    return out


def timed(fn, launches: int, warmup: int) -> float:
    """ms per launch"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--m", type=int, default=512 * 197)
    ap.add_argument("--block-n", type=int, nargs="+", default=[0], choices=[0, 1, 2])
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--residual-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm_epilogue: needs a CUDA device")
    M, dev = args.m, "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    parts = _lib.stats_parts(D)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, device=dev, generator=g) * scale)

    # the largest K of each GEMM is 4x its own; A and W are allocated once at that width and read through k=
    a_d = rnd(M, 4 * HIDDEN).bfloat16()
    w = {n: rnd(n, 4 * HIDDEN, scale=0.02).bfloat16() for n in (D, QKV, HIDDEN)}
    bias = {n: rnd(n) for n in (D, QKV, HIDDEN)}
    col_s = {n: rnd(n) for n in (D, QKV, HIDDEN)}
    sums = torch.stack([torch.zeros(M, parts, device=dev), torch.full((M, parts), 128.0, device=dev)], -1)
    x = rnd(M, D)
    xb = torch.empty(M, D, device=dev, dtype=torch.bfloat16)
    out_qkv = torch.empty(M, QKV, device=dev, dtype=torch.bfloat16)
    out_h = torch.empty(M, HIDDEN, device=dev, dtype=torch.bfloat16)
    stats = torch.empty(M, parts, 2, device=dev)

    gemms = {
        "qkv": (QKV, D, lambda k: _lib.gemm(a_d, w[QKV], out_bf16=out_qkv, bias=bias[QKV], ln_sums=sums,
                                              col_s=col_s[QKV], k=k)),
        "out_proj": (D, D, lambda k: _lib.gemm(a_d, w[D], out_bf16=xb, out_f32=x, bias=bias[D], resid=x,
                                                 stats_out=stats, k=k)),
        "fc1": (HIDDEN, D, lambda k: _lib.gemm(a_d, w[HIDDEN], out_bf16=out_h, bias=bias[HIDDEN], gelu=True,
                                                ln_sums=sums, col_s=col_s[HIDDEN], k=k)),
        "fc2": (D, HIDDEN, lambda k: _lib.gemm(a_d, w[D], out_bf16=xb, out_f32=x, bias=bias[D], resid=x,
                                                 stats_out=stats, k=k)),
    }
    if args.residual_only:
        gemms = {name: gemms[name] for name in ("out_proj", "fc2")}
    info = card()
    blocks_per_sm = lambda n: M * n / (128 * 256) / info["num_sms"]  # noqa: E731
    L = _lib.lib()
    rounds = {bn: {name: [] for name in gemms} for bn in args.block_n}  # [ms at k, 2k, 4k] per round
    try:
        for _ in range(args.rounds):
            for bn in args.block_n:
                L.b200vit_debug_set(12, bn)
                for name, (n, k, fn) in gemms.items():
                    ks = [k, 2 * k, 4 * k]
                    rounds[bn][name].append([timed(lambda kk=kk: fn(kk), args.launches, args.warmup) for kk in ks])
                    assert math.isfinite(float(x.sum())), "residual stream overflowed"
    finally:
        L.b200vit_debug_set(12, 0)
    res = {}
    for bn in args.block_n:
        res[bn] = {}
        for name, (n, k, _) in gemms.items():
            ms = np.median(np.array(rounds[bn][name]), axis=0)
            ks = np.array([k, 2 * k, 4 * k], dtype=float)
            fits = [np.polyfit(ks, np.array(r), 1) for r in rounds[bn][name]]
            slope, icpt = np.median([f[0] for f in fits]), np.median([f[1] for f in fits])
            per = blocks_per_sm(n)
            res[bn][name] = {
                "M": M, "N": n, "K": k, "ms_per_launch": ms[0], "tflops": 2.0 * M * n * k / ms[0] / 1e9,
                "ms_at_2k_4k": list(ms[1:]), "main_loop_ms": slope * k, "fixed_ms": icpt,
                "main_loop_us_per_block": 1e3 * slope * k / per, "fixed_us_per_block": 1e3 * icpt / per,
                "ms_per_launch_rounds": [r[0] for r in rounds[bn][name]],
                "main_loop_ms_rounds": [f[0] * k for f in fits], "fixed_ms_rounds": [f[1] for f in fits],
            }
    print(json.dumps({"lib": str(_lib.LIB_PATH), "card": info, "launches": args.launches, "rounds": args.rounds,
                      "gemms_by_block_n": res}), flush=True)


if __name__ == "__main__":
    main()
