"""Fixed-length attention alone, the persistent kernel against the tiled one, at the ViT-B/16 batch.

    python scripts/bench_attention.py [--launches 50] [--warmup 5] [--rounds 3] [--batch 512]

Times _lib.attention at B = 512, H = 12, dh = 64 for N = 129, 197 and 256, which b200vit_attention_ex sends to the
persistent kernel of csrc/attention_short.cu, and for N = 128 and 257 on either side, which stay on the tiled kernel of
csrc/attention.cu.  Every N runs both ways in the same process -- as dispatched, and with test hook 15 set, which keeps
every launch on the tiled kernel -- alternated over --rounds rounds; the figure reported is the median round.  CUDA
events around --launches launches after --warmup.  A launch has to read the packed qkv buffer and write the merged
heads, B N (2304 + 768) 2 bytes (620 MB at N = 197); GB/s is that over the time, and hbm_share the time the data-sheet
3.35 TB/s of an H100 SXM would need over the time taken.  The outputs of the two ways are compared bit for bit.
B200VIT_LIB selects the library.  Prints one JSON object with the card's name, power limit and maximum SM clock.
Needs a GPU; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from vit_pytorch_b200 import _lib  # noqa: E402

H, DH = 12, 64
LENGTHS = [128, 129, 197, 256, 257]
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=512)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention: needs a CUDA device")
    B, dev = args.batch, "cuda"
    L = _lib.lib()
    g = torch.Generator(device=dev).manual_seed(0)
    res = {}
    for N in LENGTHS:
        qkv = torch.randn(B * N, 3 * H * DH, device=dev, generator=g).bfloat16()
        outs = {w: torch.empty(B * N, H * DH, device=dev, dtype=torch.bfloat16) for w in ("dispatched", "tiled")}
        ms = {w: [] for w in outs}
        for _ in range(args.rounds):
            for way, out in outs.items():
                assert L.b200vit_debug_set(15, int(way == "tiled")) == 0
                try:
                    ms[way].append(timed(lambda: _lib.attention(qkv, out, B, N, H, DH, DH ** -0.5),
                                         args.launches, args.warmup))
                finally:
                    L.b200vit_debug_set(15, 0)
        nbytes = B * N * 4 * H * DH * 2
        res[str(N)] = {"persistent_kernel": 128 < N <= 256, "bytes": nbytes,
                       "same_bits": torch.equal(outs["dispatched"], outs["tiled"])}
        for way, v in ms.items():
            med = statistics.median(v)
            res[str(N)][way] = {"ms_per_launch": med, "rounds_ms": v, "gbps": nbytes / med / 1e6,
                                "hbm_share": nbytes / HBM_BYTES_PER_S * 1e3 / med}
        res[str(N)]["speedup"] = res[str(N)]["tiled"]["ms_per_launch"] / res[str(N)]["dispatched"]["ms_per_launch"]
    print(json.dumps({"lib": str(_lib.LIB_PATH), "card": card(), "B": B, "H": H, "dh": DH, "launches": args.launches,
                      "rounds": args.rounds, "lengths": res}), flush=True)


if __name__ == "__main__":
    main()
