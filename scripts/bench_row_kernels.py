"""Kernel time of the row kernels whose arithmetic order the row-bounds tests pin, for one or more builds of the library.

    python scripts/bench_row_kernels.py [--lib PATH ...] [--iters 200] [--rounds 15]

Workloads (one JSON line each, per library):
  layernorm_heads_navit  the q / k head LayerNorm of the nested-tensor NaViT at BASELINE's NaViT width: 65536 tokens
                         (256 images of 256 patches), 32 heads (q and k of 16) x 64 on the packed qkv rows (ld 3072)
  embed_tokens_vit_b16   ViT-B/16 token assembly, batch 64: LayerNorm(768) of 196 patch rows + position, a class row,
                         the bf16 copy and the LN-fold statistics
  embed_tokens_pit       PiT's first stage, batch 64: 961 unfolded patch rows of dim 256 without a LayerNorm + position,
                         a class row, the bf16 copy and the statistics
Every --lib (default: the in-tree library) is loaded side by side; the rounds alternate between them, each timing
--iters back-to-back launches with CUDA events after a warm-up, and the median round is reported with the bytes the
kernel must move over that time.  The outputs of every library are compared with the first one's.  The card's name
and power limit are read in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "vit_pytorch_b200", "lib", "libb200vit.so")


def card() -> dict:
    info = dict(gpu=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [v.strip() for v in q.split(",")]
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        info["power_limit"] = "unknown"
    return info


def load(path: str) -> C.CDLL:
    L = C.CDLL(os.path.abspath(path))
    vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float
    L.b200vit_layernorm_heads.restype = i32
    L.b200vit_layernorm_heads.argtypes = [vp, i64, vp, i32, i32, i32, f32, vp]
    L.b200vit_embed_tokens.restype = i32
    L.b200vit_embed_tokens.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, vp]
    L.b200vit_last_error.restype = C.c_char_p
    return L


def p(t):
    return None if t is None else t.data_ptr()


def workloads(dev):
    g = torch.Generator(device=dev).manual_seed(0)
    rn = lambda *s: torch.randn(*s, generator=g, device=dev)
    out = {}
    T, H2, dh = 65536, 32, 64
    qkv = rn(T, 3 * 16 * dh).bfloat16()
    gam = rn(H2 * dh)
    work = torch.empty_like(qkv)

    def heads(L, s):
        return L.b200vit_layernorm_heads(p(work), work.stride(0), p(gam), T, H2, dh, 1e-5, s)
    out["layernorm_heads_navit"] = dict(call=heads, prep=lambda: work.copy_(qkv), out=lambda: work,
                                        bytes=T * H2 * dh * 2 * 2)
    for name, (B, n, D, ln) in {"embed_tokens_vit_b16": (64, 196, 768, True),
                                "embed_tokens_pit": (64, 961, 256, False)}.items():
        y, gm, be, cls, pos = rn(B * n, D), rn(D), rn(D), rn(1, D), rn(n + 1, D)
        R = B * (n + 1)
        x, xb, st = torch.empty(R, D, device=dev), torch.empty(R, D, device=dev, dtype=torch.bfloat16), \
            torch.empty(R, 2, device=dev)

        def emb(L, s, y=y, gm=gm, be=be, cls=cls, pos=pos, x=x, xb=xb, st=st, B=B, n=n, D=D, ln=ln):
            return L.b200vit_embed_tokens(p(y), p(gm) if ln else None, p(be) if ln else None, p(cls), p(pos), None,
                                          p(x), p(xb), p(st), B, n, 1, 0, D, 1e-5, s)
        out[name] = dict(call=emb, prep=lambda: None, out=lambda x=x, st=st: torch.cat([x.flatten(), st.flatten()]),
                         bytes=(B * n * D + (n + 1) * D) * 4 + R * D * (4 + 2) + R * 8)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", help="library to time (repeatable; default: the in-tree build)")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_row_kernels needs a GPU")
    paths = args.lib or [DEFAULT_LIB]
    libs = [load(x) for x in paths]
    dev = "cuda"
    s = torch.cuda.current_stream().cuda_stream
    info = card()
    for name, w in workloads(dev).items():
        outs = []
        for L in libs:                                   # one checked call per library, outputs kept for comparison
            w["prep"]()
            rc = w["call"](L, s)
            assert rc == 0, L.b200vit_last_error()
            outs.append(w["out"]().clone())
            for _ in range(args.warmup):
                w["prep"]()
                w["call"](L, s)
        times = [[] for _ in libs]
        for _ in range(args.rounds):
            for i, L in enumerate(libs):
                w["prep"]()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    w["call"](L, s)        # heads: in place, so later launches normalise normalised heads (same bytes)
                e1.record()
                torch.cuda.synchronize()
                times[i].append(e0.elapsed_time(e1) * 1e3 / args.iters)
        for i, path in enumerate(paths):
            us = statistics.median(times[i])
            diff = (outs[i].float() - outs[0].float()).abs().nan_to_num(0).max().item()
            print(json.dumps(dict(workload=name, lib=path, us_per_call=round(us, 2),
                                  us_spread=[round(min(times[i]), 2), round(max(times[i]), 2)],
                                  gb_per_s=round(w["bytes"] / us / 1e3, 1), max_abs_diff_vs_first=diff, **info)))


if __name__ == "__main__":
    main()
