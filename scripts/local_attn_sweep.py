#!/usr/bin/env python
"""Per-launch time of the short-term local attention entry points at the AOT head shape (8 heads x 32 channels, 15 x 15
window, relative embeddings on keys and values) -- the kernel the LSTT runs once per layer and frame.

Shapes: the 31 x 54 map of the benchmark's 481x849 input (R50 / MobileNetV3 / ResNeSt encoders) and the 37 x 65 map of
SwinB-AOTL.  Seeded random q, k, v are column slices of one wider buffer and the output a column slice of another, as the
engine packs them.  Each entry point runs REP times in a CUDA graph, timed with CUDA events over 5 replays after a warm
replay; the whole sweep is repeated --reps times and each point reports its minimum and its spread.  Entry points the
loaded library does not export are reported as missing.  Also recorded: the card's name and power limit.

    python scripts/local_attn_sweep.py OUT.json [--reps 3]
"""
import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))

from aot_benchmark_b200 import ops  # noqa: E402
from bounded_bank_fps import gpu_info  # noqa: E402
from lt_attn_sweep import time_graph  # noqa: E402

H, D = 8, 32
SHAPES = ((31, 54), (37, 65))


def entry_points(q, k, v, rkw, rkb, rv, rv_t, out, h, w):
    eps = {"warp": lambda: ops.local_attention(q, k, v, rkw, rkb, rv, out, h, w, H, D, D),
           "tile": lambda: ops.local_attention_tile(q, k, v, rkw, rkb, rv_t, out, h, w, H)}
    if hasattr(ops, "local_attention_tc"):
        eps["tc"] = lambda: ops.local_attention_tc(q, k, v, rkw, rkb, rv_t, out, h, w, H)
    return eps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("local_attn_sweep.py needs a CUDA device (no CPU path)")
    d = torch.device("cuda", 0)
    torch.cuda.set_device(d)
    gpu, power = gpu_info()
    print(f"GPU: {gpu}, power limit {power}", flush=True)
    rec = {"gpu": gpu, "power_limit": power, "H": H, "d": D, "reps": a.reps, "rows": []}
    g = torch.Generator().manual_seed(0)
    C = H * D
    for h, w in SHAPES:
        N = h * w
        qkv = torch.randn(N, 3 * C + 8, generator=g).to(d)
        q, k, v = qkv[:, 8:8 + C], qkv[:, 8 + C:8 + 2 * C], qkv[:, 8 + 2 * C:]
        rkw = (0.2 * torch.randn(H * 225, D, generator=g)).to(d)
        rkb = (0.2 * torch.randn(H * 225, generator=g)).to(d)
        rv = (0.2 * torch.randn(H, D, 225, generator=g)).to(d)
        rv_t = rv.permute(0, 2, 1).contiguous()
        out = torch.empty(N, 2 * C, device=d)[:, C:]
        eps = entry_points(q, k, v, rkw, rkb, rv, rv_t, out, h, w)
        times = {n: [] for n in eps}
        for _ in range(a.reps):
            for n, fn in eps.items():
                times[n].append(time_graph(fn))
        for n in ("warp", "tile", "tc"):
            if n not in eps:
                print(f"{h}x{w} {n:4s}  missing from this build", flush=True)
                continue
            row = {"h": h, "w": w, "impl": n, "us": round(min(times[n]), 2),
                   "spread_us": round(max(times[n]) - min(times[n]), 2)}
            rec["rows"].append(row)
            print(f"{h}x{w} {n:4s}  {row['us']:8.2f} us per launch (spread {row['spread_us']:.2f} us)", flush=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
