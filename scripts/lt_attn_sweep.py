#!/usr/bin/env python
"""Sweep the KV-split count of the tensor-core long-term attention (default "tile" layout) at the benchmark's shapes -- the
data behind engine.lt_splits.

Workload: N = 1674 queries (the 481x849 input's stride-16 grid), H = 8 heads x 32, Tk = 1674 m keys for m in {1 (the
self-attention), 2, 5, 10, 15, 20} memory frames; seeded random Q, K, V packed as the engine packs them.  Each point is the
launch plus, for splits > 1, aotb_attn_merge_f32, REP times in a CUDA graph, timed with CUDA events over 5 replays after a
warm replay; the whole split sweep is repeated --reps times and each point reports its minimum and its spread.  Exact and
fast mode, splits 1 .. 16.  The rate is algorithmic: 4 N Tk C FLOP (as bench.py's roofline) over the time.  Also recorded:
the card's name and power limit, the kernel's resident CTAs per SM, registers and local bytes, and the policy's split count.

    python scripts/lt_attn_sweep.py OUT.json [--reps 3]
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
from aot_benchmark_b200.engine import lt_splits  # noqa: E402
from bounded_bank_fps import gpu_info  # noqa: E402

N, H, D = 1674, 8, 32
MEMS = (1, 2, 5, 10, 15, 20)
SPLITS = range(1, 17)
REP = 20


def time_graph(fn):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fn()
        st.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=st):
            for _ in range(REP):
                fn()
        gr.replay()
        st.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(5):
            gr.replay()
        e1.record(st)
        st.synchronize()
    return e0.elapsed_time(e1) * 1000 / (5 * REP)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lt_attn_sweep.py needs a CUDA device (no CPU path)")
    d = torch.device("cuda", 0)
    torch.cuda.set_device(d)
    gpu, power = gpu_info()
    print(f"GPU: {gpu}, power limit {power}", flush=True)
    rec = {"gpu": gpu, "power_limit": power, "N": N, "H": H, "rep_per_graph": REP, "reps": a.reps, "occupancy": {},
           "rows": []}
    for exact in (True, False):
        ctas, regs, local = ops.lt_attn_tc_occupancy(exact)
        rec["occupancy"]["exact" if exact else "fast"] = {"ctas_per_sm": ctas, "regs": regs, "local_bytes": local}
    print(json.dumps(rec["occupancy"]), flush=True)
    g = torch.Generator().manual_seed(0)
    nq_cap = (N + 255) // 256 * 256
    Qp = torch.zeros(H, nq_cap, 64, dtype=torch.float16, device=d)
    ops.tc_pack_rows(torch.randn(N, H * D, generator=g).to(d), Qp, div=D ** 0.5)
    O = torch.empty(N, H * D, device=d)
    for m in MEMS:
        tk = N * m
        Kp = torch.zeros(H, tk, 64, dtype=torch.float16, device=d)
        Vp = torch.zeros_like(Kp)
        ops.tc_pack_rows(torch.randn(tk, H * D, generator=g).to(d), Kp)
        ops.tc_pack_rows(torch.randn(tk, H * D, generator=g).to(d), Vp)
        gflop = 4.0 * N * tk * H * D / 1e9
        for exact in (True, False):
            parts = {s: (torch.empty(s, N, H * D, device=d), torch.empty(s, H, N, device=d), torch.empty(s, H, N, device=d))
                     for s in SPLITS if s > 1}
            times = {s: [] for s in SPLITS}
            for _ in range(a.reps):
                for s in SPLITS:
                    times[s].append(time_graph(lambda: ops.lt_attention_tc(Qp, Kp, Vp, N, tk, O=O, splits=s, exact=exact,
                                                                           part=parts.get(s), variant="tile")))
            us = {s: min(t) for s, t in times.items()}
            best = min(us, key=us.get)
            pol = lt_splits(N, H, tk, variant="tile")
            row = {"m": m, "Tk": tk, "mode": "exact" if exact else "fast", "gflop": round(gflop, 3),
                   "us": {s: round(t, 2) for s, t in us.items()},
                   "spread_us": {s: round(max(t) - min(t), 2) for s, t in times.items()},
                   "tflops": {s: round(gflop / t * 1e3, 1) for s, t in us.items()},
                   "best": best, "policy": pol, "policy_over_best": round(us[pol] / us[best] - 1, 4)}
            rec["rows"].append(row)
            print(f"m={m:2d} Tk={tk:5d} {row['mode']:5s}  best s={best:2d} {us[best]:8.1f} us "
                  f"{row['tflops'][best]:6.1f} TFLOP/s   policy s={pol:2d} {us[pol]:8.1f} us {row['tflops'][pol]:6.1f} TFLOP/s "
                  f"(+{100 * row['policy_over_best']:.1f} %, spread {row['spread_us'][pol]:.1f} us)", flush=True)
        del Kp, Vp
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
