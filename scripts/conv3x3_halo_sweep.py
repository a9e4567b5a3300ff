#!/usr/bin/env python
"""The stride-1 3x3 convolutions of one R50-AOTL 481 x 849 frame on the halo kernel against the chunked kernel
(aotb_set_conv_halo 0 = chunked only, 1 = tile model, 2 = halo kernel wherever eligible), both precisions, graph-replayed (scripts/conv_sweep.py's timing).
The two paths alternate within each of PASSES passes and the minimum per path is reported, with the achieved tensor-pipe
rate (executed fp16 FLOPs: 3 products per k-step when split) and the HBM bytes the shape needs at least (input, weights,
output once).  GPU only.

    python scripts/conv3x3_halo_sweep.py OUT.json [--passes 3]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from aot_benchmark_b200 import ops  # noqa: E402
from aot_benchmark_b200._lib import lib  # noqa: E402
from conv_sweep import time_graph  # noqa: E402

# name, H, W, Cin, Cout, launches per frame: layers 1-3 (layer 3's shape is also the FPN decoder's conv_16x) and the
# decoder's conv_8x and conv_4x
SHAPES = [("l1 3x3 64->64", 121, 213, 64, 64, 3), ("l2 3x3 128->128", 61, 107, 128, 128, 3),
          ("l3 / conv_16x 3x3 256->256", 31, 54, 256, 256, 6), ("dec conv_8x 3x3 256->128", 61, 107, 256, 128, 1),
          ("dec conv_4x 3x3 128->128", 121, 213, 128, 128, 1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--passes", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv3x3_halo_sweep.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    d = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    rows = []
    for name, H, W, Cin, Cout, per_frame in SHAPES:
        x = torch.randn(1, H, W, Cin, generator=g).to(d)
        w = (torch.randn(9 * Cin, Cout, generator=g) / (9 * Cin) ** 0.5).to(d)
        wh, wl, ws = ops.split_fp16_scaled(w)
        b = torch.randn(Cout, generator=g).to(d)
        out = torch.empty(1, H, W, Cout, device=d)
        flop = 2.0 * H * W * Cout * 9 * Cin
        hbm = 4.0 * H * W * (Cin + Cout) + 2.0 * 9 * Cin * Cout * 2
        for mode in ("fp32", "fp16"):
            wl_m = wl if mode == "fp32" else None
            fn = lambda: ops.conv2d_tc(x, wh, wl_m, b, out, KH=3, KW=3, pad=1, act=1, wscale=ws, const_w=True)  # noqa: E731
            t = {"chunked": [], "halo": [], "halo_forced": []}
            for _ in range(args.passes):
                for path, m in (("chunked", 0), ("halo", 1), ("halo_forced", 2)):
                    lib().aotb_set_conv_halo(m)
                    t[path].append(time_graph(fn))
            lib().aotb_set_conv_halo(1)
            best = {k: min(v) for k, v in t.items()}
            ex = flop * (3 if mode == "fp32" else 1)
            row = {"shape": name, "mode": mode, "per_frame": per_frame, "us": {k: round(v, 2) for k, v in best.items()},
                   "all_us": {k: [round(u, 2) for u in v] for k, v in t.items()},
                   "tensor_tflops": {k: round(ex / v / 1e6, 1) for k, v in best.items()},
                   "hbm_tb_s": {k: round(hbm / v / 1e6, 3) for k, v in best.items()},
                   "speedup": round(best["chunked"] / best["halo"], 2)}
            rows.append(row)
            print(json.dumps(row), flush=True)
    for mode in ("fp32", "fp16"):
        tot = {p: round(sum(r["us"][p] * r["per_frame"] for r in rows if r["mode"] == mode), 1) for p in ("chunked", "halo")}
        print(f"{mode}: stride-1 3x3 convs per frame: chunked {tot['chunked']} us, halo path {tot['halo']} us", flush=True)
    json.dump({"gpu": gpu, "rows": rows}, open(args.out, "w"), indent=1)
    print("gpu:", gpu)


if __name__ == "__main__":
    main()
