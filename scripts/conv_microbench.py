#!/usr/bin/env python
"""Per-layer timing of the tensor-core conv / linear kernel on the shapes one R50-AOTL 480p frame launches.

For every shape and every tuning mask (aotb_set_conv_tiling): a CUDA graph of REP back-to-back launches is replayed and
timed with CUDA events (L2-warm, launch overhead amortised the way the engine's frame graphs do), and one eager launch
in diagnostic mode prints the median per-CTA phase stamps.  GPU only; writes the rows as JSON to the path given
as the first argument (default conv_microbench.json).
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aot_benchmark_b200 import ops  # noqa: E402
from aot_benchmark_b200._lib import lib  # noqa: E402

SHAPES = [  # name, H, W, Cin, Cout, K, stride, pad
    ("l1 1x1 64->64", 121, 213, 64, 64, 1, 1, 0),
    ("l1 3x3 64->64", 121, 213, 64, 64, 3, 1, 1),
    ("l1 1x1 64->256", 121, 213, 64, 256, 1, 1, 0),
    ("l1 1x1 256->64", 121, 213, 256, 64, 1, 1, 0),
    ("l2 1x1 512->128", 61, 107, 512, 128, 1, 1, 0),
    ("l2 3x3 128->128", 61, 107, 128, 128, 3, 1, 1),
    ("l2 1x1 128->512", 61, 107, 128, 512, 1, 1, 0),
    ("l3 1x1 1024->256", 31, 54, 1024, 256, 1, 1, 0),
    ("l3 3x3 256->256", 31, 54, 256, 256, 3, 1, 1),
    ("l3 1x1 256->1024", 31, 54, 256, 1024, 1, 1, 0),
    ("lstt linear 256->256", 1674, 1, 256, 256, 1, 1, 0),
    ("lstt linear 256->512", 1674, 1, 256, 512, 1, 1, 0),
    ("lstt linear 256->1024", 1674, 1, 256, 1024, 1, 1, 0),
    ("lstt linear 1024->256", 1674, 1, 1024, 256, 1, 1, 0),
]
REP = 20
# stamp slots 1..10 (include/aotb200.h): consumer thread 0 except "A0 stored" and "producer done" (producer thread 256);
# "staged" is split-K only, "first acc complete" persistent only; slot 8 is the split-K finish start or the persistent
# first finish stored
NAMES = ["prologue", "A0 stored", "stage0 ready", "last acc complete", "producer done", "staged", "exit",
         "finish start / first finish stored", "last finish stored", "first acc complete"]


def main():
    d = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    ws = ops._tc_workspace(d)
    results = []
    for name, H, W, Cin, Cout, K, s, p in SHAPES:
        x = torch.randn(1, H, W, Cin, generator=g).to(d)
        w = (torch.randn(K * K * Cin, Cout, generator=g) / (K * K * Cin) ** 0.5).to(d)
        wh, wl = ops.split_fp16(w)
        b = torch.randn(Cout, generator=g).to(d)
        Ho, Wo = (H + 2 * p - K) // s + 1, (W + 2 * p - K) // s + 1
        out = torch.empty(1, Ho, Wo, Cout, device=d)
        row = {"shape": name, "M": Ho * Wo, "K": K * K * Cin, "N": Cout}
        for mode in (0, 1, 2, 3):
            lib().aotb_set_conv_tiling(mode)
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(3):
                    ops.conv2d_tc(x, wh, wl, b, out, KH=K, KW=K, stride=s, pad=p, act=1)
                st.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr, stream=st):
                    for _ in range(REP):
                        ops.conv2d_tc(x, wh, wl, b, out, KH=K, KW=K, stride=s, pad=p, act=1)
                gr.replay()
                st.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                for _ in range(5):
                    gr.replay()
                e1.record(st)
                st.synchronize()
            row[f"us_mode{mode}"] = round(e0.elapsed_time(e1) * 1000 / (5 * REP), 2)
        # phase stamps, default policy (mode 0) and narrow (mode 1)
        for mode in (0, 1):
            lib().aotb_set_conv_tiling(4 | mode)
            ws.zero_()
            ops.conv2d_tc(x, wh, wl, b, out, KH=K, KW=K, stride=s, pad=p, act=1)
            torch.cuda.synchronize()
            st8 = ws.view(torch.int64)[: 12 * 4096].view(-1, 12).cpu()
            st8 = st8[st8[:, 7] != 0][:, :11]
            rel = (st8[:, 1:] - st8[:, :1]).double() / 1965.0      # cycles -> us at 1965 MHz
            rel = torch.where(st8[:, 1:] != 0, rel, torch.full_like(rel, float("nan")))
            med = torch.nanmedian(rel, dim=0).values.tolist()
            row[f"phases_us_mode{mode}"] = {n: round(v, 2) for n, v in zip(NAMES, med)}
            row[f"ctas_mode{mode}"] = int(st8.shape[0])
        lib().aotb_set_conv_tiling(0)
        flops = 2.0 * row["M"] * row["K"] * row["N"]
        row["tflops_fp32equiv_mode0"] = round(flops / row["us_mode0"] / 1e6, 1)
        results.append(row)
        print(json.dumps(row), flush=True)
    json.dump(results, open(sys.argv[1] if len(sys.argv) > 1 else "conv_microbench.json", "w"), indent=1)


if __name__ == "__main__":
    main()
