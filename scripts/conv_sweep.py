#!/usr/bin/env python
"""Sweep the N tile x split-K factor of the tensor-core conv on the shapes of one R50-AOTL 480p frame (graph-replayed,
L2-warm, CUDA events) -- the data behind the tile policy in aotb_conv2d_nhwc_tc.  GPU only; writes the rows as JSON to the
path given as the first argument (default conv_sweep.json).  --single-pass also sweeps the single-pass kernel (wl = NULL, the
fp16 inference mode) on the same shapes and inputs: one row per shape and mode."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aot_benchmark_b200 import ops  # noqa: E402
from aot_benchmark_b200._lib import lib  # noqa: E402
from conv_microbench import SHAPES  # noqa: E402

REP = 20
EXTRA = [("dec 3x3 256->256 @8x", 61, 107, 256, 256, 3, 1, 1), ("dec 3x3 256->256 @4x", 121, 213, 256, 256, 3, 1, 1),
         ("l2 ds 1x1s2 256->512", 121, 213, 256, 512, 1, 2, 0), ("l3 ds 1x1s2 512->1024", 61, 107, 512, 1024, 1, 2, 0),
         ("l3 3x3s2 256->256", 61, 107, 256, 256, 3, 2, 1), ("l2 3x3s2 128->128", 121, 213, 128, 128, 3, 2, 1),
         ("stem 7x7s2 4->64", 481, 849, 4, 64, 7, 2, 3), ("l2 1x1 256->128", 121, 213, 256, 128, 1, 1, 0)]


def time_graph(fn):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(2):
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
    d = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    results = []
    modes = ("fp32", "fp16") if "--single-pass" in sys.argv else ("fp32",)
    for name, H, W, Cin, Cout, K, s, p in SHAPES + EXTRA:
        x = torch.randn(1, H, W, Cin, generator=g).to(d)
        w = (torch.randn(K * K * Cin, Cout, generator=g) / (K * K * Cin) ** 0.5).to(d)
        wh, wl = ops.split_fp16(w)
        b = torch.randn(Cout, generator=g).to(d)
        Ho, Wo = (H + 2 * p - K) // s + 1, (W + 2 * p - K) // s + 1
        out = torch.empty(1, Ho, Wo, Cout, device=d)
        nchunks = (K * K * Cin + 63) // 64
        mt = (Ho * Wo + 127) // 128
        for mode in modes:
            results.append(sweep_shape(name, x, wh, wl if mode == "fp32" else None, b, out, K, s, p, Cout, nchunks, mt, mode))
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    json.dump(results, open(args[0] if args else "conv_sweep.json", "w"), indent=1)


def sweep_shape(name, x, wh, wl, b, out, K, s, p, Cout, nchunks, mt, mode):
    row = {"shape": name, "mode": mode, "M": out.shape[1] * out.shape[2], "K": K * K * x.shape[3], "N": Cout, "us": {}}
    fn = lambda: ops.conv2d_tc(x, wh, wl, b, out, KH=K, KW=K, stride=s, pad=p, act=1)  # noqa: E731
    lib().aotb_set_conv_tiling(0)
    row["us"]["policy"] = round(time_graph(fn), 2)
    # the same tiling with the weights declared constant (first weight tiles fetched before the grid dependency wait)
    row["us"]["policy_const_w"] = round(time_graph(
        lambda: ops.conv2d_tc(x, wh, wl, b, out, KH=K, KW=K, stride=s, pad=p, act=1, const_w=True)), 2)
    for bi, BN in ((1, 64), (2, 128), (3, 256)):
        if Cout % BN:
            continue
        for S in (1, 2, 4, 8):
            ctas = mt * (Cout // BN) * S
            if S > nchunks or (S > 1 and ctas > 320):
                continue
            lib().aotb_set_conv_tiling((bi << 4) | (S << 8))
            row["us"][f"bn{BN}_s{S}"] = round(time_graph(fn), 2)
    lib().aotb_set_conv_tiling(0)
    best = min((k for k in row["us"] if k != "policy_const_w"), key=row["us"].get)
    row["best"] = best
    print(json.dumps(row), flush=True)
    return row


if __name__ == "__main__":
    main()
