#!/usr/bin/env python
"""Per-kernel GPU time per frame of the bench.py workload (R50-AOTL, 480p, 10 objects), from one torch.profiler pass.

The clip is the one bench.py times.  After a warm-up clip (module loads, buffers) the engine restarts, takes the reference
frame and propagates FRAMES frames under the profiler.  Launches are eager (engine.LT_PROBE set, as bench.py's probe passes
do): graph replays hide their kernels from the profiler.  Kernel times are the device durations of the trace; gaps between
kernels are not counted.  GPU only.

    python scripts/frame_kernel_shares.py OUT_DIR [--frames 20] [--model r50_aotl]

Writes OUT_DIR/frame_kernel_shares.json (per kernel: launches and microseconds per frame, share of kernel time; the
tensor-core conv family summed; the conv launches of one frame in order) and prints the table."""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402

CONV_FAMILY = ("conv_tc_kernel", "conv3x3_halo_kernel")


def _short(name):
    n = re.sub(r"\(.*", "", name).replace("void ", "").replace("aotb::", "").replace("tc::", "")
    return n.strip()


def _gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--model", default="r50_aotl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frame_kernel_shares.py needs a CUDA device")
    from aot_benchmark_b200 import engine as engine_mod
    bench.set_workload(args.model)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _, _, eng = bench.build_model(args.model, dev)
    n = args.frames
    frames, mask = bench.make_clip(n + 1, seed=1234)
    frames = [f.to(dev) for f in frames]
    mask = mask.to(dev)
    engine_mod.LT_PROBE = []                     # eager launches: every kernel shows up in the trace

    def clip(k):
        eng.restart_engine()
        eng.add_reference_frame(frames[0], mask, obj_nums=[bench.OBJS], frame_step=0)
        for t in range(1, k + 1):
            bench.step_fused(eng, frames[t])

    with torch.no_grad():
        clip(min(n, 6))
        torch.cuda.synchronize()
        eng.restart_engine()
        eng.add_reference_frame(frames[0], mask, obj_nums=[bench.OBJS], frame_step=0)
        torch.cuda.synchronize()
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            for t in range(1, n + 1):
                bench.step_fused(eng, frames[t])
            torch.cuda.synchronize()
    engine_mod.LT_PROBE = None
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    agg = collections.defaultdict(lambda: [0, 0.0])
    for ev in trace.get("traceEvents", []):
        if ev.get("cat") == "kernel" and "dur" in ev:
            a = agg[_short(ev["name"])]
            a[0] += 1
            a[1] += float(ev["dur"])
    # the conv launches of one frame in launch order (every frame launches the same sequence), time averaged over frames
    convs = sorted((ev for ev in trace.get("traceEvents", [])
                    if ev.get("cat") == "kernel" and "dur" in ev and any(f in ev["name"] for f in CONV_FAMILY)),
                   key=lambda ev: ev["ts"])
    per = len(convs) // n if n else 0
    conv_launches = [{"kernel": _short(convs[i]["name"]), "grid": convs[i].get("args", {}).get("grid"),
                      "us": round(sum(float(convs[i + f * per]["dur"]) for f in range(n)) / n, 2)} for i in range(per)]
    total = sum(v[1] for v in agg.values())
    rows = [{"kernel": k, "launches_per_frame": round(c / n, 2), "us_per_frame": round(t / n, 2),
             "share": round(t / total, 4) if total else 0.0}
            for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])]
    conv = [r for r in rows if any(f in r["kernel"] for f in CONV_FAMILY)]
    out = {"model": args.model, "frames": n, "gpu": _gpu_info(),
           "timing": "torch.profiler kernel durations, eager launches (no CUDA graphs, no PDL overlap)",
           "kernel_us_per_frame": round(total / n, 2),
           "conv_tc_family": {"us_per_frame": round(sum(r["us_per_frame"] for r in conv), 2),
                              "share": round(sum(r["share"] for r in conv), 4),
                              "launches_per_frame": round(sum(r["launches_per_frame"] for r in conv), 2)},
           "kernels": rows, "conv_launches_per_frame": conv_launches}
    os.makedirs(args.out_dir, exist_ok=True)
    json.dump(out, open(os.path.join(args.out_dir, "frame_kernel_shares.json"), "w"), indent=1)
    print(f"gpu: {out['gpu']}; kernel time {out['kernel_us_per_frame']:.1f} us/frame over {n} frames; "
          f"conv_tc family {out['conv_tc_family']['share'] * 100:.1f}%")
    for r in rows[:25]:
        print(f"{r['share'] * 100:5.1f}%  {r['launches_per_frame']:6.1f}/frame  {r['us_per_frame']:8.1f} us/frame  "
              f"{r['kernel'][:90]}")


if __name__ == "__main__":
    main()
