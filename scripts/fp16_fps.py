#!/usr/bin/env python
"""Frame time of the fp16 inference mode (precision="fp16") against the default fp32 mode on the H100 path.

Workloads, each on one seeded random-init model shared by both engines:
  R50-AOTL   480p clip of bench.py (network input 481x849), 10 objects;
  R50-DeAOTL the same clip;
  SwinB-AOTL 1.3x480p (network input 592x1040), 10 objects.
The clip has 10 distinct seeded synthetic frames, cycled; long-term gap 5 (the configs' TEST_LONG_TERM_MEM_GAP).  Per model both
engines run the clip once untimed, then alternate for --reps timed passes of --frames propagated frames.  A pass is timed with
CUDA events from its first propagate to its last memory update; each frame is propagate, decode at the input size, argmax and
memory update with the engine's own label.  Reported per model and mode: ms / frame (mean, min-max over passes), and between the
modes over the last pass: the largest |logit| difference (live channels) and the label pixels that differ.
The card's name, power limit and max SM clock are read in the same run.

    python scripts/fp16_fps.py OUT_DIR [--frames 30] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

OBJS, DISTINCT = 10, 10
MODELS = [("r50_aotl", 481, 849), ("r50_deaotl", 481, 849), ("swinb_aotl", 592, 1040)]


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return [s.strip() for s in r.stdout.strip().split(",")] if r.stdout.strip() else [torch.cuda.get_device_name(0), "?", "?"]


def run_pass(eng, frames, mask, n, out_size, keep=False):
    """Reference frame + n propagated frames -> (ms / propagated frame, [(logits, label)] per frame if keep)."""
    eng.restart_engine()
    eng.add_reference_frame(frames[0], mask, obj_nums=[OBJS], frame_step=0)
    kept = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for t in range(1, n + 1):
        eng.match_propogate_one_frame(frames[1 + (t - 1) % DISTINCT])
        lg = eng.decode_current_logits(out_size)
        label = lg.argmax(1, keepdim=True).float()
        if keep:
            kept.append((lg[:, :OBJS + 1].clone(), label.clone()))
        eng.update_memory(label)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, kept


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    from oracle.aot_oracle import synthetic_video
    dev = torch.device("cuda:0")
    name, power, clock = gpu_info()
    rows = []
    for model_name, H, W in MODELS:
        cfg = EngineConfig("fp16_fps", model_name)
        torch.manual_seed(0)
        model = build_vos_model(cfg.MODEL_VOS, cfg).to(dev).eval()
        engines = {p: build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0,
                                   long_term_mem_gap=cfg.TEST_LONG_TERM_MEM_GAP,
                                   short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP, precision=p).eval()
                   for p in ("fp32", "fp16")}
        frames, mask = synthetic_video(DISTINCT + 1, H, W, OBJS, seed=1234)
        frames, mask = [f.to(dev) for f in frames], mask.to(dev)
        times = {p: [] for p in engines}
        kept = {}
        with torch.no_grad():
            for p, eng in engines.items():
                run_pass(eng, frames, mask, args.frames, (H, W))          # warm-up: module loads, graph capture
            for rep in range(args.reps):
                for p, eng in engines.items():
                    ms, k = run_pass(eng, frames, mask, args.frames, (H, W), keep=rep == args.reps - 1)
                    times[p].append(ms)
                    if k:
                        kept[p] = k
        dlogit = max((a[0] - b[0]).abs().max().item() for a, b in zip(kept["fp32"], kept["fp16"]))
        dlabel = sum(int((a[1] != b[1]).sum().item()) for a, b in zip(kept["fp32"], kept["fp16"]))
        row = {"model": model_name, "net_input": [H, W], "objects": OBJS, "frames": args.frames,
               "reps": args.reps, "gpu": name, "power_limit": power, "max_sm_clock": clock,
               "max_abs_dlogit": dlogit, "label_pixels_differing": dlabel, "label_pixels": args.frames * H * W}
        for p, ts in times.items():
            row[f"{p}_ms_per_frame"] = round(sum(ts) / len(ts), 3)
            row[f"{p}_ms_range"] = [round(min(ts), 3), round(max(ts), 3)]
        row["speedup"] = round(row["fp32_ms_per_frame"] / row["fp16_ms_per_frame"], 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
        del engines, model
        torch.cuda.empty_cache()
    json.dump(rows, open(os.path.join(args.out_dir, "fp16_fps.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
