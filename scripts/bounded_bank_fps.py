#!/usr/bin/env python
"""Frame time over a long clip with the long-term bank unbounded and bounded to M = 8 memory frames (long_term_mem_max).

Workload: bench.py's synthetic R50-AOTL 480p clip (481x849 network input, 480x854 output, 10 objects, seeded random weights),
long-term gap 5, 600 propagated frames.  The clip cycles over 120 distinct synthetic frames (the frame content does not enter
the cost; 601 distinct frames would only add 2.4 GB of inputs).

Per frame the timed span is match_propogate_one_frame + decode_current_logits + the fused upsample / argmax kernel + the
nearest resize + update_memory, between two CUDA events on the stream.  Both engines share one model.  Each first runs the
whole clip once untimed (every buffer size, every KV-split count and every graph of the clip has then been seen), then the two
are alternated for --reps timed passes each.  Reported per arm: ms / frame averaged over frames 1-50, 251-300 and 551-600
(mean and min / max over the passes), the engine's peak device memory (torch.cuda.max_memory_allocated over its first pass
minus what was allocated before the engine was built), CUDA graph captures in the first pass, in its frames 51-600, and in the
timed passes, and the card's name and power limit.

    python scripts/bounded_bank_fps.py OUT_DIR [--frames 600] [--bound 8] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

H_IN, W_IN, H_OUT, W_OUT, OBJS, GAP, DISTINCT = 481, 849, 480, 854, 10, 5, 120
CAPTURES = [0]


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = r.stdout.strip().partition(",")
    return name.strip() or torch.cuda.get_device_name(0), power.strip() or "unknown"


def count_captures():
    begin = torch.cuda.CUDAGraph.capture_begin

    def counted(self, *args, **kwargs):
        CAPTURES[0] += 1
        return begin(self, *args, **kwargs)
    torch.cuda.CUDAGraph.capture_begin = counted


def step(eng, img):
    from aot_benchmark_b200 import ops
    eng.match_propogate_one_frame(img)
    eng.decode_current_logits(None)
    e0 = eng.aot_engines[0]
    label = torch.empty((1, 1, H_OUT, W_OUT), dtype=torch.float32, device=img.device)
    ops.logits_argmax(e0.pred_id_logits, label, e0.align_corners)
    small = torch.empty((1, 1) + tuple(eng.input_size_2d), dtype=torch.float32, device=img.device)
    ops.nearest_resize(label, small)
    eng.update_memory(small)


def run_clip(eng, frames, mask, n):
    """-> (ms per propagated frame [n], graph captures per propagated frame [n])"""
    eng.restart_engine()
    eng.add_reference_frame(frames[0], mask, obj_nums=[OBJS], frame_step=0)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
    caps = []
    ev[0].record()
    for t in range(1, n + 1):
        c0 = CAPTURES[0]
        step(eng, frames[t % len(frames)])
        ev[t].record()
        caps.append(CAPTURES[0] - c0)
    torch.cuda.synchronize()
    return [ev[t - 1].elapsed_time(ev[t]) for t in range(1, n + 1)], caps


def windows(n):
    return {"1-50": (0, 50), f"{n // 2 - 49}-{n // 2}": (n // 2 - 50, n // 2), f"{n - 49}-{n}": (n - 50, n)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--bound", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bounded_bank_fps.py needs a CUDA device (no CPU path)")
    if a.frames < 150:
        raise SystemExit("--frames must be at least 150 (three 50-frame windows)")
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    from aot_benchmark_b200.plan import get_plan
    from oracle.aot_oracle import synthetic_video            # input generator only (shared with the tests and bench.py)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    count_captures()
    gpu, power = gpu_info()
    print(f"GPU: {gpu}, power limit {power}", flush=True)
    frames, mask = synthetic_video(DISTINCT, H_IN, W_IN, OBJS, seed=1234)
    frames, mask = [f.to(dev) for f in frames], mask.to(dev)
    cfg = EngineConfig("fps", "r50_aotl")
    torch.manual_seed(0)
    model = build_vos_model(cfg.MODEL_VOS, cfg).to(dev).eval()
    get_plan(model)                                           # packed weights: shared, so in neither engine's footprint
    arms = {"unbounded": None, f"M = {a.bound}": a.bound}
    engines, rec_arms = {}, {}
    with torch.no_grad():
        for name, M in arms.items():
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=GAP,
                               short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP, long_term_mem_max=M).eval()
            _, caps = run_clip(eng, frames, mask, a.frames)
            e0 = eng.aot_engines[0]
            engines[name] = eng
            rec_arms[name] = {"engine_peak_mib": (torch.cuda.max_memory_allocated() - base) / 2 ** 20,
                              "bank_frames_live": e0.bank_len // e0.enc_hw, "bank_frames_capacity": e0.bank_cap // e0.enc_hw,
                              "captures_first_pass": sum(caps), "captures_first_pass_after_frame_50": sum(caps[50:]),
                              "captures_timed_passes": 0, "passes": []}
        for rep in range(a.reps):
            for name in arms:
                ms, caps = run_clip(engines[name], frames, mask, a.frames)
                r = rec_arms[name]
                r["captures_timed_passes"] += sum(caps)
                r["passes"].append({w: sum(ms[lo:hi]) / (hi - lo) for w, (lo, hi) in windows(a.frames).items()})
    for name, r in rec_arms.items():
        r["ms_per_frame"] = {}
        for w in windows(a.frames):
            v = [p[w] for p in r["passes"]]
            r["ms_per_frame"][w] = {"mean": sum(v) / len(v), "min": min(v), "max": max(v)}
        print(f"{name}: " + ", ".join(f"frames {w}: {s['mean']:.3f} ms ({s['min']:.3f}-{s['max']:.3f})"
                                      for w, s in r["ms_per_frame"].items())
              + f"; engine peak {r['engine_peak_mib']:.0f} MiB; bank {r['bank_frames_live']} / {r['bank_frames_capacity']} frames; "
              f"captures {r['captures_first_pass']} in the first pass ({r['captures_first_pass_after_frame_50']} after frame 50), "
              f"{r['captures_timed_passes']} in {a.reps} timed passes", flush=True)
    rec = {"gpu": gpu, "power_limit": power,
           "workload": f"synthetic R50-AOTL {H_IN}x{W_IN} -> {H_OUT}x{W_OUT}, {OBJS} objects, gap {GAP}, {a.frames} propagated "
                       f"frames cycling over {DISTINCT}, one untimed pass then {a.reps} alternated timed passes per arm",
           "arms": rec_arms}
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "bounded_bank_fps.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
