"""Aggregate frames/s of n independent videos of more than 10 objects: (a) one MultiVideoInferEngine(max_videos=n,
max_lanes=its videos' lanes) (DeAOTMultiVideoInferEngine for a DeAOT model), one batched pass per frame over every video's
ID-bank lanes; (b) n AOTInferEngines (DeAOTInferEngines) on concurrent streams through engine.fork_join; (c) the same n engines
one after another.  Per step: propagate + decode to labels at the output size (the aggregated logits' first argmax) + memory
update, timed between CUDA events; the arms alternate in one session after an untimed pass each.  Workloads: n in --videos
videos of 20 objects (2 lanes each), and a mix of 5, 14 and 23 objects (1 + 2 + 3 lanes).  Seeded random weights,
long_term_mem_max 8, gap 5.  Prints the card's name and power limit, then one JSON line per (model, workload, arm)."""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from tta_fps import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="r50_aotl,r50_deaotl")
    ap.add_argument("--videos", default="1,2,4")
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--size", default="481,849")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    from aot_benchmark_b200 import engine as E
    from aot_benchmark_b200.multi_video import DeAOTMultiVideoInferEngine, MultiVideoInferEngine
    from oracle import weights as OW
    H, W = (int(s) for s in a.size.split(","))
    out_size = (480, 854)
    M, gap = 8, 5
    gpu, power, clock = gpu_info()
    print(f"GPU: {gpu}, power limit {power}, max SM clock {clock}", flush=True)
    workloads = [(f"{n}x20", [20] * n) for n in (int(s) for s in a.videos.split(","))] + [("mix_5_14_23", [5, 14, 23])]
    rows = []
    for name in a.models.split(","):
        cfg = EngineConfig("fps", name)
        model = build_vos_model(cfg.MODEL_VOS, cfg)
        model.load_state_dict(OW.build_state_dict(name, seed=0))
        model = model.cuda().eval()
        deaot = cfg.MODEL_VOS == "deaot"
        Multi, Single = (DeAOTMultiVideoInferEngine, E.DeAOTInferEngine) if deaot else (MultiVideoInferEngine, E.AOTInferEngine)
        g = torch.Generator(device="cuda").manual_seed(0)
        frame = torch.randn(1, 3, H, W, device="cuda", generator=g)
        for label, objs in workloads:
            n = len(objs)
            masks = [torch.randint(0, o + 1, (1, 1, H, W), device="cuda", generator=g).float() for o in objs]
            lanes = sum(max(-(-o // 10), 1) for o in objs)
            multi = Multi(model, max_videos=n, long_term_mem_max=M, long_term_mem_gap=gap, max_lanes=lanes)
            singles = [Single(model, long_term_mem_gap=gap, long_term_mem_max=M) for _ in range(n)]
            owner = type("Owner", (), {})()

            def run_multi(T):
                vids = [multi.open_video(frame, m, o) for m, o in zip(masks, objs)]
                for _ in range(T):
                    multi.propagate({v: frame for v in vids})
                    labs = multi.decode_labels(out_size)
                    multi.update_memory({v: F.interpolate(labs[v][None].float(), size=(H, W), mode="nearest") for v in vids})
                for v in vids:
                    multi.close_video(v)

            def step_single(e):          # AOTInferEngine's decode: aggregated logits at the output size, then their argmax
                e.match_propogate_one_frame(frame)
                lab = e.decode_current_logits(out_size).argmax(1, keepdim=True).float()
                e.update_memory(F.interpolate(lab, size=(H, W), mode="nearest"))

            def run_single(T, concurrent):
                for e, m, o in zip(singles, masks, objs):
                    e.restart_engine()
                    e.add_reference_frame(frame, m, obj_nums=[o], frame_step=0)
                if concurrent:
                    for _ in range(T):
                        E.fork_join(owner, singles, lambda i, e: step_single(e))
                else:
                    for e in singles:
                        for _ in range(T):
                            step_single(e)

            arms = {"a_multi": run_multi, "b_streams": lambda T: run_single(T, True),
                    "c_sequential": lambda T: run_single(T, False)}
            with torch.no_grad():
                for fn in arms.values():
                    fn(3)                                  # untimed: captures, allocations
                torch.cuda.synchronize()
                times = {k: [] for k in arms}
                for _ in range(2):
                    for k, fn in arms.items():
                        torch.cuda.reset_peak_memory_stats()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        fn(a.frames)
                        e1.record()
                        torch.cuda.synchronize()
                        times[k].append((e0.elapsed_time(e1), torch.cuda.max_memory_allocated() / 2 ** 30))
            for k, v in times.items():
                best = min(t for t, _ in v)
                r = dict(model=name, workload=label, objects=objs, lanes=lanes, arm=k, frames=a.frames,
                         fps=round(n * a.frames / (best / 1e3), 1), ms_per_step=round(best / a.frames, 3),
                         peak_gib=round(max(m for _, m in v), 2), card=gpu, power_limit=power)
                print(json.dumps(r), flush=True)
                rows.append(r)
            del multi, singles
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
