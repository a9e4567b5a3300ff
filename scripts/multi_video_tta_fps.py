#!/usr/bin/env python
"""Throughput of flip + multi-scale test-time augmentation over n videos at once (flip + scales [1.0, 1.3], E = 4).

Workload (as scripts/tta_fps.py): seeded synthetic uint8 480x854 clips (10 distinct frames each, cycled, one seed per video),
FramePreprocessor with TEST_MAX_LONG_EDGE = 1040, 10 objects, long-term gap 5, bounded banks of M = 8 memory frames, seeded
random weights.  Arms, per model and n:
  (a) multi    -- MultiVideoTTAInferEngine.propagate over the n videos;
  (b) streams  -- n TTAInferEngine(long_term_mem_max=8), one per video, on concurrent streams (engine.fork_join);
  (c) serial   -- the same n engines one after another.
Each arm is built and run once untimed (its peak allocated memory above what was allocated before it was built is taken
there), then the arms alternate for --reps timed passes.  Every pass opens its videos and runs WARM untimed frames first:
(a)'s reopen trims its encoders to the new lane counts, and the first frames after that run eagerly and capture their
graphs again, so only frames WARM + 1 .. WARM + --frames are timed, with CUDA events, in every arm.  Reported: aggregate
video-frames/s (mean and min-max over the passes), the peak allocated memory per arm, the label pixels where (a) and (b)
differ over the last pass's timed frames, and the card's name, power limit and max SM clock.  Then the ensemble alone at the
workload's sizes: one aotb_tta_merge_batched_f32 launch against, per video, E logits_postproc + one aotb_tta_merge_f32.

    python scripts/multi_video_tta_fps.py OUT_DIR [--frames 30] [--reps 3] [--ns 1,2,4] [--models r50_aotl,aott,r50_deaotl]
"""
import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))

from tta_fps import gpu_info  # noqa: E402

H, W, OBJS, GAP, DISTINCT, SCALES, M = 480, 854, 10, 5, 10, [1.0, 1.3], 8
WARM = 2            # untimed frames per pass: the first runs eagerly, the second captures


class Serial:
    """n one-video TTA engines; propagate runs them concurrently (fork_join) or one after another."""

    def __init__(self, engines, concurrent):
        self.engines, self.concurrent = engines, concurrent

    def open(self, clips, mask):
        for e, c in zip(self.engines, clips):
            e.restart_engine()
            e.add_reference_frame(c[0], mask, obj_nums=OBJS)

    def frame(self, clips, t):
        from aot_benchmark_b200 import engine as E
        step = lambda i, e: e.propagate(clips[i][t % len(clips[i])], (H, W))
        if self.concurrent:
            return E.fork_join(self, self.engines, step)
        return [step(i, e) for i, e in enumerate(self.engines)]


def run(arm, eng, clips, mask, frames):
    """-> (aggregate video-frames/s, uint8 labels of video 0 .. n-1 per frame)"""
    if arm == "multi":
        for v in list(eng.videos):
            eng.close_video(v)
        vids = [eng.open_video(c[0], mask, OBJS) for c in clips]
    else:
        eng.open(clips, mask)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    labels = []
    for t in range(1, WARM + frames + 1):
        if t == WARM + 1:
            torch.cuda.synchronize()
            e0.record()
        if arm == "multi":
            out = eng.propagate({v: clips[i][t % len(clips[i])] for i, v in enumerate(vids)}, (H, W))
            labs = [out[v] for v in vids]
        else:
            labs = eng.frame(clips, t)
        if t > WARM:
            labels.append(torch.stack([l.reshape(H, W) for l in labs]).to(torch.uint8))
    e1.record()
    torch.cuda.synchronize()
    return len(clips) * frames / (e0.elapsed_time(e1) / 1e3), labels


def merge_timing(n, sizes, reps=50):
    """-> (us per batched merge of n videos, us per n x (E logits_postproc + tta_merge)) at the given low-res sizes."""
    from aot_benchmark_b200 import ops
    E, NC = 2 * len(sizes), 11
    g = torch.Generator(device="cpu").manual_seed(0)
    pools = [(torch.randn((2 * n,) + s + (NC,), generator=g) * 8).cuda() for s in sizes]
    maps = [pools[e // 2] for e in range(E)]
    flips = [bool(e % 2) for e in range(E)]
    lanes = [[2 * b + e % 2 for e in range(E)] for b in range(n)]
    label = torch.empty((n, 1, H, W), device="cuda")
    prob = torch.empty((n, NC, H, W), device="cuda")
    lo = [torch.empty((1, NC) + s, device="cuda") for s in sizes for _ in range(2)]
    lab1 = torch.empty((1, 1, H, W), device="cuda")

    def batched():
        ops.tta_merge_batched(maps, flips, lanes, [OBJS] * n, label, True, prob=prob)

    def per_video():
        for b in range(n):
            for e in range(E):
                ops.logits_postproc(maps[e][lanes[b][e]:lanes[b][e] + 1], lo[e], None, OBJS, True)
            ops.tta_merge(lo, flips, lab1, True, prob=prob[b:b + 1])
    out = []
    for fn in (batched, per_video):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e3 / reps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ns", default="1,2,4")
    ap.add_argument("--models", default="r50_aotl,aott,r50_deaotl")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_video_tta_fps.py needs a CUDA device (no CPU path)")
    from aot_benchmark_b200 import EngineConfig, MultiVideoTTAInferEngine, TTAInferEngine, build_vos_model
    from aot_benchmark_b200.io_side import FramePreprocessor
    from oracle.aot_oracle import synthetic_video                 # input generators only
    from oracle.tta_oracle import synthetic_frames_u8
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu, power, clock = gpu_info()
    print(f"GPU: {gpu}, power limit {power}, max SM clock {clock}", flush=True)
    _, mask = synthetic_video(1, H, W, OBJS, seed=1234)
    mask = mask.to(dev)
    rec = {"gpu": gpu, "power_limit": power, "max_sm_clock": clock,
           "workload": f"n synthetic uint8 {H}x{W} clips ({DISTINCT} distinct frames each), flip + scales {SCALES} (E = 4, "
                       f"max long edge 1040), {OBJS} objects, gap {GAP}, M = {M}, {a.frames} timed frames per pass after "
                       f"{WARM} untimed ones; one untimed pass per arm, then {a.reps} alternated timed passes", "models": {}}
    for name in filter(None, a.models.split(",")):          # --models "": the ensemble timing alone
        cfg = EngineConfig("fps", name)
        torch.manual_seed(0)
        model = build_vos_model(cfg.MODEL_VOS, cfg).to(dev).eval()
        prep = FramePreprocessor(None, 800 * 1.3, True, SCALES, cfg.MODEL_ALIGN_CORNERS)
        rec["models"][name] = {}
        for n in [int(x) for x in a.ns.split(",")]:
            clips = [[prep(f) for f in synthetic_frames_u8(DISTINCT, H, W, seed=99 + v)] for v in range(n)]
            builders = {
                "multi": lambda: MultiVideoTTAInferEngine(model, max_videos=n, long_term_mem_max=M, long_term_mem_gap=GAP,
                                                          flip=True, multi_scale=SCALES),
                "streams": lambda: Serial([TTAInferEngine(model, long_term_mem_gap=GAP, flip=True, multi_scale=SCALES,
                                                          long_term_mem_max=M) for _ in range(n)], True),
                "serial": lambda: Serial([TTAInferEngine(model, long_term_mem_gap=GAP, flip=True, multi_scale=SCALES,
                                                         long_term_mem_max=M) for _ in range(n)], False)}
            engines, peak, fps, last = {}, {}, {k: [] for k in builders}, {}
            try:
                with torch.no_grad():
                    for arm, mk in builders.items():
                        torch.cuda.synchronize()
                        base = torch.cuda.memory_allocated()
                        torch.cuda.reset_peak_memory_stats()
                        engines[arm] = mk()
                        run(arm, engines[arm], clips, mask, a.frames)
                        torch.cuda.synchronize()
                        peak[arm] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
                    for _ in range(a.reps):
                        for arm, eng in engines.items():
                            f, labels = run(arm, eng, clips, mask, a.frames)
                            fps[arm].append(f)
                            last[arm] = labels
            except torch.cuda.OutOfMemoryError:
                print(f"{name} n={n}: out of memory", flush=True)
                rec["models"][name][n] = "out of memory"
                del engines
                torch.cuda.empty_cache()
                continue
            diff = sum(int((x != y).sum()) for x, y in zip(last["multi"], last["streams"]))
            out = {arm: {"video_frames_per_s_mean": sum(v) / len(v), "min": min(v), "max": max(v),
                         "peak_alloc_gib": peak[arm]} for arm, v in fps.items()}
            out["label_pixels_differing_multi_vs_streams"] = diff
            out["label_pixels_total"] = a.frames * n * H * W
            rec["models"][name][n] = out
            print(f"{name} n={n}: " + "; ".join(f"{arm} {out[arm]['video_frames_per_s_mean']:.1f} fr/s ({out[arm]['min']:.1f}-"
                                               f"{out[arm]['max']:.1f}), peak {peak[arm]:.2f} GiB" for arm in fps)
                  + f"; multi vs streams label pixels differing: {diff} of {a.frames * n * H * W}", flush=True)
            del engines
            torch.cuda.empty_cache()
    # the decoder's stride-4 maps of the two scales' network inputs (FramePreprocessor: 481x849 and 625x1105 here)
    sizes = [((h + 3) // 4, (w + 3) // 4) for h, w in ((481, 849), (625, 1105))]
    rec["merge_us"] = {}
    for n in [int(x) for x in a.ns.split(",")]:
        bat, per = merge_timing(n, sizes)
        rec["merge_us"][n] = {"batched": bat, "per_video": per}
        print(f"ensemble, n={n}, E=4, low-res {sizes}: one batched merge {bat:.1f} us; per video E postproc + merge "
              f"{per:.1f} us", flush=True)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "multi_video_tta_fps.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
