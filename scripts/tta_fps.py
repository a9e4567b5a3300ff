#!/usr/bin/env python
"""Frame time of test-time augmentation (flip + scales [1.0, 1.3], E = 4 augmentations) on the H100 path.

Workload: a seeded synthetic uint8 480x854 clip (10 distinct frames, cycled), FramePreprocessor with the reference's
TEST_MAX_LONG_EDGE = 1040, 10 objects, long-term gap 5, 50 propagated frames, R50-AOTL and AOTT with seeded random weights.
Arms, all in one process on one model per network:
  (a) evaluator  -- the exact calls of networks/managers/evaluator.py:284-422 over four drop-in AOTInferEngines, including
                    torch.cuda.empty_cache() per augmentation and the eager flip / softmax / mean / argmax / interpolate;
  (b) tta        -- TTAInferEngine.propagate;
  (c) no_tta     -- one engine on the unflipped 1.0 image: propagate, decode, fused upsample + argmax, nearest resize, memory.
Each arm runs the clip once untimed, then the arms alternate for --reps timed passes.  A frame is timed with CUDA events from
before augmentation 0's propagate to after the last update_memory.  Reported: ms / frame (mean and min-max over the passes),
the count of label pixels where (a) and (b) differ over the last pass, and the card's name, power limit and max SM clock.

    python scripts/tta_fps.py OUT_DIR [--frames 50] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

H, W, OBJS, GAP, DISTINCT, SCALES = 480, 854, 10, 5, 10, [1.0, 1.3]


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return [s.strip() for s in r.stdout.strip().split(",")] if r.stdout.strip() else [torch.cuda.get_device_name(0), "?", "?"]


def evaluator_frame(engines, imgs, flips):
    """evaluator.py:284-361 and :400-422 (no new objects, MODEL_USE_PREV_PROB off)."""
    all_preds = []
    for eng, img, f in zip(engines, imgs, flips):
        torch.cuda.empty_cache()
        eng.match_propogate_one_frame(img)
        logit = eng.decode_current_logits((H, W))
        if f:
            logit = torch.flip(logit, dims=[3])
        all_preds.append(torch.softmax(logit, dim=1))
    labels = [torch.argmax(torch.mean(p, dim=0, keepdim=True), dim=1, keepdim=True).float() for p in all_preds]
    pred_label = torch.argmax(torch.mean(torch.cat(all_preds, dim=0), dim=0, keepdim=True), dim=1, keepdim=True).float()
    for eng, lab, f in zip(engines, labels, flips):
        lab = torch.flip(lab, dims=[3]) if f else lab
        eng.update_memory(F.interpolate(lab, size=eng.input_size_2d, mode="nearest"))
    return pred_label


def no_tta_frame(eng, img):
    from aot_benchmark_b200 import ops
    eng.match_propogate_one_frame(img)
    eng.decode_current_logits(None)
    e0 = eng.aot_engines[0]
    label = torch.empty((1, 1, H, W), dtype=torch.float32, device=img.device)
    ops.logits_argmax(e0.pred_id_logits, label, e0.align_corners)
    small = torch.empty((1, 1) + tuple(eng.input_size_2d), dtype=torch.float32, device=img.device)
    ops.nearest_resize(label, small)
    eng.update_memory(small)
    return label


def run(arm, eng, clip, mask, n, flips):
    """-> (ms per propagated frame, uint8 labels per frame)"""
    if arm == "evaluator":
        for e, img, f in zip(eng, clip[0], flips):
            e.restart_engine()
            m = torch.flip(mask, dims=[3]) if f else mask
            e.add_reference_frame(img, F.interpolate(m, size=img.shape[2:], mode="nearest"), frame_step=0, obj_nums=[OBJS])
    elif arm == "tta":
        eng.restart_engine()
        eng.add_reference_frame(clip[0], mask, obj_nums=OBJS)
    else:
        eng.restart_engine()
        eng.add_reference_frame(clip[0][0], F.interpolate(mask, size=clip[0][0].shape[2:], mode="nearest"), frame_step=0,
                                obj_nums=[OBJS])
    torch.cuda.synchronize()
    ms, labels = [], []
    for t in range(1, n + 1):
        imgs = clip[t % len(clip)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if arm == "evaluator":
            lab = evaluator_frame(eng, imgs, flips)
        elif arm == "tta":
            lab = eng.propagate(imgs, (H, W))
        else:
            lab = no_tta_frame(eng, imgs[0])
        e1.record()
        labels.append(lab.to(torch.uint8).reshape(H, W))
        ms.append((e0, e1))
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ms], labels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--models", default="r50_aotl,aott")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tta_fps.py needs a CUDA device (no CPU path)")
    from aot_benchmark_b200 import EngineConfig, TTAInferEngine, build_engine, build_vos_model
    from aot_benchmark_b200.io_side import FramePreprocessor
    from oracle.aot_oracle import synthetic_video                 # input generators only
    from oracle.tta_oracle import synthetic_frames_u8
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu, power, clock = gpu_info()
    print(f"GPU: {gpu}, power limit {power}, max SM clock {clock}", flush=True)
    _, mask = synthetic_video(1, H, W, OBJS, seed=1234)
    mask = mask.to(dev)
    flips = [f for _ in SCALES for f in (False, True)]
    rec = {"gpu": gpu, "power_limit": power, "max_sm_clock": clock,
           "workload": f"synthetic uint8 {H}x{W} clip ({DISTINCT} distinct frames), flip + scales {SCALES} (E = 4, max long "
                       f"edge 1040), {OBJS} objects, gap {GAP}, {a.frames} propagated frames; one untimed pass per arm, then "
                       f"{a.reps} alternated timed passes", "models": {}}
    for name in a.models.split(","):
        cfg = EngineConfig("fps", name)
        torch.manual_seed(0)
        model = build_vos_model(cfg.MODEL_VOS, cfg).to(dev).eval()
        prep = FramePreprocessor(None, 800 * 1.3, True, SCALES, cfg.MODEL_ALIGN_CORNERS)
        clip = [prep(f) for f in synthetic_frames_u8(DISTINCT, H, W, seed=99)]
        mk = lambda: build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=GAP).eval()
        engines = {"evaluator": [mk() for _ in flips],
                   "tta": TTAInferEngine(model, long_term_mem_gap=GAP, flip=True, multi_scale=SCALES),
                   "no_tta": mk()}
        res = {k: [] for k in engines}
        last = {}
        with torch.no_grad():
            for arm, eng in engines.items():
                run(arm, eng, clip, mask, a.frames, flips)
            for _ in range(a.reps):
                for arm, eng in engines.items():
                    ms, labels = run(arm, eng, clip, mask, a.frames, flips)
                    res[arm].append(sum(ms) / len(ms))
                    last[arm] = labels
        diff = sum(int((x != y).sum()) for x, y in zip(last["evaluator"], last["tta"]))
        out = {arm: {"ms_per_frame_mean": sum(v) / len(v), "min": min(v), "max": max(v)} for arm, v in res.items()}
        out["label_pixels_differing_evaluator_vs_tta"] = diff
        out["label_pixels_total"] = a.frames * H * W
        out["aug_sizes"] = [tuple(i.shape[2:]) for i in clip[0]]
        rec["models"][name] = out
        print(f"{name}: " + "; ".join(f"{arm} {out[arm]['ms_per_frame_mean']:.2f} ms ({out[arm]['min']:.2f}-"
                                      f"{out[arm]['max']:.2f})" for arm in res)
              + f"; evaluator vs tta label pixels differing: {diff} of {a.frames * H * W}; augs {out['aug_sizes']}", flush=True)
        del engines
        torch.cuda.empty_cache()
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "tta_fps.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
