#!/usr/bin/env python
"""Frames per second of the encoder variants a user selects through cfg.MODEL_ENCODER: R50-AOTL, AOTL with MobileNetV3-Large
(MODEL_ENCODER_DIM [24, 40, 112, 960]) and R50-AOTL with ResNeSt-50, on the synthetic 480p clip (481x849 network input,
480x854 output, 10 objects, long-term gap 5) with seeded random weights.

The timed span is the evaluator's per frame (evaluator.py:302-305,332-339,355-361,418-422): match_propogate_one_frame, decode
to the output size, softmax / argmax, nearest resize and update_memory, after the reference frame; 5 warm-up frames, then 20
frames between two CUDA events.  A separate probe pass with eager launches (no CUDA graphs) under torch.profiler reports the
summed device time of the squeeze-excite kernels (gate and gate * x) per frame.

    python scripts/encoder_variants_fps.py OUT_DIR [--warmup 5] [--steps 20]
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

H_IN, W_IN, H_OUT, W_OUT, OBJS = 481, 849, 480, 854, 10
# name: (model config, MODEL_ENCODER, MODEL_ENCODER_DIM or None for the config's own)
VARIANTS = {
    "R50-AOTL": ("r50_aotl", "resnet50", None),
    "AOTL+MobileNetV3": ("aotl", "mobilenetv3", [24, 40, 112, 960]),
    "R50-AOTL+ResNeSt-50": ("r50_aotl", "resnest50", None),
}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = r.stdout.strip().partition(",")
    return name.strip() or torch.cuda.get_device_name(0), power.strip() or "unknown"


def build(variant, dev):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    model_name, enc, dims = VARIANTS[variant]
    cfg = EngineConfig("fps", model_name)
    cfg.MODEL_ENCODER = enc
    if dims is not None:
        cfg.MODEL_ENCODER_DIM = list(dims)
    torch.manual_seed(0)
    model = build_vos_model(cfg.MODEL_VOS, cfg).to(dev).eval()
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=dev.index,
                       long_term_mem_gap=cfg.TEST_LONG_TERM_MEM_GAP, short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP)
    return eng.eval()


def step(eng, img):
    eng.match_propogate_one_frame(img)
    logit = eng.decode_current_logits((H_OUT, W_OUT))
    label = torch.argmax(torch.softmax(logit, dim=1), dim=1, keepdim=True).float()
    eng.update_memory(F.interpolate(label, size=eng.input_size_2d, mode="nearest"))


def run(eng, frames, mask, warmup, steps):
    eng.restart_engine()
    eng.add_reference_frame(frames[0], mask, obj_nums=[OBJS], frame_step=0)
    for t in range(1, warmup + 1):
        step(eng, frames[t])
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for t in range(warmup + 1, warmup + steps + 1):
        step(eng, frames[t])
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def se_probe(eng, frames, mask, warmup, steps):
    """Summed device time (ms) of the SE gate and gate-scale kernels per frame and their launch count, from a torch.profiler
    trace of an eager pass (no CUDA graphs; the two are splat_attention_kernel<1> and splat_combine_kernel<1>)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    from aot_benchmark_b200 import engine
    graphs = engine.USE_GRAPHS
    engine.USE_GRAPHS = False
    try:
        eng.restart_engine()
        eng.add_reference_frame(frames[0], mask, obj_nums=[OBJS], frame_step=0)
        for t in range(1, warmup + 1):
            step(eng, frames[t])
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for t in range(warmup + 1, warmup + steps + 1):
                step(eng, frames[t])
            torch.cuda.synchronize()
    finally:
        engine.USE_GRAPHS = graphs
    us, n = 0.0, 0
    for e in prof.events():
        if e.device_type == DeviceType.CUDA and ("splat_attention_kernel<1>" in e.name or "splat_combine_kernel<1>" in e.name):
            us += e.time_range.elapsed_us()
            n += 1
    return us / 1000.0 / steps, n // steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encoder_variants_fps.py needs a CUDA device (no CPU path)")
    from oracle.aot_oracle import synthetic_video            # input generator only (shared with the tests and bench.py)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu, power = gpu_info()
    print(f"GPU: {gpu}, power limit {power}")
    frames, mask = synthetic_video(a.warmup + a.steps + 1, H_IN, W_IN, OBJS, seed=1234)
    frames = [f.to(dev) for f in frames]
    mask = mask.to(dev)
    rec = {"gpu": gpu, "power_limit": power, "workload": f"synthetic {H_IN}x{W_IN} -> {H_OUT}x{W_OUT}, {OBJS} objects, "
           f"gap 5, {a.warmup} warm-up + {a.steps} timed frames", "variants": {}}
    with torch.no_grad():
        for name in VARIANTS:
            eng = build(name, dev)
            run(eng, frames, mask, a.warmup, a.steps)                       # first pass: buffers, graph capture
            ms = run(eng, frames, mask, a.warmup, a.steps)
            r = {"ms_per_frame": ms / a.steps, "fps": 1000.0 * a.steps / ms}
            if VARIANTS[name][1] == "mobilenetv3":
                se_ms, n = se_probe(eng, frames, mask, a.warmup, a.steps)
                r.update(se_ms_per_frame=se_ms, se_launches_per_frame=n)
            rec["variants"][name] = r
            print(f"{name}: {r['ms_per_frame']:.3f} ms/frame, {r['fps']:.1f} frames/s"
                  + (f"; SE gate + gate-scale {r['se_ms_per_frame']:.4f} ms/frame over {r['se_launches_per_frame']} launches"
                     if "se_ms_per_frame" in r else ""))
            del eng
            torch.cuda.empty_cache()
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "encoder_variants_fps.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
