#!/usr/bin/env python
"""What batching the image encoder buys on a stored clip (AOTEngine.offline_encoder).

1. Encoder sweep: ms per frame of the image encoder + projection (one captured graph per chunk size B, replayed) at
   B in {1, 2, 4, 8, 16} for R50-AOTL, AOTT and RS101-AOTL at the bench input 481x849 and SwinB-AOTL at 592x1040, in fp32
   and fp16.  B = 1 is the per-frame path's encoder.  Each point: two untimed calls (eager, capture), then replays timed with
   CUDA events over about 64 frames.
2. Clip: a 99-frame R50-AOTL clip at 481x849 with 10 objects (10 distinct seeded synthetic frames, cycled; long-term gap 5),
   run end to end on the per-frame path (add_reference_frame with the frame, then propagate, decode at the input size,
   argmax and memory update with the engine's own label) and on the offline path (offline_encoder over the clip, then the
   same loop without images), alternated for --reps timed passes after one untimed pass of each.  ms / frame = the whole
   clip (the offline path's offline_encoder call included) over 99 frames, CUDA events from the first call to the last
   memory update.  Also: the copy of one stored frame into the per-frame feature buffers, and the largest logit difference
   and differing label pixels between the paths on the last pass.
The card's name, power limit and max SM clock are read in the same run.

    python scripts/offline_encoder_fps.py OUT_DIR [--reps 3] [--skip-sweep]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

CHUNKS = [1, 2, 4, 8, 16]
SWEEP = [("r50_aotl", 481, 849), ("aott", 481, 849), ("rs101_aotl", 481, 849), ("swinb_aotl", 592, 1040)]
CLIP_T, OBJS, DISTINCT, H, W = 99, 10, 10, 481, 849


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return [s.strip() for s in r.stdout.strip().split(",")] if r.stdout.strip() else [torch.cuda.get_device_name(0), "?", "?"]


def model_of(name):
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    from oracle import resnest_oracle as RO
    from oracle import weights as OW
    cfg = EngineConfig("fps", name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict((RO if name in RO.MODELS else OW).build_state_dict(name, seed=0))
    return model.cuda().eval()


def sweep():
    from aot_benchmark_b200 import engine, ops, plan
    rows = []
    st = torch.cuda.current_stream().cuda_stream
    for name, h, w in SWEEP:
        model = model_of(name)
        P = plan.get_plan(model)
        for prec in ("fp32", "fp16"):
            enc = engine._Encoder(P, h, w)
            for B in CHUNKS:
                img = torch.randn(B, 3, h, w, generator=torch.Generator().manual_seed(B)).cuda()
                reps = max(4, 64 // B)
                with torch.no_grad(), ops.precision(prec):
                    enc(img, st)
                    enc(img, st)
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        enc(img, st)
                    e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / (reps * B)
                rows.append({"model": name, "H": h, "W": w, "precision": prec, "B": B, "ms_per_frame": round(ms, 4)})
                print(json.dumps(rows[-1]), flush=True)
            del enc
            torch.cuda.empty_cache()
        del model, P
        torch.cuda.empty_cache()
    return rows


def clip_pass(eng, frames, clip, mask, offline):
    """-> (ms / frame over the whole clip, [(logits, label)] of the last frame)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    eng.restart_engine()
    if offline:
        eng.offline_encoder(clip)
        eng.add_reference_frame(mask=mask, obj_nums=[OBJS], frame_step=0)
    else:
        eng.add_reference_frame(frames[0], mask, obj_nums=[OBJS], frame_step=0)
    for t in range(1, CLIP_T):
        if offline:
            eng.match_propogate_one_frame()
        else:
            eng.match_propogate_one_frame(clip[t:t + 1])
        lg = eng.decode_current_logits((H, W))
        label = lg.argmax(1, keepdim=True).float()
        eng.update_memory(label)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / CLIP_T, (lg[:, :OBJS + 1].clone(), label.clone())


def clip_bench(reps):
    from aot_benchmark_b200 import build_engine, engine
    from oracle import aot_oracle as O
    model = model_of("r50_aotl")
    frames, mask = O.synthetic_video(DISTINCT, H, W, OBJS, seed=3)
    frames = [f.cuda() for f in frames]
    clip = torch.cat([frames[0]] + [frames[1 + (t - 1) % (DISTINCT - 1)] for t in range(1, CLIP_T)]).contiguous()
    mask = mask.cuda()
    eng = build_engine("aotengine", phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=5)
    eng.eval()
    res = {"per_frame": [], "offline": []}
    with torch.no_grad():
        clip_pass(eng, frames, clip, mask, False)
        clip_pass(eng, frames, clip, mask, True)
        last = {}
        for _ in range(reps):
            for mode, off in (("per_frame", False), ("offline", True)):
                ms, last[mode] = clip_pass(eng, frames, clip, mask, off)
                res[mode].append(round(ms, 4))
        # the per-frame copy of a stored frame (eager, four device copies)
        e0 = eng.aot_engines[0]
        st = torch.cuda.current_stream().cuda_stream
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ev0.record()
        for t in range(CLIP_T):
            e0._offline_embs(t, st)
        ev1.record()
        torch.cuda.synchronize()
        copy_us = ev0.elapsed_time(ev1) * 1000 / CLIP_T
    (la, ba), (lb, bb) = last["per_frame"], last["offline"]
    out = {"clip": f"r50_aotl {H}x{W} {OBJS} objects, {CLIP_T} frames, gap 5", "chunk": engine.OFFLINE_ENC_CHUNK,
           "ms_per_frame": {k: {"mean": round(sum(v) / len(v), 4), "min": min(v), "max": max(v), "all": v}
                            for k, v in res.items()},
           "stored_frame_copy_us": round(copy_us, 2),
           "last_frame_max_dlogit": (la - lb).abs().max().item(), "last_frame_label_diff_px": int((ba != bb).sum().item())}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-sweep", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this script measures the H100 path: it needs a CUDA device"
    os.makedirs(args.out_dir, exist_ok=True)
    name, power, clock = gpu_info()
    print(f"gpu: {name}, power limit {power}, max SM clock {clock}", flush=True)
    result = {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    if not args.skip_sweep:
        result["encoder_sweep"] = sweep()
    result["clip"] = clip_bench(args.reps)
    with open(os.path.join(args.out_dir, "offline_encoder_fps.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
