#!/usr/bin/env python
"""Frame time of the bounded long-term bank with the FIFO and the usage eviction policy (long_term_mem_policy).

Workload: bench.py's synthetic 480p clip (481x849 network input, 480x854 output, 10 objects, seeded random weights) on
R50-AOTL and R50-DeAOTL, long-term gap 5, --frames propagated frames cycling over 120 distinct synthetic frames, with the bank
bounded to M = 8 and M = 32 memory frames.  Both policies run the same clip; usage mode differs in the long-term attention (one
KV split per memory slot, and the merge that also counts each slot's attention mass) and in one selection launch per store.

Per frame the timed span is match_propogate_one_frame + decode_current_logits + the fused upsample / argmax kernel + the
nearest resize + update_memory, between two CUDA events on the stream.  Per model and M, both policies first run the whole
clip once untimed, then they are alternated for --reps timed passes each.  Reported per arm: ms / frame over the last 50
frames (the bank is full from frame 5 (M - 1) + 1 on), mean and min / max over the passes; the bytes of split-KV partials the
usage-mode attention writes and its merge reads per layer and frame (M x N x d_v fp32, computed from the shapes); and the card's
name and power limit.

    python scripts/usage_bank_fps.py OUT_DIR [--frames 300] [--reps 3]
"""
import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))

from bounded_bank_fps import DISTINCT, GAP, H_IN, OBJS, W_IN, gpu_info, run_clip  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--models", default="r50_aotl,r50_deaotl")
    ap.add_argument("--bounds", default="8,32")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("usage_bank_fps.py needs a CUDA device (no CPU path)")
    bounds = [int(m) for m in a.bounds.split(",")]
    if a.frames < GAP * (max(bounds) - 1) + 51:
        raise SystemExit(f"--frames must leave 50 frames after the bank fills (at least {GAP * (max(bounds) - 1) + 51})")
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    from aot_benchmark_b200.plan import get_plan
    from oracle.aot_oracle import synthetic_video            # input generator only (shared with the tests and bench.py)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu, power = gpu_info()
    print(f"GPU: {gpu}, power limit {power}", flush=True)
    frames, mask = synthetic_video(DISTINCT, H_IN, W_IN, OBJS, seed=1234)
    frames, mask = [f.to(dev) for f in frames], mask.to(dev)
    rec = {"gpu": gpu, "power_limit": power,
           "workload": f"synthetic {H_IN}x{W_IN}, {OBJS} objects, gap {GAP}, {a.frames} propagated frames cycling over "
                       f"{DISTINCT}, one untimed pass then {a.reps} alternated timed passes per policy; ms / frame over the "
                       f"last 50 frames", "arms": {}}
    for model_name in a.models.split(","):
        cfg = EngineConfig("fps", model_name)
        torch.manual_seed(0)
        model = build_vos_model(cfg.MODEL_VOS, cfg).to(dev).eval()
        get_plan(model)
        for M in bounds:
            engines = {}
            with torch.no_grad():
                for policy in ("fifo", "usage"):
                    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=GAP,
                                       short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP, long_term_mem_max=M,
                                       long_term_mem_policy=policy).eval()
                    run_clip(eng, frames, mask, a.frames)
                    engines[policy] = eng
                passes = {p: [] for p in engines}
                for _ in range(a.reps):
                    for policy, eng in engines.items():
                        ms, _ = run_clip(eng, frames, mask, a.frames)
                        passes[policy].append(sum(ms[-50:]) / 50)
            e0 = engines["usage"].aot_engines[0]
            dv = e0._vdim if e0._gp_tc else e0._plan().C
            opart_mb = M * e0.enc_hw * dv * 4 / 1e6
            for policy, v in passes.items():
                key = f"{model_name} M={M} {policy}"
                rec["arms"][key] = {"ms_per_frame_last50": {"mean": sum(v) / len(v), "min": min(v), "max": max(v)},
                                    "passes": v}
                if policy == "usage":
                    rec["arms"][key]["opart_mb_per_layer"] = opart_mb
                print(f"{key}: {sum(v) / len(v):.3f} ms/frame ({min(v):.3f}-{max(v):.3f})"
                      + (f"; partials {opart_mb:.1f} MB per layer written and read" if policy == "usage" else ""), flush=True)
            del engines
            torch.cuda.empty_cache()
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "usage_bank_fps.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
