"""Generate the test-time augmentation fixtures tests/golden/tta_*.pt by running the REAL reference.

TEST INFRASTRUCTURE ONLY.  Run where the reference checkout exists (it is not on the GPU machines):

    python oracle/gen_golden_tta.py [--out tests/golden] [--only NAME]

For every case it loads a seeded weight set into the reference's own model, turns seeded uint8 frames into the augmented
images with the reference's own MultiRestrictSize + MultiToTensor (dataloaders/video_transforms.py:594-715), drives one
reference eval engine per augmentation through the evaluator's TTA loop (networks/managers/evaluator.py:265-446, restated by
oracle/tta_oracle.run_video_tta) and stores the ensemble labels of every frame, every augmentation's own label of every frame
(the label its engine is fed, at the output size and original orientation) and the mean probabilities of a few frames.  It
prints how far the oracle engines (teacher-forced with the reference's per-augmentation labels) and oracle/io_side.preprocess
are from the reference: the pins.  The reference is patched only as oracle/gen_golden.py documents.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import gen_golden as G  # noqa: E402  (puts the reference on sys.path and applies its one patch)
from oracle import aot_oracle as O  # noqa: E402
from oracle import io_side as IO  # noqa: E402
from oracle import tta_oracle as TO  # noqa: E402
from oracle import weights as OW  # noqa: E402

import dataloaders.video_transforms as tr  # noqa: E402  (reference)

MAX_LONG_EDGE = 800 * 1.3       # configs/default.py:99-100
# name: (model, H, W, scales, objects at frame 0, objects in all (more appear at event_frame), frames, gap, event_frame,
#        frames whose mean probabilities are stored)
CASES = {
    "aott_flip_ms": ("aott", 97, 129, [1.0, 1.3], 3, 3, 6, 2, None, (1, 5)),
    # 6 augmentations, one a downscale (113x177, 161x241, 193x305)
    "r50_aotl_flip_ms3": ("r50_aotl", 161, 241, [0.75, 1.0, 1.25], 10, 10, 4, 2, None, (1, 3)),
    # 8 objects at frame 0, ids 9..14 annotated at frame 2: two sub-engines per augmentation from frame 2, overlay under flip
    "deaott_multi14": ("deaott", 97, 129, [1.0, 1.3], 8, 14, 5, 2, 2, (2, 4)),
    # align_corners = False: multiples of 16 (144x208, 192x272) and the half-pixel bilinear form
    "swinb_aotl_flip_ms": ("swinb_aotl", 144, 208, [1.0, 1.3], 6, 6, 4, 2, None, (1, 3)),
}
VIDEO_SEED = 2024


def case_inputs(name):
    """-> (uint8 frames, first label [1,1,H,W], {event frame: new label} or {}, align_corners): what the tests regenerate."""
    model, H, W, scales, first_objs, objs, T, gap, event, _ = CASES[name]
    frames, first, new = TO.tta_clip({"H": H, "W": W, "frames": T, "video_seed": VIDEO_SEED, "objs": objs,
                                      "first_objs": first_objs, "event_frame": event})
    return frames, first, new, O.OracleConfig(model).MODEL_ALIGN_CORNERS


def ref_augment(frame_u8, scales, align):
    sample = {"current_img": np.array(frame_u8, dtype=np.float32), "meta": {"flip": False}}
    out = tr.MultiToTensor()(tr.MultiRestrictSize(None, MAX_LONG_EDGE, True, scales, align)(sample))
    return [o["current_img"].float().unsqueeze(0).contiguous() for o in out]


def oracle_augment(frame_u8, scales, align):
    return [IO.preprocess(frame_u8, None, MAX_LONG_EDGE, s, align, 16, f).unsqueeze(0) for s in scales for f in (False, True)]


def run_case(name, out_dir):
    model, H, W, scales, first_objs, objs, T, gap, event, prob_frames = CASES[name]
    frames, first, new, align = case_inputs(name)
    flips = [f for _ in scales for f in (False, True)]
    torch.manual_seed(0)
    sd = OW.build_state_dict(model, seed=0, flavour="calibrated")
    rcfg = G.DefaultEngineConfig("golden", model)
    ref_model = G.ref_build_model(rcfg.MODEL_VOS, rcfg).eval()
    ref_model.load_state_dict(sd, strict=True)
    engines = [G.ref_build_engine(rcfg.MODEL_ENGINE, phase="eval", aot_model=ref_model, gpu_id=-1, long_term_mem_gap=gap,
                                  short_term_mem_skip=1).eval() for _ in flips]
    aug = [ref_augment(f, scales, align) for f in frames]
    mine = [oracle_augment(f, scales, align) for f in frames]
    io_pin = max((a - b).abs().max().item() for fa, fb in zip(aug, mine) for a, b in zip(fa, fb))
    with torch.no_grad():
        ens, per_aug, probs = TO.run_video_tta(engines, aug, flips, first, first_objs, (H, W), new_objects=new,
                                               prob_frames=prob_frames)
        oe = [O.OracleInferEngine(sd, O.OracleConfig(model), long_term_mem_gap=gap) for _ in flips]
        o_ens, _, o_probs = TO.run_video_tta(oe, aug, flips, first, first_objs, (H, W), new_objects=new,
                                             forced_labels=per_aug, prob_frames=prob_frames)
    dprob = max((probs[t] - o_probs[t]).abs().max().item() for t in prob_frames)
    mism = sum((a != b).sum().item() for a, b in zip(ens, o_ens))
    subs = [len(e.aot_engines) for e in engines]
    print(f"[tta {name}] augs {[tuple(a.shape[2:]) for a in aug[0]]} sub-engines {subs}: oracle vs reference "
          f"max|dprob|={dprob:.3e} ensemble label mismatches={mism}; io_side vs MultiRestrictSize max|d|={io_pin:.2e}; "
          f"labels used={sorted(set(int(v) for l in ens for v in l.unique().tolist()))}")
    torch.save({
        "model": model, "H": H, "W": W, "scales": scales, "flip": True, "max_long_edge": MAX_LONG_EDGE,
        "first_objs": first_objs, "objs": objs, "frames": T, "gap": gap, "event_frame": event, "seed": 0,
        "video_seed": VIDEO_SEED, "weights_checksum": OW.checksum(sd), "frames_sha256": TO.frames_sha256(frames),
        "aug_sizes": [tuple(a.shape[2:]) for a in aug[0]], "sub_engines": subs,
        "ens_labels": TO.pack(torch.stack([l.reshape(H, W) for l in ens]).to(torch.uint8)),              # [T-1, H, W]
        "aug_labels": TO.pack(torch.stack([torch.stack([l.reshape(H, W) for l in ls]) for ls in per_aug]).to(torch.uint8)),
        # [NC, H, W] in steps of 1 / PROB_SCALE; one sub-engine: the channels up to the object count (the others are exactly 0)
        "prob_frames": list(prob_frames), "prob_scale": TO.PROB_SCALE,
        "probs": {t: TO.pack_prob(probs[t][0, :(first_objs + 1 if subs[0] == 1 else None)]) for t in prob_frames},
        "oracle_pin_max_dprob": dprob, "oracle_pin_label_mismatch": mism, "io_pin": io_pin,
    }, os.path.join(out_dir, f"tta_{name}.pt"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(REPO, "tests", "golden"))
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    for name in CASES:
        if a.only in (None, name):
            run_case(name, a.out)


if __name__ == "__main__":
    main()
