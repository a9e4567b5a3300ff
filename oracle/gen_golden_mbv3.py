"""Generate the MobileNetV3 / ResNeSt-50 golden fixtures under tests/golden/ by running the REAL reference, and the state_dict /
config contract of the two cases (tests/golden/reference_contract_mbv3_rs50.json).

TEST INFRASTRUCTURE ONLY; the sibling of oracle/gen_golden_resnest.py for the two encoders that oracle/mobilenetv3_oracle.py
restates.  Run where the reference checkout exists (argument-free, $AOT_REFERENCE or /root/reference):

    python oracle/gen_golden_mbv3.py [--out tests/golden] [--only NAME | contract | full]

Same procedure as gen_golden_resnest.py: seeded weights (mobilenetv3_oracle.build_state_dict) loaded with strict=True into the
reference's own model, built from its model config with MODEL_ENCODER / MODEL_ENCODER_DIM set as a user sets them, the
reference's own eval engine driven through the evaluator's per-frame protocol on seeded synthetic clips, the outputs stored, and
the oracle's distance from them printed (the pin).  Only the V3 -> V2 patch of gen_golden.py is applied.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import zlib

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("AOT_REFERENCE", "/root/reference")
sys.path.insert(0, REPO)
sys.path.insert(0, REF)

from oracle import aot_oracle as O  # noqa: E402
from oracle import mobilenetv3_oracle as MO  # noqa: E402
from oracle import weights as OW  # noqa: E402
from oracle.gen_contract import norm, state_dict_digest  # noqa: E402

import networks.layers.attention as RA  # noqa: E402  (reference)
import networks.layers.transformer as RT  # noqa: E402

RT.MultiheadLocalAttentionV3 = RA.MultiheadLocalAttentionV2  # SURVEY 0.4

from configs.default import DefaultEngineConfig  # noqa: E402
from networks.engines import build_engine as ref_build_engine  # noqa: E402
from networks.models import build_vos_model as ref_build_model  # noqa: E402

MBV3, RS50 = "AOTL with mobilenetv3", "R50-AOTL with resnest50"
# name: (case, H, W, out_h, out_w, frames, objs, gap, flavour)
VIDEO_CASES = {
    "aotl_mbv3_small": (MBV3, 161, 241, 150, 230, 7, 10, 2, "calibrated"),
    "rs50_aotl_small": (RS50, 161, 241, 150, 230, 7, 10, 2, "calibrated"),
}
# 481x849 -> 480x854, 10 objects, gap 5: zlib-packed labels of every frame, and the low-res logits of frames 1 and 6 at every
# second row and column
FULL_CASES = {"aotl_mbv3_480p": (MBV3, 481, 849, 480, 854, 8, 10, 5, "calibrated", (1, 6))}
LOGIT_STRIDE = 2


def reference_config(case, exp="golden"):
    model, enc, dims = MO.CASES[case]
    rc = DefaultEngineConfig(exp, model)
    rc.MODEL_ENCODER = enc
    rc.MODEL_ENCODER_DIM = list(dims)
    return rc


def run_reference_video(case, H, W, oh, ow, T, objs, gap, flavour, seed=0):
    torch.manual_seed(0)
    sd = MO.build_state_dict(case, seed=seed, flavour=flavour)
    rcfg = reference_config(case)
    ref_model = ref_build_model(rcfg.MODEL_VOS, rcfg).eval()
    ref_model.load_state_dict(sd, strict=True)
    engine = ref_build_engine(rcfg.MODEL_ENGINE, phase="eval", aot_model=ref_model, gpu_id=-1, long_term_mem_gap=gap,
                              short_term_mem_skip=1)
    engine.eval()
    frames, mask = O.synthetic_video(T, H, W, objs, seed=1234 + seed)
    with torch.no_grad():
        logits_lo, labels = O.run_video(engine, frames, mask, objs, (oh, ow))
    oe = MO.OracleEngine(sd, MO.OracleConfig(case), long_term_mem_gap=gap)
    with torch.no_grad():
        o_lo, o_labels = O.run_video(oe, frames, mask, objs, (oh, ow), forced_masks=labels)
    max_d = max((a - b).abs().max().item() for a, b in zip(logits_lo, o_lo))
    mism = sum((a != b).sum().item() for a, b in zip(labels, o_labels))
    return sd, logits_lo, labels, max_d, mism


def video_case(name, out_dir):
    case, H, W, oh, ow, T, objs, gap, flavour = VIDEO_CASES[name]
    sd, ref_lo, ref_labels, max_d, mism = run_reference_video(case, H, W, oh, ow, T, objs, gap, flavour)
    print(f"[{name}] oracle vs reference: max|dlogit|={max_d:.3e} label mismatches={mism}")
    torch.save({
        "model": case, "H": H, "W": W, "out_size": (oh, ow), "frames": T, "objs": objs, "gap": gap,
        "flavour": flavour, "seed": 0, "skip": 1, "weights_checksum": OW.checksum(sd),
        "ref_logits_lo": [t.to(torch.float32) for t in ref_lo],
        "ref_labels": [t.to(torch.uint8) for t in ref_labels],
        "oracle_pin_max_dlogit": max_d, "oracle_pin_label_mismatch": mism,
    }, os.path.join(out_dir, f"video_{name}.pt"))


def full_case(name, out_dir):
    case, H, W, oh, ow, T, objs, gap, flavour, keep = FULL_CASES[name]
    t0 = time.time()
    sd, ref_lo, ref_labels, max_d, mism = run_reference_video(case, H, W, oh, ow, T, objs, gap, flavour)
    print(f"[{name}] reference + oracle in {time.time() - t0:.1f} s; oracle vs reference: max|dlogit|={max_d:.3e} "
          f"label mismatches={mism}")
    lab = torch.stack([t.to(torch.uint8).reshape(oh, ow) for t in ref_labels]).contiguous()
    s = LOGIT_STRIDE
    torch.save({
        "model": case, "H": H, "W": W, "out_size": (oh, ow), "frames": T, "objs": objs, "gap": gap,
        "flavour": flavour, "seed": 0, "weights_checksum": OW.checksum(sd), "logit_frames": list(keep), "logit_stride": s,
        "ref_logits_lo": {int(t): ref_lo[t - 1][:, :, ::s, ::s].to(torch.float32).clone() for t in keep},
        "ref_labels_zlib": zlib.compress(lab.numpy().tobytes(), 9), "ref_labels_shape": tuple(lab.shape),
        "oracle_pin_max_dlogit": max_d, "oracle_pin_label_mismatch": mism,
    }, os.path.join(out_dir, f"full_{name}.pt"))


def contract(out_dir):
    """The state_dict digest / key count and config values of the two cases, as oracle/gen_contract.py writes them."""
    out = {"models": {}}
    for case in MO.CASES:
        rc = reference_config(case, "x")
        sd = ref_build_model(rc.MODEL_VOS, rc).state_dict()
        out["models"][case] = {"state_dict_sha256": state_dict_digest(sd), "state_dict_keys": len(sd),
                               "config": {k: norm(v) for k, v in rc.__dict__.items() if k not in ("EXP_NAME", "MODEL_NAME")}}
    with open(os.path.join(out_dir, "reference_contract_mbv3_rs50.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(REPO, "tests", "golden"))
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    if a.only in (None, "contract"):
        contract(a.out)
    for name in VIDEO_CASES:
        if a.only in (None, name):
            video_case(name, a.out)
    for name in FULL_CASES:
        if a.only in (None, "full", name):
            full_case(name, a.out)


if __name__ == "__main__":
    main()
