"""Shared by the test-time augmentation tests: the fixtures' inputs, the engines, and the label checks."""
import os

import torch
import torch.nn.functional as F

from oracle import aot_oracle as O
from oracle import io_side as IO
from oracle import tta_oracle as TO
from oracle import weights as OW

CASES = ["aott_flip_ms", "r50_aotl_flip_ms3", "deaott_multi14", "swinb_aotl_flip_ms"]
# A label may differ from the reference's only where the top-2 probability margin is inside the error the probabilities are
# held to (1e-3 against the reference probabilities, which the fixtures store in steps of 1/2048: at most 2.5e-4 off).
PROB_TOL = 1e-3


def load(golden_dir, name):
    g = torch.load(os.path.join(golden_dir, f"tta_{name}.pt"))
    sd = OW.build_state_dict(g["model"], seed=g["seed"], flavour="calibrated")
    assert OW.checksum(sd) == g["weights_checksum"], "seeded weights are not reproducible on this machine"
    frames, first, new = TO.tta_clip(g)
    assert TO.frames_sha256(frames) == g["frames_sha256"], "seeded frames are not reproducible on this machine"
    g["ens"] = TO.unpack(g["ens_labels"]).float()
    g["aug"] = TO.unpack(g["aug_labels"]).float()
    g["prob"] = {t: TO.unpack_prob(p) for t, p in g["probs"].items()}
    g["flips"] = [f for _ in g["scales"] for f in (False, True)]
    return g, sd, frames, first, new


def aug_images(g, frames, device="cpu"):
    """Per frame, the augmented images of MultiRestrictSize + MultiToTensor (oracle/io_side.py, pinned to the reference)."""
    ac = O.OracleConfig(g["model"]).MODEL_ALIGN_CORNERS
    return [[IO.preprocess(f, None, g["max_long_edge"], s, ac, 16, fl).unsqueeze(0).to(device)
             for s in g["scales"] for fl in (False, True)] for f in frames]


def model(name, sd, device="cpu"):
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    cfg = EngineConfig("t", name)
    m = build_vos_model(cfg.MODEL_VOS, cfg)
    m.load_state_dict(sd, strict=True)
    return m.to(device).eval()


def own_label(logit_map, size, flip, align, new=None):
    """evaluator.py:333-353 for one augmentation: argmax softmax of its upsampled logits, in the original orientation, with the
    new-object overlay -> (label [1,1,H,W], its probabilities)."""
    lo = logit_map.reshape(1, *logit_map.shape[-3:]).float().cpu()
    up = F.interpolate(lo, size=size, mode="bilinear", align_corners=align)
    if flip:
        up = torch.flip(up, dims=[3])
    p = torch.softmax(up, dim=1)
    lab = torch.argmax(p, dim=1, keepdim=True).float()
    if new is not None:
        keep = (new == 0).float()
        lab = lab * keep + new * (1 - keep)
    return lab, p


def outside_band(label, ref, prob, band=PROB_TOL, new=None):
    """Pixels where label != ref although the top-2 margin of prob [1, NC, H, W] exceeds band (new-object pixels excluded)."""
    mm = label.reshape(ref.shape).cpu() != ref
    if new is not None:
        mm &= new.reshape(ref.shape) == 0
    if not mm.any():
        return 0
    top2 = prob.float().cpu().topk(2, dim=1).values
    margin = (top2[:, 0] - top2[:, 1]).reshape(ref.shape)
    return int((mm & (margin > band)).sum())
