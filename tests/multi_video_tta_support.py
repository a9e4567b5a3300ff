"""TEST INFRASTRUCTURE ONLY: torch restatements of the two batched TTA entry points (include/aotb200.h:
aotb_tta_merge_batched_f32, aotb_tta_feedback_batched_f32), and the CPU install for MultiVideoTTAInferEngine.

Their contract is that each video (merge) or lane (feedback) equals aotb_logits_postproc_f32 on its lanes followed by the
one-video TTA entry point, so each restatement masks the lane's NHWC logits as logits_postproc does and runs the one-video
emulation of tests/test_cpu_tta_host.py.  Nothing under aot_benchmark_b200/ imports this module."""
import torch

import emu_multi_video_deaot
import test_cpu_tta_host as TH


def lowres(lg, lane, obj):
    """logits_postproc's low-resolution map of one lane: [lanes, h, w, NC] -> [1, NC, h, w], ids above obj at -1e10."""
    lo = lg[lane].permute(2, 0, 1).contiguous().clone()
    lo[obj + 1:] = -1e10
    return lo.unsqueeze(0)


def tta_merge_batched(logits, flips, lanes, obj_nums, label, align_corners, new_labels=None, prob=None, stream=None):
    n = len(lanes)
    H, W = label.shape[-2:]
    lab = label.reshape(n, H, W)
    pr = None if prob is None else prob.reshape(n, -1, H, W)
    for b in range(n):
        maps = [lowres(lg, lanes[b][e], obj_nums[b]) for e, lg in enumerate(logits)]
        TH.emu_tta_merge(maps, flips, lab[b], align_corners, new_label=None if new_labels is None else new_labels[b],
                         prob=None if pr is None else pr[b])
    return label


def tta_feedback_batched(logits, out, obj_nums, flips, output_size, align_corners, new_labels=None, stream=None):
    for k in range(len(flips)):
        lo = None if logits is None else lowres(logits, k, obj_nums[k])
        TH.emu_tta_feedback(lo, out[k], output_size, align_corners, flips[k],
                            new_label=None if new_labels is None else new_labels[k])
    return out


EMULATED = ("tta_merge_batched", "tta_feedback_batched")


def install_engine(monkeypatch):
    """The AOT and DeAOT multi-video emulations, the one-video TTA emulations and the two batched TTA restatements."""
    from aot_benchmark_b200 import ops
    emu_multi_video_deaot.install_engine(monkeypatch)
    monkeypatch.setattr(ops, "tta_merge", TH.emu_tta_merge)
    monkeypatch.setattr(ops, "tta_feedback", TH.emu_tta_feedback)
    for name in EMULATED:
        monkeypatch.setattr(ops, name, globals()[name])


def lane_lowres(eng, vid, e):
    """Augmentation e's masked low-resolution logits of video vid [1, NC, h, w] after eng.propagate."""
    lg = eng.aug_logits[vid][e]
    return lowres(lg, 0, eng._video(vid)["obj"])
