"""TEST INFRASTRUCTURE ONLY: CPU emulations of the three entry points behind the multi-video engines' ID-bank lanes
(include/aotb200.h: aotb_lane_gather_f32, aotb_separate_labels_batched_f32, aotb_soft_logit_aggregation_batched_f32).  Each
contract is stated in terms of the one-video entry points, so each emulation is built from their emulations (tests/emu_ops.py):
a copy per lane, separate_labels per entry, and logits_postproc per lane followed by soft_logit_aggregation per video.  Nothing
under aot_benchmark_b200/ imports this module."""
import torch

import emu_multi_video
import emu_multi_video_deaot
import emu_ops


def lane_gather(src, dst, lane_video, n_lanes, stream=None):
    for s, d in zip(src, dst):
        for l in range(n_lanes):
            v = int(lane_video[l])
            if 0 <= v < s.shape[0]:
                d[l].copy_(s[v])
    return dst


def separate_labels_batched(labels, parts, out, max_obj=10, stream=None):
    for m, p, o in zip(labels, parts, out):
        rows = torch.empty((int(p) + 1, m.numel()), dtype=torch.float32, device=m.device)
        emu_ops.separate_labels(m.reshape(-1), rows, max_obj)
        o.copy_(rows[int(p)].view(o.shape))
    return out


def soft_logit_aggregation_batched(logits, lanes, obj_nums, align_corners, out=None, labels=None, max_obj=10, stream=None):
    _, h, w, NC = logits.shape
    for b, (ls, objs) in enumerate(zip(lanes, obj_nums)):
        o = None if out is None else out[b]
        lab = None if labels is None else labels[b]
        size = tuple((o if o is not None else lab).shape[-2:])
        maps = []
        for l, obj in zip(ls, objs):
            lo = torch.empty((1, NC, h, w), dtype=torch.float32, device=logits.device)
            up = None if size == (h, w) else torch.empty((1, NC) + size, dtype=torch.float32, device=logits.device)
            emu_ops.logits_postproc(logits[l:l + 1], lo, up, obj, align_corners)
            maps.append(lo if up is None else up)
        agg = torch.empty((1, 1 + len(ls) * max_obj) + size, dtype=torch.float32, device=logits.device)
        emu_ops.soft_logit_aggregation(maps, agg, max_obj)
        if o is not None:
            o.copy_(agg.view(o.shape))
        if lab is not None:
            lab.copy_(agg.argmax(1).to(lab.dtype).view(lab.shape))
    return out, labels


EMULATED = ("lane_gather", "separate_labels_batched", "soft_logit_aggregation_batched")


def install_engine(monkeypatch, deaot=False):
    """The AOT (or, deaot=True, the DeAOT) multi-video emulations and the three lane entry points."""
    from aot_benchmark_b200 import ops
    (emu_multi_video_deaot if deaot else emu_multi_video).install_engine(monkeypatch)
    for name in EMULATED:
        monkeypatch.setattr(ops, name, globals()[name])
