"""CPU oracle for test-time augmentation (flip / multi-scale): the evaluator's TTA loop over any engines that expose the
reference protocol, and seeded uint8 clips for the TTA fixtures.

TEST INFRASTRUCTURE ONLY, like oracle/aot_oracle.py: tests/, oracle/gen_golden_tta.py and scripts/ may import it; the product
path never does.  oracle/gen_golden_tta.py pins run_video_tta over the oracle engines against the real reference's evaluator
loop and stores the reference's outputs under tests/golden/tta_*.pt.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle import aot_oracle as O

Tensor = torch.Tensor


def run_video_tta(engines, aug_frames: Sequence[Sequence[Tensor]], flips: Sequence[bool], first_label: Tensor, obj_num: int,
                  output_size: Tuple[int, int], new_objects: Optional[Dict[int, Tensor]] = None,
                  forced_labels: Optional[Sequence[Sequence[Tensor]]] = None, prob_frames: Sequence[int] = ()):
    """Evaluator.evaluating with test-time augmentation (evaluator.py:265-446): one engine per augmentation, aug_frames[t][e]
    = augmentation e's image of frame t (MultiRestrictSize's order), flips[e] its flip bit, first_label / new_objects[t] at
    the output size and original orientation.  Every engine is fed its own prediction (:346-353, :400-422), mirrored back for
    a flipped augmentation, then nearest-resized; new objects overwrite the ensemble and every engine's label and the frame
    becomes a reference frame of every engine with the ensemble's largest id as the object count (:363-399).
    forced_labels[t - 1][e] replaces engine e's label of frame t (teacher forcing; the overlay is the caller's).
    Returns (ensemble labels, per-frame lists of per-augmentation labels at the output size and original orientation,
    {t: mean probabilities} for t in prob_frames)."""
    new_objects = new_objects or {}
    flip = lambda x: torch.flip(x, dims=[3])                                             # utils/image.py:108-112, dim 3
    for eng, img, f in zip(engines, aug_frames[0], flips):
        eng.restart_engine()
        lab = flip(first_label) if f else first_label                                   # video_transforms.py:686 (labels)
        eng.add_reference_frame(img, F.interpolate(lab, size=tuple(img.shape[2:]), mode="nearest"), frame_step=0,
                                obj_nums=[obj_num])
    ens, per_aug, probs = [], [], {}
    for t in range(1, len(aug_frames)):
        all_preds = []
        for eng, img, f in zip(engines, aug_frames[t], flips):
            eng.match_propogate_one_frame(img)
            logit = eng.decode_current_logits(output_size)
            all_preds.append(torch.softmax(flip(logit) if f else logit, dim=1))
        labels = [torch.argmax(p, dim=1, keepdim=True).to(p.dtype) for p in all_preds]
        pred_prob = torch.mean(torch.cat(all_preds, dim=0), dim=0, keepdim=True)
        pred_label = torch.argmax(pred_prob, dim=1, keepdim=True).to(pred_prob.dtype)
        new = new_objects.get(t)
        if new is not None:
            new = new.to(pred_label.device, pred_label.dtype)
            keep = (new == 0).to(pred_label.dtype)
            labels = [l * keep + new * (1 - keep) for l in labels]
            pred_label = pred_label * keep + new * (1 - keep)
            obj_num = int(pred_label.max().item())
        if forced_labels is not None:
            labels = [l.to(pred_label.device, pred_label.dtype) for l in forced_labels[t - 1]]
        ens.append(pred_label.detach().clone())
        per_aug.append([l.detach().clone() for l in labels])
        if t in prob_frames:
            probs[t] = pred_prob.detach().clone()
        for eng, img, f, lab in zip(engines, aug_frames[t], flips, labels):
            fb = F.interpolate(flip(lab) if f else lab, size=tuple(eng.input_size_2d), mode="nearest")
            if new is not None:
                eng.add_reference_frame(img, fb, obj_nums=[obj_num], frame_step=t)
                eng.decode_current_logits(output_size)
            eng.update_memory(fb)
    return ens, per_aug, probs


def synthetic_frames_u8(num_frames: int, h: int, w: int, seed: int):
    """Seeded uint8 frames [h, w, 3] (numpy, the dtype cv2.imread returns) from synthetic_video's low-pass noise."""
    import numpy as np
    frames, _ = O.synthetic_video(num_frames, h, w, 0, seed=seed)
    return [np.ascontiguousarray((f[0].permute(1, 2, 0) * 60 + 128).round().clamp(0, 255).to(torch.uint8).numpy())
            for f in frames]


def tta_clip(g):
    """The inputs of a tests/golden/tta_*.pt case from its metadata: (uint8 frames, first label [1,1,H,W] with ids
    1..first_objs, {event_frame: label [1,1,H,W] of ids first_objs+1..objs} or {})."""
    H, W = g["H"], g["W"]
    frames = synthetic_frames_u8(g["frames"], H, W, seed=g["video_seed"])
    _, full = O.synthetic_video(1, H, W, g["objs"], seed=g["video_seed"] + 1)
    first = torch.where(full <= g["first_objs"], full, torch.zeros_like(full))
    new = {} if g["event_frame"] is None else {g["event_frame"]: torch.where(full > g["first_objs"], full, torch.zeros_like(full))}
    return frames, first, new


PROB_SCALE = 2048      # fixture probabilities are stored as round(p * PROB_SCALE): rounding error <= 2.5e-4


def pack(t: Tensor):
    """A fixture tensor zlib-compressed into a uint8 tensor (label maps and quantised probabilities compress several-fold;
    a uint8 tensor is saved as raw storage, where a pickled bytes object would grow by up to half)."""
    import zlib
    import numpy as np
    t = t.contiguous()
    z = zlib.compress(t.numpy().tobytes(), 9)
    return {"zlib": torch.from_numpy(np.frombuffer(z, dtype=np.uint8).copy()), "shape": tuple(t.shape),
            "dtype": str(t.dtype).split(".")[-1]}


def unpack(p) -> Tensor:
    import zlib
    import numpy as np
    raw = zlib.decompress(p["zlib"].numpy().tobytes())
    return torch.from_numpy(np.frombuffer(raw, dtype=p["dtype"]).copy()).reshape(p["shape"])


def pack_prob(p: Tensor):
    return pack((p.double() * PROB_SCALE).round().to(torch.int16))


def unpack_prob(p) -> Tensor:
    return unpack(p).float() / PROB_SCALE


def frames_sha256(frames) -> str:
    import hashlib
    hsh = hashlib.sha256()
    for f in frames:
        hsh.update(f.tobytes())
    return hsh.hexdigest()
