"""Test-time augmentation (flip / multi-scale) on the H100 path.

networks/managers/evaluator.py:265-446 with TEST_FLIP / TEST_MULTISCALE builds one eval engine per augmentation (scale-major,
unflipped before flipped: MultiRestrictSize, dataloaders/video_transforms.py:613-688), runs every frame through all of them
one after another, and merges them in eager PyTorch over full-resolution logit maps.  TTAInferEngine keeps the same engines
(AOTInferEngine / DeAOTInferEngine, one per augmentation, all on one model) and computes the same labels, but

* the augmentations' propagate + decode run concurrently, one per stream (an engine with > 10 objects forks its sub-engines
  again from its own stream);
* the ensemble (upsample, flip, softmax, mean, argmax, new-object overlay) is one kernel launch that reads the low-resolution
  logits, and each augmentation's memory label (argmax, flip back, nearest resize) is one more, run on the augmentation's stream
  just before its memory update;
* there is no torch.cuda.empty_cache() per augmentation (evaluator.py:284-285).

Each engine is fed its own prediction, not the ensemble (evaluator.py:346-353, :400-422): the ensemble only decides the output
and, on a frame with new objects, the object count.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops
from .engine import _ENGINES, fork_join

MAX_AUGS = 8        # aotb_tta_merge_f32 takes up to 8 logit maps


def tta_augmentations(cfg, flip, multi_scale):
    """The augmentations of a TTA engine -> (flip, scales, per-augmentation flip bits), scale-major with the unflipped one
    first (FramePreprocessor's order).  flip / multi_scale default to cfg.TEST_FLIP / cfg.TEST_MULTISCALE.  Refuses
    MODEL_USE_PREV_PROB and more than MAX_AUGS augmentations."""
    if getattr(cfg, "MODEL_USE_PREV_PROB", False):
        raise NotImplementedError(
            "MODEL_USE_PREV_PROB with test-time augmentation has no reference behaviour to follow: "
            "networks/managers/evaluator.py:438 reads current_prob before any assignment (its only assignment, :433, is "
            "commented out), so the reference cannot run it")
    flip = bool(getattr(cfg, "TEST_FLIP", False) if flip is None else flip)
    scales = [float(s) for s in (getattr(cfg, "TEST_MULTISCALE", [1]) if multi_scale is None else multi_scale)]
    flips = [f for _ in scales for f in ((False, True) if flip else (False,))]
    if not 1 <= len(flips) <= MAX_AUGS:
        raise ValueError(f"test-time augmentation runs 1 to {MAX_AUGS} augmentations, got {len(flips)} "
                         f"({len(scales)} scales{' x 2 flips' if flip else ''})")
    return flip, scales, flips


class TTAInferEngine(nn.Module):
    def __init__(self, aot_model, gpu_id=0, long_term_mem_gap=9999, short_term_mem_skip=1, flip=None, multi_scale=None,
                 long_term_mem_max=None, precision=None, long_term_mem_policy=None):
        """flip / multi_scale default to cfg.TEST_FLIP / cfg.TEST_MULTISCALE; the augmentations are, in this order, every scale
        unflipped and (with flip) flipped, the order of FramePreprocessor's outputs.  long_term_mem_max bounds every
        augmentation engine's long-term bank; precision ("fp32" | "fp16", default cfg.TEST_PRECISION, else "fp32") and
        long_term_mem_policy ("fifo" | "usage", default cfg.TEST_LONG_TERM_MEM_POLICY, else "fifo") are every augmentation
        engine's (see AOTEngine for all three)."""
        super().__init__()
        cfg = aot_model.cfg
        self.cfg = cfg
        self.AOT = aot_model
        self.flip, self.multi_scale, self.flips = tta_augmentations(cfg, flip, multi_scale)
        cls = _ENGINES.get((cfg.MODEL_ENGINE, "eval"))
        if cls is None:
            raise NotImplementedError(f"no eval engine '{cfg.MODEL_ENGINE}'")
        self.align_corners = cfg.MODEL_ALIGN_CORNERS
        self.aug_engines = [cls(aot_model, gpu_id=gpu_id, long_term_mem_gap=long_term_mem_gap,
                                short_term_mem_skip=short_term_mem_skip, long_term_mem_max=long_term_mem_max,
                                precision=precision, long_term_mem_policy=long_term_mem_policy)
                            for _ in self.flips]
        for e in self.aug_engines:
            e.eval()
        self._outs = {}
        self._fbs = {}
        self.restart_engine()

    def enable_kv_sharding(self, rank, world, group=None):
        raise NotImplementedError("test-time augmentation is not built for a long-term bank sharded over GPUs")

    def restart_engine(self):
        """Start a new video; the augmentation engines keep their sub-engines, buffers and captured graphs."""
        for e in self.aug_engines:
            e.restart_engine()
        self.frame_step = 0
        self.obj_nums = None
        self.pred_prob = None
        self.aug_logits = None

    # ------------------------------------------------------------------ buffers
    def _feedback_buf(self, i, size):
        key = (i, int(size[0]), int(size[1]))
        b = self._fbs.get(key)
        if b is None:
            b = self._fbs[key] = torch.empty((1, 1) + key[1:], dtype=torch.float32, device=self._device())
        return b

    def _outputs(self, H, W, NC):
        key = (H, W, NC)
        o = self._outs.get(key)
        if o is None:
            dev = self._device()
            o = self._outs[key] = (torch.empty((1, 1, H, W), dtype=torch.float32, device=dev),
                                   torch.empty((1, NC, H, W), dtype=torch.float32, device=dev))
        return o

    def _device(self):
        return next(self.AOT.parameters()).device

    def _check(self, imgs):
        if len(imgs) != len(self.aug_engines):
            raise ValueError(f"expected {len(self.aug_engines)} augmented images (one per scale and flip, in "
                             f"FramePreprocessor's order), got {len(imgs)}")

    @staticmethod
    def _label_map(t, H, W):
        return t.reshape(H, W).float().contiguous()

    # ------------------------------------------------------------------ protocol
    def add_reference_frame(self, imgs, label, obj_nums, frame_step=0):
        """imgs: the augmented images [1, 3, h_e, w_e] of the frame (FramePreprocessor's list); label: the annotation at the
        original size and orientation.  Each engine gets it mirrored if its augmentation is flipped, then nearest-resized to its
        input size (evaluator.py:315-323)."""
        self._check(imgs)
        if isinstance(obj_nums, (list, tuple)):
            obj_nums = obj_nums[0]
        self.obj_nums = int(obj_nums)
        H, W = int(label.shape[-2]), int(label.shape[-1])
        lab = self._label_map(label, H, W)
        for i, (eng, img) in enumerate(zip(self.aug_engines, imgs)):
            fb = self._feedback_buf(i, img.shape[-2:])
            ops.tta_feedback(None, fb, (H, W), self.align_corners, self.flips[i], new_label=lab)
            eng.add_reference_frame(img, fb, obj_nums=[self.obj_nums], frame_step=frame_step)
        self.frame_step = frame_step

    def propagate(self, imgs, output_size, new_label=None, keep_prob=False, forced_labels=None):
        """One frame of the evaluator's TTA loop (evaluator.py:325-422) -> the ensemble label [1, 1, H, W] at output_size, a
        static buffer the next call overwrites.

        new_label: annotation of objects that appear at this frame, at the output size and original orientation (ids where
        new, 0 elsewhere); it overwrites the ensemble and every engine's label, and the frame is added as a reference frame to
        every engine with the new object count.  keep_prob: also keep the mean probabilities [1, NC, H, W] in ``pred_prob``.
        forced_labels: one label map per augmentation at the output size and original orientation, fed to the engines instead
        of their own predictions (teacher forcing)."""
        self._check(imgs)
        H, W = int(output_size[0]), int(output_size[1])
        self.frame_step += 1
        ac, flips = self.align_corners, self.flips

        def infer(i, eng):
            eng.match_propogate_one_frame(imgs[i])
            if len(eng.aot_engines) == 1:
                return eng.decode_current_logits(None)          # masked low-resolution logits: the merge upsamples them
            return eng.decode_current_logits((H, W))            # > 10 objects: the aggregated logits at the output size

        maps = fork_join(self, self.aug_engines, infer)
        label, prob = self._outputs(H, W, int(maps[0].shape[1]))
        new = None if new_label is None else self._label_map(new_label.to(label.device), H, W)
        ops.tta_merge(maps, flips, label, ac, new_label=new, prob=prob if keep_prob else None)
        self.pred_prob = prob if keep_prob else None
        self.aug_logits = maps
        forced = None if forced_labels is None else [self._label_map(t.to(label.device), H, W) for t in forced_labels]
        fbs = [self._feedback_buf(i, e.input_size_2d) for i, e in enumerate(self.aug_engines)]

        def feedback(i, overlay):
            if forced is not None:
                ops.tta_feedback(None, fbs[i], (H, W), ac, flips[i], new_label=forced[i])
            else:
                ops.tta_feedback(maps[i], fbs[i], (H, W), ac, flips[i], new_label=overlay)
            return fbs[i]

        if new is None:
            fork_join(self, self.aug_engines, lambda i, eng: eng.update_memory(feedback(i, None)))
            return label
        # new objects (evaluator.py:363-399): the object count is the ensemble's largest id, then every engine takes the frame
        # as a reference frame with its own overlaid label
        self.obj_nums = int(label.max().item())
        for i, eng in enumerate(self.aug_engines):
            fb = feedback(i, new)
            eng.add_reference_frame(imgs[i], fb, obj_nums=[self.obj_nums], frame_step=self.frame_step)
            eng.decode_current_logits((H, W))
            eng.update_memory(fb)
        return label
