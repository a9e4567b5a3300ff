"""Flip / multi-scale test-time augmentation over several videos: TTAInferEngine's semantics per video, with the multi-video
engine's one batched pass per frame (DESIGN §3.9.2).

One multi-video engine ("pool") per scale, each with max_videos x (2 with flip, else 1) slots.  A (video, flip) pair of a scale
is one video of that scale's pool -- a *lane*: the flipped and unflipped images of a scale have the same network input size,
so they batch together.  Per frame:

1. every pool runs its batched propagate + decoder on its own stream (engine.fork_join), leaving its raw NHWC logits;
2. one aotb_tta_merge_batched_f32 launch reads every lane's logits, masks each at its video's object count, and writes every
   video's ensemble label (and mean probabilities);
3. per pool, one aotb_tta_feedback_batched_f32 launch writes every lane's memory label (its own prediction, evaluator.py:346-353,
   :400-422) straight into the pool's label rows;
4. the pool's captured memory-update body runs on those rows.

Nothing waits for the host except on a frame with new objects, where the object count is read from the ensemble label and each
lane of that video gets a one-lane reference pass with its own overlaid label, as TTAInferEngine does.
"""
from __future__ import annotations

import torch

from . import engine as E
from . import ops
from .multi_video import DeAOTMultiVideoInferEngine, MultiVideoInferEngine
from .tta import tta_augmentations


class MultiVideoTTAInferEngine:
    """MultiVideoTTAInferEngine(aot_model, max_videos=S, long_term_mem_max=M, gpu_id=0, long_term_mem_gap=None,
    short_term_mem_skip=1, flip=None, multi_scale=None, precision=None, long_term_mem_policy=None).

    open_video(imgs, label, obj_nums, long_term_mem_gap=None) -> vid      imgs: FramePreprocessor's list for the frame
    propagate({vid: imgs}, (H, W), new_labels=None, keep_prob=False, forced_labels=None) -> {vid: label [1,1,H,W]}
    close_video(vid); videos; frame_step(vid); pred_prob {vid: [1,NC,H,W]} after a keep_prob frame

    Per video the result is TTAInferEngine(aot_model, long_term_mem_max=M, ...)'s on that video, with the same argument
    meanings; the AOT models run on MultiVideoInferEngine pools, the DeAOT models on DeAOTMultiVideoInferEngine pools, and
    whatever those refuse is refused here.  Every open video has one original size.  Returned labels and probabilities are
    views of static buffers that the next propagate overwrites."""

    def __init__(self, aot_model, max_videos=4, long_term_mem_max=None, gpu_id=0, long_term_mem_gap=None,
                 short_term_mem_skip=1, flip=None, multi_scale=None, precision=None, long_term_mem_policy=None):
        cfg = aot_model.cfg
        self.cfg, self.AOT = cfg, aot_model
        self.flip, self.multi_scale, self.flips = tta_augmentations(cfg, flip, multi_scale)
        if int(max_videos) != max_videos or max_videos < 1:
            raise ValueError(f"max_videos must be a positive integer, got {max_videos}")
        self.max_videos = int(max_videos)
        self.per_scale = 2 if self.flip else 1
        cls = DeAOTMultiVideoInferEngine if cfg.MODEL_VOS == "deaot" else MultiVideoInferEngine
        self.pools = [cls(aot_model, max_videos=self.max_videos * self.per_scale, long_term_mem_max=long_term_mem_max,
                          gpu_id=gpu_id, long_term_mem_gap=long_term_mem_gap, short_term_mem_skip=short_term_mem_skip,
                          precision=precision, long_term_mem_policy=long_term_mem_policy)
                      for _ in self.multi_scale]
        self.align_corners = cfg.MODEL_ALIGN_CORNERS
        self.max_obj_num = aot_model.max_obj_num
        self._videos = []            # open videos in merge order: dict(vid, obj, lanes = pool video id per augmentation)
        self._lane_of = [{} for _ in self.pools]      # per pool: pool video id -> (vid, augmentation)
        self._size = None            # the open videos' original (H, W)
        self._next_vid = 0
        self._fbs = {}
        self._outs = {}
        self.pred_prob = None
        self.aug_logits = None

    def enable_kv_sharding(self, rank, world, group=None):
        raise NotImplementedError("MultiVideoTTAInferEngine pools bounded banks on one GPU; a bank sharded over GPUs is not "
                                  "built for it")

    # ------------------------------------------------------------------ videos
    @property
    def videos(self):
        """The open videos' ids, in merge order."""
        return [v["vid"] for v in self._videos]

    def frame_step(self, vid):
        return self.pools[0].frame_step(self._video(vid)["lanes"][0])

    def _video(self, vid):
        for v in self._videos:
            if v["vid"] == vid:
                return v
        raise KeyError(f"video {vid} is not open (open: {self.videos})")

    def _pool_of(self, e):
        return self.pools[e // self.per_scale]

    def _device(self):
        return next(self.AOT.parameters()).device

    def _check_imgs(self, imgs):
        if len(imgs) != len(self.flips):
            raise ValueError(f"expected {len(self.flips)} augmented images (one per scale and flip, in FramePreprocessor's "
                             f"order), got {len(imgs)}")

    def _check_size(self, size):
        if self._videos and size != self._size:
            raise ValueError(f"original frame size {size} differs from the open videos' {self._size}: one engine serves one "
                             f"original size while videos are open")

    def _label_map(self, t, H, W):
        if t.numel() != H * W:
            raise ValueError(f"expected a label map of the original size {(H, W)}, got {tuple(t.shape)}")
        return t.to(self._device()).reshape(H, W).float().contiguous()

    def _check_lane_imgs(self, imgs):
        """Refuse a frame's augmented images before any pool opens a lane: one [1,3,h,w] image per augmentation, one size per
        scale, and that of the scale's pool while it has lanes."""
        self._check_imgs(imgs)
        for e, img in enumerate(imgs):
            if not isinstance(img, torch.Tensor) or img.dim() != 4 or img.shape[0] != 1 or img.shape[1] != 3:
                raise ValueError(f"augmentation {e}: expected one image [1,3,h,w], got "
                                 f"{tuple(img.shape) if isinstance(img, torch.Tensor) else img}")
            first = imgs[e - e % self.per_scale]
            if img.shape[2:] != first.shape[2:]:
                raise ValueError(f"augmentation {e}: image size {tuple(img.shape[2:])} differs from {tuple(first.shape[2:])}, "
                                 f"the unflipped image of its scale")
            p = self._pool_of(e)
            if p.videos:
                p._check_img(img)
            else:
                E.AOTEngine._check_img(p, img)

    def _trim_encoders(self):
        """Keep each pool's batched encoder buffers for one frame (reference passes) and its current lane count only.  The
        pool's LSTT graphs captured over a dropped batch size read its freed encoder buffers: they go too."""
        for p in self.pools:
            if p._enc is None:
                continue
            keep = (1, max(len(p.videos), 1))
            dropped = set(p._enc.batch_sizes()) - set(keep)
            stale = [k for k in p.graphs.slots if k[0] == "lstt" and k[1] in dropped]
            if stale:
                torch.cuda.current_stream().synchronize()     # no replay of a dropped graph is still running
            for k in stale:
                del p.graphs.slots[k]
            p._enc.keep_batch_sizes(keep)

    def open_video(self, imgs, label, obj_nums, long_term_mem_gap=None):
        """Open a video at its reference frame -> its id.  imgs: the frame's augmented images [1,3,h_e,w_e]
        (FramePreprocessor's list); label: the annotation [1,1,H,W] at the original size and orientation, which each lane
        gets mirrored if flipped and nearest-resized to its input size (evaluator.py:315-323)."""
        if len(self._videos) >= self.max_videos:
            raise ValueError(f"{self.max_videos} videos are open already (max_videos)")
        self._check_lane_imgs(imgs)
        H, W = int(label.shape[-2]), int(label.shape[-1])
        self._check_size((H, W))
        obj = self._check_objs(obj_nums)
        lab = self._label_map(label, H, W)
        v = dict(vid=self._next_vid, obj=obj, lanes=[])
        try:
            for e, img in enumerate(imgs):
                p, s = self._pool_of(e), e // self.per_scale
                fb = self._fb(s, tuple(img.shape[-2:]))
                ops.tta_feedback(None, fb, (H, W), self.align_corners, self.flips[e], new_label=lab)
                pv = p.open_video(img, fb, obj, long_term_mem_gap=long_term_mem_gap)
                v["lanes"].append(pv)
                self._lane_of[s][pv] = (v["vid"], e)
        except BaseException:
            # leave no lane of the half-opened video behind, including one whose pool failed inside its own open
            for e, pv in enumerate(v["lanes"]):
                del self._lane_of[e // self.per_scale][pv]
            for s, p in enumerate(self.pools):
                for pv in [pv for pv in p.videos if pv not in self._lane_of[s]]:
                    p.close_video(pv)
            raise
        self._next_vid += 1
        self._videos.append(v)
        self._size = (H, W)
        self._trim_encoders()
        return v["vid"]

    def _check_objs(self, obj_nums):
        if isinstance(obj_nums, (list, tuple)):
            obj_nums = obj_nums[0]
        obj = int(obj_nums)
        if obj > self.max_obj_num:
            raise NotImplementedError(f"{type(self).__name__} propagates at most {self.max_obj_num} objects per video (one "
                                      f"ID bank per augmentation), got {obj}")
        return obj

    def close_video(self, vid):
        """Close every lane of the video (each pool compacts its own slots)."""
        v = self._video(vid)
        for e, pv in enumerate(v["lanes"]):
            s = e // self.per_scale
            self.pools[s].close_video(pv)
            del self._lane_of[s][pv]
        self._videos.remove(v)
        self._trim_encoders()

    # ------------------------------------------------------------------ buffers
    def _fb(self, s, size):
        key = (s,) + size
        b = self._fbs.get(key)
        if b is None:
            b = self._fbs[key] = torch.empty(size, dtype=torch.float32, device=self._device())
        return b

    def _outputs(self, H, W, NC, prob):
        key = (H, W, NC)
        o = self._outs.get(key)
        if o is None:
            o = self._outs[key] = [torch.empty((self.max_videos, 1, H, W), dtype=torch.float32, device=self._device()), None]
        if prob and o[1] is None:
            o[1] = torch.empty((self.max_videos, NC, H, W), dtype=torch.float32, device=self._device())
        return o

    # ------------------------------------------------------------------ frame
    def propagate(self, frames, output_size, new_labels=None, keep_prob=False, forced_labels=None):
        """One frame of every open video -> {vid: ensemble label [1,1,H,W]} at output_size (the videos' original size).

        frames {vid: augmented images} for exactly the open videos.  new_labels {vid: annotation of the objects that appear
        at this frame, [1,1,H,W] at the original size and orientation}: it overwrites that video's ensemble and lane labels,
        and the frame becomes a reference frame of each of its lanes with the new object count.  keep_prob: keep the mean
        probabilities in pred_prob.  forced_labels {vid: one label map per augmentation}, for exactly the open videos: fed to
        the lanes instead of their own predictions (teacher forcing)."""
        if not self._videos:
            raise ValueError("no video is open")
        if set(frames) != set(self.videos) or len(frames) != len(self._videos):
            raise ValueError(f"propagate needs the frames of exactly the open videos {sorted(self.videos)}, got "
                             f"{sorted(frames)}")
        H, W = int(output_size[0]), int(output_size[1])
        self._check_size((H, W))
        for v in self._videos:
            self._check_imgs(frames[v["vid"]])
        new_labels = dict(new_labels or {})
        if not set(new_labels) <= set(self.videos):
            raise ValueError(f"new_labels names videos that are not open: {sorted(set(new_labels) - set(self.videos))}")
        if forced_labels is not None and (set(forced_labels) != set(self.videos)
                                          or any(len(forced_labels[v]) != len(self.flips) for v in forced_labels)):
            raise ValueError(f"forced_labels needs {len(self.flips)} label maps for each of exactly the open videos "
                             f"{sorted(self.videos)}")
        new = {vid: self._label_map(t, H, W) for vid, t in new_labels.items()}
        for vid, t in new.items():                          # refuse before anything runs (the event's count is <= its max)
            top = int(t.max().item())
            if top > self.max_obj_num:
                raise NotImplementedError(f"MultiVideoTTAInferEngine propagates at most {self.max_obj_num} objects per "
                                          f"video, got {top} in the new label of video {vid}")
        forced = None if forced_labels is None else \
            {vid: [self._label_map(t, H, W) for t in ts] for vid, ts in forced_labels.items()}
        per, ac = self.per_scale, self.align_corners

        lane_frames = [{} for _ in self.pools]
        for v in self._videos:
            for e, pv in enumerate(v["lanes"]):
                lane_frames[e // per][pv] = frames[v["vid"]][e]

        def infer(s, pool):
            pool.propagate(lane_frames[s])
            return pool.decode_nhwc()

        lgs = E.fork_join(self, self.pools, infer)
        slot = [{pv: k for k, pv in enumerate(p.videos)} for p in self.pools]
        n, NC = len(self._videos), int(lgs[0].shape[-1])
        label, prob = self._outputs(H, W, NC, keep_prob)
        ops.tta_merge_batched([lgs[e // per] for e in range(len(self.flips))], self.flips,
                              [[slot[e // per][pv] for e, pv in enumerate(v["lanes"])] for v in self._videos],
                              [v["obj"] for v in self._videos], label[:n], ac,
                              new_labels=[new.get(v["vid"]) for v in self._videos],
                              prob=prob[:n] if keep_prob else None)
        out = {v["vid"]: label[b:b + 1] for b, v in enumerate(self._videos)}
        self.pred_prob = {v["vid"]: prob[b:b + 1] for b, v in enumerate(self._videos)} if keep_prob else None
        self.aug_logits = {v["vid"]: [lgs[e // per][slot[e // per][pv]:slot[e // per][pv] + 1]
                                      for e, pv in enumerate(v["lanes"])] for v in self._videos}
        objs = {v["vid"]: v["obj"] for v in self._videos}

        def feedback(s, pool):
            lanes = [self._lane_of[s][pv] for pv in pool.videos]          # slot order
            if forced is not None:
                ops.tta_feedback_batched(None, pool.mask_rows(), None, [self.flips[e] for _, e in lanes], (H, W), ac,
                                         new_labels=[forced[vid][e] for vid, e in lanes])
            else:
                ops.tta_feedback_batched(lgs[s], pool.mask_rows(), [objs[vid] for vid, _ in lanes],
                                         [self.flips[e] for _, e in lanes], (H, W), ac,
                                         new_labels=[new.get(vid) for vid, _ in lanes])

        if not new:
            def update(s, pool):
                feedback(s, pool)
                pool.update_memory_from_masks()
            E.fork_join(self, self.pools, update)
            return out
        # new objects (evaluator.py:363-399): the video's object count is its ensemble's largest id, then each of its lanes
        # takes the frame as a reference frame with its own overlaid label
        for s, pool in enumerate(self.pools):
            feedback(s, pool)
        for b, v in enumerate(self._videos):
            if v["vid"] in new:
                v["obj"] = int(label[b].max().item())
                for e, pv in enumerate(v["lanes"]):
                    p = self._pool_of(e)
                    p.add_reference_frame(pv, frames[v["vid"]][e], p.mask_rows()[slot[e // per][pv]], v["obj"])
        for pool in self.pools:
            pool.update_memory_from_masks()
        return out

