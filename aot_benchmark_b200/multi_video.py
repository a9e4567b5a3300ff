"""Several independent videos propagated through one engine, one batched encoder + LSTT + decoder pass per frame.

Per video, the semantics are those of AOTInferEngine(long_term_mem_max=M) with up to 80 objects (DeAOTInferEngine for
DeAOTMultiVideoInferEngine): each video has its own frame step, object count, long-term gap, and per ID-bank lane (one per
10 objects, AOTInferEngine's sub-engines) its own short-term memory and bounded long-term bank (the first memory frame pinned,
the newest M - 1 in a ring).  Videos open and close independently; the nl open lanes always occupy lanes 0 .. nl - 1 of a
pool allocated once per (geometry, lanes, M) and the nv open videos rows 0 .. nv - 1 of the frame batch, so every launch
covers exactly nv videos or nl lanes and every captured graph is keyed on those counts (DESIGN §3.9).
"""
from __future__ import annotations

import math
import types

import torch

from . import engine as E
from . import ops
from .plan import get_plan


class MultiVideoInferEngine:
    """MultiVideoInferEngine(aot_model, max_videos=S, long_term_mem_max=M, gpu_id=0, long_term_mem_gap=None,
    short_term_mem_skip=1, precision=None, long_term_mem_policy=None, max_lanes=None).

    open_video(img, mask, obj_nums) -> vid            the video's reference frame (its step 0)
    propagate({vid: img})                              one batched pass over every open video; each frame step advances
    decode_current_logits(output_size) -> {vid: logits}, decode_labels(output_size) -> {vid: label}
    add_reference_frame(vid, img, mask, obj_nums, frame_step)   objects that appear mid-video (a one-video pass)
    update_memory({vid: label}, skip_long_term_update=False)    each video's own long-term gap
    close_video(vid)

    A video of k objects holds ceil(k / 10) ID-bank lanes (at least one, at most 8), the batched counterparts of
    AOTInferEngine's sub-engines: lane e carries the video's ids 10e+1 .. 10e+10, renumbered 1 .. 10.  max_lanes (default
    max_videos) sizes every per-lane buffer (banks, LSTT and decoder rows); a video whose objects need more lanes than its own
    and the free ones is refused.  Returned logits / labels are views of static buffers that the next call overwrites."""

    def __init__(self, aot_model, max_videos=4, long_term_mem_max=None, gpu_id=0, long_term_mem_gap=None,
                 short_term_mem_skip=1, precision=None, long_term_mem_policy=None, max_lanes=None):
        cfg = aot_model.cfg
        self._check_family(cfg)
        policy = getattr(cfg, "TEST_LONG_TERM_MEM_POLICY", None) if long_term_mem_policy is None else long_term_mem_policy
        if policy is not None and policy not in E.MEM_POLICIES:
            raise ValueError(f"long_term_mem_policy must be one of {E.MEM_POLICIES}, got {policy!r}")
        name = type(self).__name__
        if policy not in (None, "fifo"):
            raise NotImplementedError(f"{name} keeps FIFO banks; long_term_mem_policy='usage' counts attention mass per "
                                      f"video, which the batched attention does not")
        self._check_kernels()
        if short_term_mem_skip != 1:
            raise NotImplementedError(f"{name} keeps one short-term memory frame per video (short_term_mem_skip=1)")
        if int(max_videos) != max_videos or max_videos < 1:
            raise ValueError(f"max_videos must be a positive integer, got {max_videos}")
        if max_lanes is None:
            max_lanes = max_videos
        if isinstance(max_lanes, bool) or not isinstance(max_lanes, (int, float)) or int(max_lanes) != max_lanes \
                or max_lanes < max_videos:
            raise ValueError(f"max_lanes must be an integer >= max_videos ({max_videos}), got {max_lanes}")
        M = E._resolve_mem_max(aot_model, long_term_mem_max)
        if M is None:
            raise ValueError(f"{name} pools a bounded long-term bank per video: give long_term_mem_max (or "
                             f"cfg.TEST_LONG_TERM_MEM_MAX)")
        self.precision = E._resolve_precision(aot_model, precision)
        self.AOT, self.cfg = aot_model, cfg
        self.max_videos, self.max_lanes, self.long_term_mem_max = int(max_videos), int(max_lanes), M
        self.long_term_mem_gap = getattr(cfg, "TEST_LONG_TERM_MEM_GAP", 9999) if long_term_mem_gap is None \
            else long_term_mem_gap
        self.short_term_mem_skip = 1
        self.gpu_id = gpu_id
        self.max_obj_num = aot_model.max_obj_num
        self._P = None
        self._enc = None
        self._geom = None                # (input H, W) of the open videos' network input
        self._pool = None
        self.graphs = E.GraphCache()
        # video row -> per-video host state (dict; "lanes": its lanes in sub-engine order).  Rows follow the videos' first
        # lanes, so while every video holds one lane, video row b is lane b.
        self._videos = []
        self._lanes = []                 # lane -> per-lane host state (dict); lane order = stacking order of every pool buffer
        self._next_vid = 0

    # per-layer workspace buffers that carry a lane's state from propagate to update_memory (close_video moves them)
    _CARRIED = ("st_K", "st_V", "curr_Q", "curr_V")
    MAX_LANES_PER_VIDEO = 8              # the logit aggregation kernel's limit: 8 sub-engines

    def _check_family(self, cfg):
        if cfg.MODEL_VOS == "deaot":
            raise NotImplementedError("MultiVideoInferEngine runs the AOT models; DeAOT's gated propagation runs on "
                                      "DeAOTMultiVideoInferEngine")

    def _check_kernels(self):
        """Refuse the knobs that select a kernel other than the batched entry points' (read at construction)."""
        if E.LT_IMPL == "simt":
            raise NotImplementedError("MultiVideoInferEngine runs the tensor-core long-term attention; AOTB_LT_IMPL=simt "
                                      "selects the fp32 CUDA-core kernel")
        if ops.CONV_IMPL == "simt":
            raise NotImplementedError("MultiVideoInferEngine runs the tensor-core conv; AOTB_CONV_IMPL=simt selects the fp32 "
                                      "CUDA-core conv")
        if ops.LT_VARIANT != "tile":
            raise NotImplementedError(f"MultiVideoInferEngine runs the default 'tile' layout of the long-term attention; "
                                      f"AOTB_LT_VARIANT={ops.LT_VARIANT} selects another")
        if E.LOCAL_IMPL != "tc":
            raise NotImplementedError(f"MultiVideoInferEngine runs the tensor-core local attention; AOTB_LOCAL_IMPL="
                                      f"{E.LOCAL_IMPL} selects a CUDA-core kernel")

    # ------------------------------------------------------------------ protocol
    def enable_kv_sharding(self, rank, world, group=None):
        raise NotImplementedError(f"{type(self).__name__} pools bounded banks on one GPU; a bank sharded over GPUs is not "
                                  f"built for it")

    @property
    def videos(self):
        """The open videos' ids, in video-row order."""
        return [v["vid"] for v in self._videos]

    def frame_step(self, vid):
        return self._videos[self._row(vid)]["frame_step"]

    def video_lanes(self, vid):
        """The lanes of video vid, in sub-engine order."""
        return list(self._videos[self._row(vid)]["lanes"])

    def _row(self, vid):
        for i, v in enumerate(self._videos):
            if v["vid"] == vid:
                return i
        raise KeyError(f"video {vid} is not open (open: {self.videos})")

    def _lanes_for(self, obj_nums, own=0):
        """-> (object count, lanes it needs) for a video holding `own` lanes; NotImplementedError when they do not fit."""
        if isinstance(obj_nums, (list, tuple)):
            obj_nums = obj_nums[0]
        obj, per, name = int(obj_nums), self.max_obj_num, type(self).__name__
        top = per * self.MAX_LANES_PER_VIDEO
        if obj > top:
            raise NotImplementedError(f"{name} propagates at most {top} objects per video ({self.MAX_LANES_PER_VIDEO} ID "
                                      f"banks of {per}), got {obj}")
        want = max(-(-obj // per), 1, own)
        avail = own + self.max_lanes - len(self._lanes)
        if want > avail:
            raise NotImplementedError(f"{name} propagates at most {per * avail} objects in this video: {avail} ID-bank "
                                      f"lane(s) of max_lanes={self.max_lanes} are its own or free, got {obj}")
        return obj, want

    def _set_objs(self, v, obj):
        """AOTInferEngine.separate_mask's object counts: every lane but the last holds max_obj_num objects."""
        k, per = len(v["lanes"]), self.max_obj_num
        counts = [obj] if k == 1 else [per] * (k - 1) + [obj % per or per]
        v["obj"] = obj
        for l, c in zip(v["lanes"], counts):
            self._lanes[l]["obj"] = c

    def _add_lanes(self, v, want):
        pl = self._pool
        while len(v["lanes"]) < want:
            b = len(self._lanes)
            self._lanes.append(dict(video=v, obj=0, bank_len=0))
            v["lanes"].append(b)
            pl.tk[b].zero_()
            pl.wr[b].zero_()

    def _check_img(self, img):
        if not isinstance(img, torch.Tensor) or img.dim() != 4 or img.shape[0] != 1 or img.shape[1] != 3:
            raise ValueError(f"expected one frame [1,3,H,W], got {tuple(img.shape) if isinstance(img, torch.Tensor) else img}")
        E.AOTEngine._check_img(self, img)
        if self._geom is not None and tuple(img.shape[2:]) != self._geom:
            raise ValueError(f"frame size {tuple(img.shape[2:])} differs from the open videos' {self._geom}: one engine "
                             f"serves one network input size")

    @E._in_precision
    def open_video(self, img, mask, obj_nums, long_term_mem_gap=None):
        """Open a video at its reference frame (frame step 0) -> its id.  long_term_mem_gap: this video's gap (default: the
        engine's)."""
        if len(self._videos) >= self.max_videos:
            raise ValueError(f"{self.max_videos} videos are open already (max_videos)")
        obj, want = self._lanes_for(obj_nums)
        if not self._videos:
            self._geom = None
        self._check_img(img)
        E._apply_pdl()
        self._plan(refresh=True)
        self._ensure_pool(tuple(img.shape[2:]))
        v = dict(vid=self._next_vid, frame_step=0, last_mem_step=0, obj=obj, lanes=[],
                 gap=self.long_term_mem_gap if long_term_mem_gap is None else long_term_mem_gap)
        self._videos.append(v)
        self._next_vid += 1
        self._add_lanes(v, want)
        self._set_objs(v, obj)
        self._reference_passes(v, img, mask)
        return v["vid"]

    @E._in_precision
    def add_reference_frame(self, vid, img, mask, obj_nums, frame_step=-1):
        """New objects in video `vid` at its current frame (AOTInferEngine.add_reference_frame): a one-video pass on each of
        its lanes, after taking the lanes a larger object count needs; the frame becomes a memory frame of every lane's bank
        (a new lane's bank starts at it).  frame_step is accepted for the evaluator's call form and, as on AOTEngine without
        a stored clip, not used: the frame is the video's current step."""
        v = self._videos[self._row(vid)]
        obj, want = self._lanes_for(obj_nums, own=len(v["lanes"]))
        self._check_img(img)
        E._apply_pdl()
        self._plan(refresh=True)
        self._add_lanes(v, want)
        self._set_objs(v, obj)
        self._reference_passes(v, img, mask)

    def _reference_passes(self, v, img, mask):
        if len(v["lanes"]) == 1:
            self._reference_pass(v["lanes"][0], img, mask)
        else:
            self._reference_pass_lanes(v["lanes"], img, mask)
        v["last_mem_step"] = v["frame_step"]

    def _reference_pass(self, b, img, mask):
        """AOTEngine.add_reference_frame on lane b: encode (B = 1), ID embedding of the mask, LSTT with the frame's own K / V
        as its long-term memory, store into the lane's bank."""
        pl, N = self._pool, self._N
        st = E._cur_stream()
        embs = self._enc(img, st).nhwc
        for src, dst in zip(embs[:3], pl.dec_in):
            ops.eltwise(ops.EW_COPY, src.reshape(-1, src.shape[3]), None, dst[b:b + 1].reshape(-1, dst.shape[3]), stream=st)
        self._copy_mask(b, mask, st)
        self._lane_reference(b, embs, st)

    def _reference_pass_lanes(self, lanes, img, mask):
        """AOTInferEngine.add_reference_frame over a video's lanes: one encoder pass, the mask separated into every lane's
        row by one launch, then _reference_pass's ID embedding, LSTT and store on each lane."""
        pl = self._pool
        st = E._cur_stream()
        embs = self._enc(img, st).nhwc
        m = self._label_map(mask)
        ops.separate_labels_batched([m] * len(lanes), list(range(len(lanes))), [pl.mask[b] for b in lanes],
                                    self.max_obj_num, stream=st)
        for b in lanes:
            for src, dst in zip(embs[:3], pl.dec_in):
                ops.eltwise(ops.EW_COPY, src.reshape(-1, src.shape[3]), None, dst[b:b + 1].reshape(-1, dst.shape[3]),
                            stream=st)
            self._lane_reference(b, embs, st)

    def _lane_reference(self, b, embs, st):
        N = self._N
        self._id_embed(b, 1, st)
        self._lstt(b, 1, embs[-1].reshape(N, self._P.C), st, ref=True)
        self._store(b, 1, st, flags=[1])
        s = self._lanes[b]
        s["bank_len"] = min(s["bank_len"] + N, self.long_term_mem_max * N)

    def _one_lane_each(self):
        """True while every open video holds one lane: then video row b is lane b and no lane table is needed."""
        return len(self._lanes) == len(self._videos)

    @E._in_precision
    def propagate(self, frames):
        """frames {vid: img [1,3,H,W]} with exactly the open videos: one batched encoder pass over the videos, one LSTT pass
        over their lanes; every frame step advances by one."""
        if not self._videos:
            raise ValueError("no video is open")
        if set(frames) != set(self.videos) or len(frames) != len(self._videos):
            raise ValueError(f"propagate needs a frame for exactly the open videos {sorted(self.videos)}, got "
                             f"{sorted(frames)}")
        nv, nl, pl, N = len(self._videos), len(self._lanes), self._pool, self._N
        for v in self._videos:
            self._check_img(frames[v["vid"]])
        st = E._cur_stream()
        for b, v in enumerate(self._videos):
            pl.frames[b:b + 1].copy_(frames[v["vid"]])
        embs = self._enc(pl.frames[:nv], st).nhwc
        splits = self._splits(nl * N, max(max(s["bank_len"] for s in self._lanes), 1))

        if self._one_lane_each():
            def body():
                s2 = E._cur_stream()
                for src, dst in zip(embs[:3], pl.dec_in):
                    ops.eltwise(ops.EW_COPY, src.reshape(-1, src.shape[3]), None, dst[:nl].reshape(-1, dst.shape[3]),
                                stream=s2)
                self._lstt(0, nl, embs[-1].reshape(nl * N, self._P.C), s2, ref=False, splits=splits)
        else:
            # the encoder maps of lane l are those of video lane_video[l]: one gather launch reading the device table, which
            # is written here, before the replay, so a graph does not depend on which video owns which lane
            x16 = self._lane_tables()
            self._write_i32(pl.lane_video, [self._videos.index(s["video"]) for s in self._lanes])

            def body():
                s2 = E._cur_stream()
                ops.lane_gather(list(embs), list(pl.dec_in) + [x16], pl.lane_video, nl, stream=s2)
                self._lstt(0, nl, x16[:nl].reshape(nl * N, self._P.C), s2, ref=False, splits=splits)
        self.graphs.run(("lstt", nv, nl, splits) + tuple(t.data_ptr() for t in embs), body)
        for v in self._videos:
            v["frame_step"] += 1

    def _write_i32(self, dev, values):
        host = torch.tensor(values, dtype=torch.int32)
        if dev.is_cuda:
            # pinned by the caching host allocator, which keeps the block until the asynchronous copy has run: no host sync
            host = host.pin_memory()
        dev[:len(values)].copy_(host, non_blocking=True)

    def _lane_tables(self):
        """The lane-ordered stride-16 encoder map and the device lane table, allocated when a video first holds two lanes."""
        pl = self._pool
        if pl.x16 is None:
            dev = pl.tk.device
            pl.x16 = torch.empty((self.max_lanes,) + self._hw + (self._P.C,), dtype=torch.float32, device=dev)
            pl.lane_video = torch.zeros(self.max_lanes, dtype=torch.int32, device=dev)
        return pl.x16

    @E._in_precision
    def decode_current_logits(self, output_size=None):
        """-> {vid: logits [1, 1 + 10k, h, w]} for a video of k lanes (output_size None: the stride-4 map, else upsampled to
        output_size).  The decoder over the lanes is one graph keyed on their count; each one-lane video's logit
        post-processing (masking the ids above its object count, upsampling) follows it as an eager launch, and the videos of
        several lanes are post-processed and aggregated (AOTInferEngine.soft_logit_aggregation) by one more, so object
        counts that change as videos open, close or gain objects need no new graph."""
        size = None if output_size is None else (int(output_size[0]), int(output_size[1]))
        out, multi, lg = self._postproc(size)
        if multi:
            hw = size or (lg.shape[1], lg.shape[2])
            maps = [E._static_buf(self._pool.dec, ("agg", b), (1, 1 + self.max_obj_num * len(self._videos[b]["lanes"])) + hw,
                                  lg.device) for b in multi]
            self._aggregate(lg, multi, out=maps)
            for b, t in zip(multi, maps):
                out[self._videos[b]["vid"]] = t
        return {v["vid"]: out[v["vid"]] for v in self._videos}

    def _postproc(self, size):
        """The decoder, then logits_postproc for each one-lane video -> ({vid: its logits}, rows of the videos of several
        lanes, the decoder output)."""
        lg = self.decode_nhwc()
        st = E._cur_stream()
        h4, w4, NC = lg.shape[1], lg.shape[2], lg.shape[3]
        self._last_lowres, out, multi = {}, {}, []
        for b, v in enumerate(self._videos):
            if len(v["lanes"]) > 1:
                multi.append(b)
                continue
            l = v["lanes"][0]
            lo = E._static_buf(self._pool.dec, ("lo", b), (1, NC, h4, w4), lg.device)
            up = None if size is None else E._static_buf(self._pool.dec, ("out", b), (1, NC) + size, lg.device)
            ops.logits_postproc(lg[l:l + 1], lo, up, self._lanes[l]["obj"], self._P.align_corners, stream=st)
            self._last_lowres[b] = lo
            out[v["vid"]] = lo if up is None else up
        return out, multi, lg

    def _aggregate(self, lg, rows, out=None, labels=None):
        lanes = [self._videos[b]["lanes"] for b in rows]
        ops.soft_logit_aggregation_batched(lg, lanes, [[self._lanes[l]["obj"] for l in r] for r in lanes],
                                           self._P.align_corners, out=out, labels=labels, max_obj=self.max_obj_num,
                                           stream=E._cur_stream())

    @E._in_precision
    def decode_nhwc(self):
        """The decoder over the open lanes -> their raw logits [lanes, h/4, w/4, 11] (NHWC, lane order, no object-count
        mask): a static buffer the next decode overwrites.  decode_current_logits post-processes it per video."""
        nl = len(self._lanes)
        return self.graphs.run(("dec", nl), lambda: self._decode(nl))

    def decode_labels(self, output_size=None):
        """decode_current_logits fused with the argmax of each video's upsampled logits -> {vid: label [1, H, W] int64}.  A
        video of several lanes takes the first argmax of its lanes' logits aggregated at the output size."""
        _, multi, lg = self._postproc(None)
        size = self._geom if output_size is None else (int(output_size[0]), int(output_size[1]))
        st = E._cur_stream()
        out = {}
        for b, lo in self._last_lowres.items():
            label = torch.empty((1,) + tuple(size), dtype=torch.float32, device=lo.device)
            ops.logits_argmax(lo, label, self._P.align_corners, stream=st)
            out[self._videos[b]["vid"]] = label
        if multi:
            labels = [torch.empty((1,) + tuple(size), dtype=torch.float32, device=lg.device) for _ in multi]
            self._aggregate(lg, multi, labels=labels)
            for b, t in zip(multi, labels):
                out[self._videos[b]["vid"]] = t
        return {v["vid"]: out[v["vid"]].long() for v in self._videos}

    @E._in_precision
    def update_memory(self, labels, skip_long_term_update=False):
        """labels {vid: label map [1,1,H,W] | [1,H,W]} for exactly the open videos: every lane's short-term memory, and
        the long-term banks of each video whose own gap has passed since its last memory frame.  A video of several lanes
        has its map separated into its lanes' rows (AOTInferEngine.separate_mask), one launch for all such videos."""
        if set(labels) != set(self.videos):
            raise ValueError(f"update_memory needs a label map for exactly the open videos {sorted(self.videos)}, got "
                             f"{sorted(labels)}")
        st = E._cur_stream()
        src, parts, dst = [], [], []
        for v in self._videos:
            if len(v["lanes"]) == 1:
                self._copy_mask(v["lanes"][0], labels[v["vid"]], st)
                continue
            m = self._label_map(labels[v["vid"]])
            for e, l in enumerate(v["lanes"]):
                src.append(m)
                parts.append(e)
                dst.append(self._pool.mask[l])
        if src:
            ops.separate_labels_batched(src, parts, dst, self.max_obj_num, stream=st)
        self.update_memory_from_masks(skip_long_term_update)

    def mask_rows(self):
        """The open lanes' label-map rows [lanes, H, W] at the network input size (lane order), which update_memory fills
        and update_memory_from_masks reads."""
        return self._pool.mask[:len(self._lanes)]

    @E._in_precision
    def update_memory_from_masks(self, skip_long_term_update=False):
        """update_memory on the label maps already in mask_rows() (written on the current stream): every lane's
        short-term memory, and the long-term banks of each video whose own gap has passed since its last memory frame."""
        nl, pl = len(self._lanes), self._pool
        for v in self._videos:
            v["store"] = 0
            if v["frame_step"] - v["last_mem_step"] >= v["gap"]:
                v["store"] = 0 if skip_long_term_update else 1
                v["last_mem_step"] = v["frame_step"]
        flags = [s["video"]["store"] for s in self._lanes]
        self._write_i32(pl.flags, flags)

        def body():
            s2 = E._cur_stream()
            self._id_embed(0, nl, s2)
            self._fuse_memories(self._rows(0, nl), s2)
            self._store(0, nl, s2)
        self.graphs.run(("upd", nl), body)
        for s, f in zip(self._lanes, flags):
            if f:
                s["bank_len"] = min(s["bank_len"] + self._N, self.long_term_mem_max * self._N)

    def close_video(self, vid):
        """Free the video's lanes and row: the highest open lanes move into its lanes below the new lane count (one device
        copy per buffer), so the open lanes stay in lanes 0 .. n - 1, and the video rows follow the videos' first lanes."""
        v = self._videos[self._row(vid)]
        freed = sorted(v["lanes"])
        keep = len(self._lanes) - len(freed)
        movers = [l for l in range(len(self._lanes) - 1, keep - 1, -1) if l not in freed]
        for dst, src in zip([l for l in freed if l < keep], movers):
            self._move_lane(dst, src)
            s = self._lanes[dst] = self._lanes[src]
            lanes = s["video"]["lanes"]
            lanes[lanes.index(src)] = dst
        del self._lanes[keep:]
        self._videos.remove(v)
        self._videos.sort(key=lambda u: u["lanes"][0])

    def _move_lane(self, b, last):
        pl, N, MN = self._pool, self._N, self.long_term_mem_max * self._N
        rows = lambda t, s, r: t[s * r:(s + 1) * r]
        for li in range(self._P.L):
            for t in (pl.bank_K[li], pl.bank_V[li]):
                rows(t, b, MN).copy_(rows(t, last, MN))
            for t in (pl.bank_Kp[li], pl.bank_Vp[li]):
                t[:, b * MN:(b + 1) * MN].copy_(t[:, last * MN:(last + 1) * MN])
            for name in self._CARRIED:
                t = pl.lstt[name][li]
                if t is not None:                              # DeAOT's curr_IDV[0]
                    rows(t, b, N).copy_(rows(t, last, N))
        rows(pl.cat, b, N).copy_(rows(pl.cat, last, N))          # the decoder's inputs: LSTT output, encoder maps
        for t in pl.dec_in:
            t[b].copy_(t[last])
        for t in (pl.tk, pl.wr):
            t[b].copy_(t[last])

    def _lane_bank(self, b):
        pl, MN, n = self._pool, self.long_term_mem_max * self._N, self._lanes[b]["bank_len"]
        return [[pl.bank_K[li][b * MN:b * MN + n], pl.bank_V[li][b * MN:b * MN + n]] for li in range(self._P.L)]

    @property
    def long_term_memories(self):
        """{vid: per layer [K, V] fp32 live rows of the bank of the video's first lane} (AOTInferEngine's sub-engine 0; see
        AOTEngine.long_term_memories)."""
        return {v["vid"]: self._lane_bank(v["lanes"][0]) for v in self._videos}

    def lane_long_term_memories(self, vid):
        """Per lane of video vid (sub-engine order): per layer [K, V] fp32 live rows of its bank."""
        return [self._lane_bank(b) for b in self._videos[self._row(vid)]["lanes"]]

    # ------------------------------------------------------------------ pool
    def _plan(self, refresh=False):
        if self._P is None or refresh:
            P = get_plan(self.AOT)
            self._check_plan(P)
            if self._P is not None and P is not self._P:
                self.graphs.clear()
            self._P = P
        return self._P

    def _check_plan(self, P):
        if P.C != 256 or P.C // P.H != 32:
            raise NotImplementedError(f"MultiVideoInferEngine runs the 8 x 32 attention heads of the AOT models with "
                                      f"256 channels, got {P.H} heads of {P.C // P.H}")

    def _ensure_pool(self, geom):
        P = self._P
        key = (id(P), geom)
        if self._pool is not None and self._pool.key == key:
            self._geom = geom
            return
        self.graphs.clear()
        dev = P.device
        S, V, M, C, L = self.max_lanes, self.max_videos, self.long_term_mem_max, P.C, P.L
        self._enc = E._Encoder(P, geom[0], geom[1])
        with torch.no_grad():
            probe = self._enc(torch.zeros((1, 3) + geom, device=dev), E._cur_stream()).nhwc
        h, w = probe[-1].shape[1], probe[-1].shape[2]
        N = h * w
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        hz = lambda *s: torch.zeros(s, dtype=torch.float16, device=dev)
        pl = type("Pool", (), {})()
        pl.key = key
        pl.frames = torch.zeros((V, 3) + geom, dtype=torch.float32, device=dev)        # per video; the rest per lane
        pl.dec_in = [torch.zeros((S,) + tuple(t.shape[1:]), dtype=torch.float32, device=dev) for t in probe[:3]]
        pl.mask = torch.zeros((S,) + geom, dtype=torch.float32, device=dev)
        pl.flags = torch.zeros(S, dtype=torch.int32, device=dev)
        pl.tk = torch.zeros(S, dtype=torch.int32, device=dev)
        pl.wr = torch.zeros(S, dtype=torch.int32, device=dev)
        R = S * N
        pl.lstt = self._lstt_buffers(R, C, L, dev)
        vars(pl).update(pl.lstt)
        kc, vc = pl.st_K[0].shape[1], pl.st_V[0].shape[1]      # widths of a memory frame's K / V rows
        pl.bank_K, pl.bank_V = [f(S * M * N, kc) for _ in range(L)], [f(S * M * N, vc) for _ in range(L)]
        # packed operands, one 32-channel chunk per "head"
        pl.bank_Kp, pl.bank_Vp = [hz(kc // 32, S * M * N, 64) for _ in range(L)], [hz(vc // 32, S * M * N, 64) for _ in range(L)]
        pl.Qp, pl.saKp, pl.saVp = hz(kc // 32, R, 64), hz(kc // 32, R, 64), hz(vc // 32, R, 64)
        pl.part = {}
        pl.gn_ws = ops.groupnorm_workspace(S, 32, dev)
        pl.pos = E._pos_emb_sine(h, w, npf=C // 2).to(dev).repeat(S, 1).contiguous()
        pl.dec = {}
        pl.x16 = pl.lane_video = None    # _lane_tables
        self._pool, self._N, self._hw, self._geom = pl, N, (h, w), geom

    def _lstt_buffers(self, rows, C, L, dev):
        return E._aot_lstt_buffers(rows, C, L, dev)

    def _splits(self, rows, tk):
        """KV-split count of the batched long-term attention over `rows` query rows and at most tk live keys."""
        return E.lt_splits(rows, self._P.H, tk)

    def _id_embed(self, b, n, st):
        """The ID embedding of lanes [b, b + n)'s label maps into their id_emb rows."""
        P, pl, N = self._P, self._pool, self._N
        ops.id_embed_runs_batched(pl.mask[b:b + n], P.id_wp, P.id_b, pl.id_emb[b * N:(b + n) * N], P.C, P.nid, P.id_k,
                                  P.id_stride, P.id_pad, ln_gamma=P.id_norm[0] if P.deaot else None,
                                  ln_beta=P.id_norm[1] if P.deaot else None, stream=st)

    def _fuse_memories(self, a, st):
        E.aot_fuse_memories(self._P, a, a.id_emb, a.st_K, a.st_V, st)

    def _label_map(self, mask):
        m = mask.reshape(mask.shape[-2], mask.shape[-1]) if mask.dim() >= 2 else None
        if m is None or mask.numel() != m.numel() or tuple(m.shape) != self._geom:
            raise ValueError(f"expected a label map of the network input size {self._geom}, got {tuple(mask.shape)}")
        return m.float().contiguous()

    def _copy_mask(self, b, mask, st):
        ops.eltwise(ops.EW_COPY, self._label_map(mask), None, self._pool.mask[b], stream=st)

    def _attention(self, Q, Kp, Vp, kv_stride, n, Tk, Tk_dev, out, splits, st):
        P, N = self._P, self._N
        pl = self._pool
        ops.tc_pack_rows(Q, pl.Qp, 0, div=math.sqrt(P.C // P.H), stream=st)
        exact = E.LT_IMPL == "tc_exact" and self.precision == "fp32"
        part = E._split_partials(pl.part, splits, n * N, P.H, P.C, pl.x.device, cap_rows=self.max_lanes * N) \
            if splits > 1 else None
        ops.lt_attention_tc_batched(pl.Qp, N, Kp, Vp, kv_stride, n, N, Tk=Tk, Tk_dev=Tk_dev, O=out, splits=splits,
                                    exact=exact, part=part, stream=st)

    # ------------------------------------------------------------------ batched bodies (rows of lanes b .. b + n - 1)
    def _rows(self, b, n):
        """The LSTT workspace of lanes [b, b + n): every activation (and per-layer list) sliced to their rows."""
        r = slice(b * self._N, (b + n) * self._N)
        a = types.SimpleNamespace(gn_ws=self._pool.gn_ws)
        for k, t in self._pool.lstt.items():
            setattr(a, k, t[r] if isinstance(t, torch.Tensor) else [None if u is None else u[r] for u in t])
        return a

    def _lstt(self, b, n, proj, st, ref, splits=None):
        """engine.aot_lstt over lanes [b, b + n): ref = the reference-frame form, else the propagation form over the
        lanes' banks.  Each attention step packs its operands and runs the batched tensor-core kernel."""
        P, pl, N = self._P, self._pool, self._N
        a = self._rows(b, n)
        sa_splits = E.lt_splits(n * N, P.H, N)

        def own(Q, K, V, out, st, long_term):
            ops.tc_pack_rows(K, pl.saKp, 0, stream=st)
            ops.tc_pack_rows(V, pl.saVp, 0, stream=st)
            self._attention(Q, pl.saKp, pl.saVp, N, n, N, None, out, sa_splits, st)

        def bank(li, Q, out, st):
            MN = self.long_term_mem_max * N
            self._attention(Q, pl.bank_Kp[li], pl.bank_Vp[li], MN, n, 0, pl.tk[b:b + n], out, splits, st)

        def local(li, Q, K, V, out, st):
            Lw = P.layers[li]
            ops.local_attention_tc_batched(Q, K, V, Lw.relk_w, Lw.relk_b, Lw.relv_t, out, *self._hw, P.H, n, stream=st)

        E.aot_lstt(P, a, proj, pl.pos[:n * N], self._hw, n, a.st_K, a.st_V, a.id_emb if ref else None, own, bank, local,
                   st)

    def _store(self, b, n, st, flags=None):
        """Store lanes [b, b + n)'s short-term K / V into their banks where the store flag is set (flags: written here
        first, for the eager one-video pass), then advance those banks' rings."""
        pl, N, MN = self._pool, self._N, self.long_term_mem_max * self._N
        if flags is not None:
            pl.flags[b:b + n].fill_(flags[0])
        r = slice(b * N, (b + n) * N)
        for li in range(self._P.L):
            ops.bank_ring_store_batched(pl.st_K[li][r], pl.st_V[li][r], pl.bank_K[li][b * MN:], pl.bank_V[li][b * MN:],
                                        pl.bank_Kp[li][:, b * MN:], pl.bank_Vp[li][:, b * MN:], pl.wr[b:b + n],
                                        pl.flags[b:b + n], n, MN, stream=st)
        ops.ring_advance_batched(pl.tk[b:b + n], pl.wr[b:b + n], pl.flags[b:b + n], n, N, MN, N, stream=st)

    def _decode(self, n):
        """engine.fpn_decode over the n open lanes (B = n) -> their logits [n, h/4, w/4, 11] (NHWC)."""
        pl = self._pool
        x4, x8, x16 = (t[:n] for t in pl.dec_in)
        return E.fpn_decode(self._P, pl.cat[:n * self._N].view(n, *self._hw, -1), x4, x8, x16, pl.dec, pl.gn_ws,
                            E._cur_stream())


class DeAOTMultiVideoInferEngine(MultiVideoInferEngine):
    """DeAOTMultiVideoInferEngine(aot_model, max_videos=S, long_term_mem_max=M, gpu_id=0, long_term_mem_gap=None,
    short_term_mem_skip=1, precision=None, long_term_mem_policy=None, max_lanes=None).

    MultiVideoInferEngine for the DeAOT models: the same protocol, with per video the semantics of
    DeAOTInferEngine(long_term_mem_max=M) with up to 80 objects.  Each frame's gated propagation (engine.deaot_lstt) runs
    over the open lanes through the batched fused long-term / self-attention and the batched gated local attention."""

    _CARRIED = MultiVideoInferEngine._CARRIED + ("curr_IDV",)

    def _check_family(self, cfg):
        if cfg.MODEL_VOS != "deaot":
            raise NotImplementedError("DeAOTMultiVideoInferEngine runs the DeAOT models; AOT models run on "
                                      "MultiVideoInferEngine")

    def _check_kernels(self):
        if ops.CONV_IMPL == "simt":
            raise NotImplementedError("DeAOTMultiVideoInferEngine runs the tensor-core conv; AOTB_CONV_IMPL=simt selects "
                                      "the fp32 CUDA-core conv")
        if E.DEAOT_LT != "tc":
            raise NotImplementedError(f"DeAOTMultiVideoInferEngine runs DeAOT's fused tensor-core attention; "
                                      f"AOTB_DEAOT_LT={E.DEAOT_LT} selects another path")
        if E.LOCAL_IMPL == "warp":
            raise NotImplementedError("DeAOTMultiVideoInferEngine runs the tiled gated local attention; AOTB_LOCAL_IMPL=warp "
                                      "selects the per-warp kernel")

    def _check_plan(self, P):
        if P.C != 256:
            raise NotImplementedError(f"DeAOTMultiVideoInferEngine runs the gated attention of 128 key and 1024 value "
                                      f"channels (256-channel models), got {P.C} channels")

    def _lstt_buffers(self, rows, C, L, dev):
        return E._deaot_gpm_buffers(rows, C, L, dev)

    def _splits(self, rows, tk):
        return E.gp_splits(rows, self._P.C, tk)

    def _fuse_memories(self, a, st):
        E.deaot_fuse_memories(self._P, a, a.id_emb, a.st_K, a.st_V, st)

    def _lstt(self, b, n, proj, st, ref, splits=None):
        """engine.deaot_lstt over lanes [b, b + n): ref = the reference-frame form, else the propagation form over the
        lanes' banks.  Each attention step packs its operands and runs the batched fused kernel."""
        P, pl, N = self._P, self._pool, self._N
        a = self._rows(b, n)
        MN = self.long_term_mem_max * N
        exact = self.precision == "fp32"

        def attend(Q, Kp, Vp, kv_stride, Tk, Tk_dev, out, splits, st):
            ops.tc_pack_rows(Q, pl.Qp, 0, div=math.sqrt(Q.shape[1]), stream=st)      # Q / T (attention.py:672)
            part = E._split_partials(pl.part, splits, n * N, 1, out.shape[1], out.device, cap_rows=self.max_lanes * N) \
                if splits > 1 else None
            ops.gp_attention_tc_batched(pl.Qp, N, Kp, Vp, kv_stride, n, N, Tk=Tk, Tk_dev=Tk_dev, O=out, splits=splits,
                                        exact=exact, part=part, stream=st)

        def own(Q, K, V, out, st, long_term):
            ops.tc_pack_rows(K, pl.saKp, 0, stream=st)
            ops.tc_pack_rows(V, pl.saVp, 0, stream=st)
            attend(Q, pl.saKp, pl.saVp, N, N, None, out, E.gp_splits(n * N, P.C, N), st)

        def bank(li, Q, out, st):
            attend(Q, pl.bank_Kp[li], pl.bank_Vp[li], MN, 0, pl.tk[b:b + n], out, splits, st)

        def local(li, Q, K, V, out, st):
            Lw = P.layers[li]
            ops.local_gated_tile_batched(Q, K, V, Lw.relk_w, Lw.relk_b, out, *self._hw, n, stream=st)

        E.deaot_lstt(P, a, proj, self._hw, n, a.st_K, a.st_V, a.id_emb if ref else None, own, bank, local, st)
