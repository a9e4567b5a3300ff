"""Several independent videos propagated through one engine, one batched encoder + LSTT + decoder pass per frame.

Per video, the semantics are those of AOTInferEngine(long_term_mem_max=M) with at most 10 objects (DeAOTInferEngine for
DeAOTMultiVideoInferEngine): each video has its own frame step, object count, long-term gap, short-term memory and bounded
long-term bank (the first memory frame pinned, the newest M - 1 in a ring).  Videos open and close independently; the n open
videos always occupy slots 0 .. n - 1 of a pool allocated once per (geometry, S, M), so every launch covers exactly n videos
and every captured graph is keyed on n (DESIGN §3.9).
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
    short_term_mem_skip=1, precision=None, long_term_mem_policy=None).

    open_video(img, mask, obj_nums) -> vid            the video's reference frame (its step 0)
    propagate({vid: img})                              one batched pass over every open video; each frame step advances
    decode_current_logits(output_size) -> {vid: logits}, decode_labels(output_size) -> {vid: label}
    add_reference_frame(vid, img, mask, obj_nums, frame_step)   objects that appear mid-video (a one-video pass)
    update_memory({vid: label}, skip_long_term_update=False)    each video's own long-term gap
    close_video(vid)

    Returned logits / labels are views of static buffers that the next call overwrites."""

    def __init__(self, aot_model, max_videos=4, long_term_mem_max=None, gpu_id=0, long_term_mem_gap=None,
                 short_term_mem_skip=1, precision=None, long_term_mem_policy=None):
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
        M = E._resolve_mem_max(aot_model, long_term_mem_max)
        if M is None:
            raise ValueError(f"{name} pools a bounded long-term bank per video: give long_term_mem_max (or "
                             f"cfg.TEST_LONG_TERM_MEM_MAX)")
        self.precision = E._resolve_precision(aot_model, precision)
        self.AOT, self.cfg = aot_model, cfg
        self.max_videos, self.long_term_mem_max = int(max_videos), M
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
        self._slots = []                 # slot -> per-video host state (dict); slot order = stacking order of every buffer
        self._next_vid = 0

    # per-layer workspace buffers that carry a video's state from propagate to update_memory (close_video moves them)
    _CARRIED = ("st_K", "st_V", "curr_Q", "curr_V")

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
        """The open videos' ids, in slot order."""
        return [s["vid"] for s in self._slots]

    def frame_step(self, vid):
        return self._slots[self._slot(vid)]["frame_step"]

    def _slot(self, vid):
        for i, s in enumerate(self._slots):
            if s["vid"] == vid:
                return i
        raise KeyError(f"video {vid} is not open (open: {self.videos})")

    def _check_objs(self, obj_nums):
        if isinstance(obj_nums, (list, tuple)):
            obj_nums = obj_nums[0]
        obj = int(obj_nums)
        if obj > self.max_obj_num:
            raise NotImplementedError(f"{type(self).__name__} propagates at most {self.max_obj_num} objects per video (one "
                                      f"ID bank), got {obj}")
        return obj

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
        if len(self._slots) >= self.max_videos:
            raise ValueError(f"{self.max_videos} videos are open already (max_videos)")
        obj = self._check_objs(obj_nums)
        if not self._slots:
            self._geom = None
        self._check_img(img)
        E._apply_pdl()
        P = self._plan(refresh=True)
        self._ensure_pool(tuple(img.shape[2:]))
        b = len(self._slots)
        self._slots.append(dict(vid=self._next_vid, frame_step=0, last_mem_step=0, obj=obj, bank_len=0,
                                gap=self.long_term_mem_gap if long_term_mem_gap is None else long_term_mem_gap))
        self._next_vid += 1
        pl = self._pool
        pl.tk[b].zero_()
        pl.wr[b].zero_()
        self._reference_pass(b, img, mask)
        return self._slots[b]["vid"]

    @E._in_precision
    def add_reference_frame(self, vid, img, mask, obj_nums, frame_step=-1):
        """New objects in video `vid` at its current frame (AOTEngine.add_reference_frame): a one-video pass on its slot;
        the frame becomes a memory frame of its bank.  frame_step is accepted for the evaluator's call form and, as on
        AOTEngine without a stored clip, not used: the frame is the video's current step."""
        b = self._slot(vid)
        obj = self._check_objs(obj_nums)
        self._check_img(img)
        E._apply_pdl()
        self._plan(refresh=True)
        self._slots[b]["obj"] = obj
        self._reference_pass(b, img, mask)

    def _reference_pass(self, b, img, mask):
        """AOTEngine.add_reference_frame on slot b: encode (B = 1), ID embedding of the mask, LSTT with the frame's own K / V
        as its long-term memory, store into the slot's bank."""
        pl, N = self._pool, self._N
        st = E._cur_stream()
        embs = self._enc(img, st).nhwc
        for src, dst in zip(embs[:3], pl.dec_in):
            ops.eltwise(ops.EW_COPY, src.reshape(-1, src.shape[3]), None, dst[b:b + 1].reshape(-1, dst.shape[3]), stream=st)
        self._copy_mask(b, mask, st)
        self._id_embed(b, 1, st)
        self._lstt(b, 1, embs[-1].reshape(N, self._P.C), st, ref=True)
        self._store(b, 1, st, flags=[1])
        s = self._slots[b]
        s["last_mem_step"] = s["frame_step"]
        s["bank_len"] = min(s["bank_len"] + N, self.long_term_mem_max * N)

    @E._in_precision
    def propagate(self, frames):
        """frames {vid: img [1,3,H,W]} with exactly the open videos: one batched encoder + LSTT pass; every frame step
        advances by one."""
        if not self._slots:
            raise ValueError("no video is open")
        if set(frames) != set(self.videos) or len(frames) != len(self._slots):
            raise ValueError(f"propagate needs a frame for exactly the open videos {sorted(self.videos)}, got "
                             f"{sorted(frames)}")
        n, pl, N = len(self._slots), self._pool, self._N
        for s in self._slots:
            self._check_img(frames[s["vid"]])
        st = E._cur_stream()
        for b, s in enumerate(self._slots):
            pl.frames[b:b + 1].copy_(frames[s["vid"]])
        embs = self._enc(pl.frames[:n], st).nhwc
        splits = self._splits(n * N, max(max(s["bank_len"] for s in self._slots), 1))

        def body():
            s2 = E._cur_stream()
            for src, dst in zip(embs[:3], pl.dec_in):
                ops.eltwise(ops.EW_COPY, src.reshape(-1, src.shape[3]), None, dst[:n].reshape(-1, dst.shape[3]), stream=s2)
            self._lstt(0, n, embs[-1].reshape(n * N, self._P.C), s2, ref=False, splits=splits)
        self.graphs.run(("lstt", n, splits) + tuple(t.data_ptr() for t in embs), body)
        for s in self._slots:
            s["frame_step"] += 1

    @E._in_precision
    def decode_current_logits(self, output_size=None):
        """-> {vid: logits [1, 11, h, w]} (output_size None: the stride-4 map, else upsampled to output_size).  The decoder
        over the n videos is one graph keyed on n; each video's logit post-processing (masking the ids above its object
        count, upsampling) follows it as an eager launch, so object counts that change as videos open, close or gain objects
        need no new graph."""
        size = None if output_size is None else (int(output_size[0]), int(output_size[1]))
        lg = self.decode_nhwc()
        st = E._cur_stream()
        h4, w4, NC = lg.shape[1], lg.shape[2], lg.shape[3]
        self._last_lowres, out = [], {}
        for b, s in enumerate(self._slots):
            lo = E._static_buf(self._pool.dec, ("lo", b), (1, NC, h4, w4), lg.device)
            up = None if size is None else E._static_buf(self._pool.dec, ("out", b), (1, NC) + size, lg.device)
            ops.logits_postproc(lg[b:b + 1], lo, up, s["obj"], self._P.align_corners, stream=st)
            self._last_lowres.append(lo)
            out[s["vid"]] = lo if up is None else up
        return out

    @E._in_precision
    def decode_nhwc(self):
        """The decoder over the n open videos -> their raw logits [n, h/4, w/4, 11] (NHWC, slot order, no object-count
        mask): a static buffer the next decode overwrites.  decode_current_logits post-processes it per video."""
        n = len(self._slots)
        return self.graphs.run(("dec", n), lambda: self._decode(n))

    def decode_labels(self, output_size=None):
        """decode_current_logits fused with the argmax of each video's upsampled logits -> {vid: label [1, H, W] int64}."""
        self.decode_current_logits(None)
        size = self._geom if output_size is None else (int(output_size[0]), int(output_size[1]))
        st = E._cur_stream()
        out = {}
        for s, lo in zip(self._slots, self._last_lowres):
            label = torch.empty((1,) + tuple(size), dtype=torch.float32, device=lo.device)
            ops.logits_argmax(lo, label, self._P.align_corners, stream=st)
            out[s["vid"]] = label.long()
        return out

    @E._in_precision
    def update_memory(self, labels, skip_long_term_update=False):
        """labels {vid: label map [1,1,H,W] | [1,H,W]} for exactly the open videos: every video's short-term memory, and
        the long-term bank of each video whose own gap has passed since its last memory frame."""
        if set(labels) != set(self.videos):
            raise ValueError(f"update_memory needs a label map for exactly the open videos {sorted(self.videos)}, got "
                             f"{sorted(labels)}")
        st = E._cur_stream()
        for b, s in enumerate(self._slots):
            self._copy_mask(b, labels[s["vid"]], st)
        self.update_memory_from_masks(skip_long_term_update)

    def mask_rows(self):
        """The open videos' label-map rows [n, H, W] at the network input size (slot order), which update_memory fills and
        update_memory_from_masks reads."""
        return self._pool.mask[:len(self._slots)]

    @E._in_precision
    def update_memory_from_masks(self, skip_long_term_update=False):
        """update_memory on the label maps already in mask_rows() (written on the current stream): every video's
        short-term memory, and the long-term bank of each video whose own gap has passed since its last memory frame."""
        n, pl = len(self._slots), self._pool
        flags = []
        for s in self._slots:
            store = 0
            if s["frame_step"] - s["last_mem_step"] >= s["gap"]:
                store = 0 if skip_long_term_update else 1
                s["last_mem_step"] = s["frame_step"]
            flags.append(store)
        host = torch.tensor(flags, dtype=torch.int32)
        if pl.flags.is_cuda:
            # pinned by the caching host allocator, which keeps the block until the asynchronous copy has run: no host sync
            host = host.pin_memory()
        pl.flags[:n].copy_(host, non_blocking=True)

        def body():
            s2 = E._cur_stream()
            self._id_embed(0, n, s2)
            self._fuse_memories(self._rows(0, n), s2)
            self._store(0, n, s2)
        self.graphs.run(("upd", n), body)
        for s, f in zip(self._slots, flags):
            if f:
                s["bank_len"] = min(s["bank_len"] + self._N, self.long_term_mem_max * self._N)

    def close_video(self, vid):
        """Free the video's slot: the last slot's state moves into it (one device copy per buffer), so the open videos stay
        in slots 0 .. n - 2."""
        b = self._slot(vid)
        last = len(self._slots) - 1
        if b != last:
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
            self._slots[b] = self._slots[last]
        self._slots.pop()

    @property
    def long_term_memories(self):
        """{vid: per layer [K, V] fp32 live rows of the video's bank in slot order} (see AOTEngine.long_term_memories)."""
        pl, MN = self._pool, self.long_term_mem_max * self._N
        return {s["vid"]: [[pl.bank_K[li][b * MN:b * MN + s["bank_len"]], pl.bank_V[li][b * MN:b * MN + s["bank_len"]]]
                           for li in range(self._P.L)] for b, s in enumerate(self._slots)}

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
        S, M, C, L = self.max_videos, self.long_term_mem_max, P.C, P.L
        self._enc = E._Encoder(P, geom[0], geom[1])
        with torch.no_grad():
            probe = self._enc(torch.zeros((1, 3) + geom, device=dev), E._cur_stream()).nhwc
        h, w = probe[-1].shape[1], probe[-1].shape[2]
        N = h * w
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        hz = lambda *s: torch.zeros(s, dtype=torch.float16, device=dev)
        pl = type("Pool", (), {})()
        pl.key = key
        pl.frames = torch.zeros((S, 3) + geom, dtype=torch.float32, device=dev)
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
        self._pool, self._N, self._hw, self._geom = pl, N, (h, w), geom

    def _lstt_buffers(self, rows, C, L, dev):
        return E._aot_lstt_buffers(rows, C, L, dev)

    def _splits(self, rows, tk):
        """KV-split count of the batched long-term attention over `rows` query rows and at most tk live keys."""
        return E.lt_splits(rows, self._P.H, tk)

    def _id_embed(self, b, n, st):
        """The ID embedding of slots [b, b + n)'s label maps into their id_emb rows."""
        P, pl, N = self._P, self._pool, self._N
        ops.id_embed_runs_batched(pl.mask[b:b + n], P.id_wp, P.id_b, pl.id_emb[b * N:(b + n) * N], P.C, P.nid, P.id_k,
                                  P.id_stride, P.id_pad, ln_gamma=P.id_norm[0] if P.deaot else None,
                                  ln_beta=P.id_norm[1] if P.deaot else None, stream=st)

    def _fuse_memories(self, a, st):
        E.aot_fuse_memories(self._P, a, a.id_emb, a.st_K, a.st_V, st)

    def _copy_mask(self, b, mask, st):
        m = mask.reshape(mask.shape[-2], mask.shape[-1]) if mask.dim() >= 2 else None
        if m is None or mask.numel() != m.numel() or tuple(m.shape) != self._geom:
            raise ValueError(f"expected a label map of the network input size {self._geom}, got {tuple(mask.shape)}")
        ops.eltwise(ops.EW_COPY, m.float().contiguous(), None, self._pool.mask[b], stream=st)

    def _attention(self, Q, Kp, Vp, kv_stride, n, Tk, Tk_dev, out, splits, st):
        P, N = self._P, self._N
        pl = self._pool
        ops.tc_pack_rows(Q, pl.Qp, 0, div=math.sqrt(P.C // P.H), stream=st)
        exact = E.LT_IMPL == "tc_exact" and self.precision == "fp32"
        part = E._split_partials(pl.part, splits, n * N, P.H, P.C, pl.x.device, cap_rows=self.max_videos * N) \
            if splits > 1 else None
        ops.lt_attention_tc_batched(pl.Qp, N, Kp, Vp, kv_stride, n, N, Tk=Tk, Tk_dev=Tk_dev, O=out, splits=splits,
                                    exact=exact, part=part, stream=st)

    # ------------------------------------------------------------------ batched bodies (rows of slots b .. b + n - 1)
    def _rows(self, b, n):
        """The LSTT workspace of slots [b, b + n): every activation (and per-layer list) sliced to their rows."""
        r = slice(b * self._N, (b + n) * self._N)
        a = types.SimpleNamespace(gn_ws=self._pool.gn_ws)
        for k, t in self._pool.lstt.items():
            setattr(a, k, t[r] if isinstance(t, torch.Tensor) else [None if u is None else u[r] for u in t])
        return a

    def _lstt(self, b, n, proj, st, ref, splits=None):
        """engine.aot_lstt over slots [b, b + n): ref = the reference-frame form, else the propagation form over the
        slots' banks.  Each attention step packs its operands and runs the batched tensor-core kernel."""
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
        """Store slots [b, b + n)'s short-term K / V into their banks where the store flag is set (flags: written here
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
        """engine.fpn_decode over the n open videos (B = n) -> their logits [n, h/4, w/4, 11] (NHWC)."""
        pl = self._pool
        x4, x8, x16 = (t[:n] for t in pl.dec_in)
        return E.fpn_decode(self._P, pl.cat[:n * self._N].view(n, *self._hw, -1), x4, x8, x16, pl.dec, pl.gn_ws,
                            E._cur_stream())


class DeAOTMultiVideoInferEngine(MultiVideoInferEngine):
    """DeAOTMultiVideoInferEngine(aot_model, max_videos=S, long_term_mem_max=M, gpu_id=0, long_term_mem_gap=None,
    short_term_mem_skip=1, precision=None, long_term_mem_policy=None).

    MultiVideoInferEngine for the DeAOT models: the same protocol, with per video the semantics of
    DeAOTInferEngine(long_term_mem_max=M) with at most 10 objects.  Each frame's gated propagation (engine.deaot_lstt) runs
    over the n open videos through the batched fused long-term / self-attention and the batched gated local attention."""

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
        """engine.deaot_lstt over slots [b, b + n): ref = the reference-frame form, else the propagation form over the
        slots' banks.  Each attention step packs its operands and runs the batched fused kernel."""
        P, pl, N = self._P, self._pool, self._N
        a = self._rows(b, n)
        MN = self.long_term_mem_max * N
        exact = self.precision == "fp32"

        def attend(Q, Kp, Vp, kv_stride, Tk, Tk_dev, out, splits, st):
            ops.tc_pack_rows(Q, pl.Qp, 0, div=math.sqrt(Q.shape[1]), stream=st)      # Q / T (attention.py:672)
            part = E._split_partials(pl.part, splits, n * N, 1, out.shape[1], out.device, cap_rows=self.max_videos * N) \
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
