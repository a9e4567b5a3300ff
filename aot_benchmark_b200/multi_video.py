"""Several independent videos propagated through one engine, one batched encoder + LSTT + decoder pass per frame.

Per video, the semantics are those of AOTInferEngine(long_term_mem_max=M) with at most 10 objects: each video has its own
frame step, object count, long-term gap, short-term memory and bounded long-term bank (the first memory frame pinned, the
newest M - 1 in a ring).  Videos open and close independently; the n open videos always occupy slots 0 .. n - 1 of a pool
allocated once per (geometry, S, M), so every launch covers exactly n videos and every captured graph is keyed on n (DESIGN
§3.9).
"""
from __future__ import annotations

import math

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
        if cfg.MODEL_VOS == "deaot":
            raise NotImplementedError("MultiVideoInferEngine runs the AOT models; DeAOT's gated propagation has no batched "
                                      "entry points yet")
        policy = getattr(cfg, "TEST_LONG_TERM_MEM_POLICY", None) if long_term_mem_policy is None else long_term_mem_policy
        if policy is not None and policy not in E.MEM_POLICIES:
            raise ValueError(f"long_term_mem_policy must be one of {E.MEM_POLICIES}, got {policy!r}")
        if policy not in (None, "fifo"):
            raise NotImplementedError("MultiVideoInferEngine keeps FIFO banks; long_term_mem_policy='usage' counts attention "
                                      "mass per video, which the batched attention does not")
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
        if short_term_mem_skip != 1:
            raise NotImplementedError("MultiVideoInferEngine keeps one short-term memory frame per video "
                                      "(short_term_mem_skip=1)")
        if int(max_videos) != max_videos or max_videos < 1:
            raise ValueError(f"max_videos must be a positive integer, got {max_videos}")
        M = E._resolve_mem_max(aot_model, long_term_mem_max)
        if M is None:
            raise ValueError("MultiVideoInferEngine pools a bounded long-term bank per video: give long_term_mem_max (or "
                             "cfg.TEST_LONG_TERM_MEM_MAX)")
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

    # ------------------------------------------------------------------ protocol
    def enable_kv_sharding(self, rank, world, group=None):
        raise NotImplementedError("MultiVideoInferEngine pools bounded banks on one GPU; a bank sharded over GPUs is not "
                                  "built for it")

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
            raise NotImplementedError(f"MultiVideoInferEngine propagates at most {self.max_obj_num} objects per video (one "
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
        P = self._P
        ops.id_embed_runs_batched(pl.mask[b:b + 1], P.id_wp, P.id_b, pl.id_emb[b * N:(b + 1) * N], P.C, P.nid, P.id_k,
                                  P.id_stride, P.id_pad, stream=st)
        self._lstt(b, 1, embs[-1].reshape(N, P.C), st, ref=True)
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
        splits = E.lt_splits(n * N, self._P.H, max(max(s["bank_len"] for s in self._slots), 1))

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
        n = len(self._slots)
        size = None if output_size is None else (int(output_size[0]), int(output_size[1]))
        lg = self.graphs.run(("dec", n), lambda: self._decode(n))
        st = E._cur_stream()
        h4, w4, NC = lg.shape[1], lg.shape[2], lg.shape[3]
        self._last_lowres, out = [], {}
        for b, s in enumerate(self._slots):
            lo = self._dbuf(("lo", b), (1, NC, h4, w4))
            up = None if size is None else self._dbuf(("out", b), (1, NC) + size)
            ops.logits_postproc(lg[b:b + 1], lo, up, s["obj"], self._P.align_corners, stream=st)
            self._last_lowres.append(lo)
            out[s["vid"]] = lo if up is None else up
        return out

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
        n, pl = len(self._slots), self._pool
        st = E._cur_stream()
        flags = []
        for b, s in enumerate(self._slots):
            store = 0
            if s["frame_step"] - s["last_mem_step"] >= s["gap"]:
                store = 0 if skip_long_term_update else 1
                s["last_mem_step"] = s["frame_step"]
            flags.append(store)
            self._copy_mask(b, labels[s["vid"]], st)
        host = torch.tensor(flags, dtype=torch.int32)
        if pl.flags.is_cuda:
            # pinned by the caching host allocator, which keeps the block until the asynchronous copy has run: no host sync
            host = host.pin_memory()
        pl.flags[:n].copy_(host, non_blocking=True)

        def body():
            s2 = E._cur_stream()
            P, N = self._P, self._N
            ops.id_embed_runs_batched(pl.mask[:n], P.id_wp, P.id_b, pl.id_emb[:n * N], P.C, P.nid, P.id_k, P.id_stride,
                                      P.id_pad, stream=s2)
            self._fuse(0, n, s2)
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
                for t in (pl.st_K[li], pl.st_V[li], pl.curr_Q[li], pl.curr_V[li]):
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
            if P.C != 256 or P.C // P.H != 32:
                raise NotImplementedError(f"MultiVideoInferEngine runs the 8 x 32 attention heads of the AOT models with "
                                          f"256 channels, got {P.H} heads of {P.C // P.H}")
            if self._P is not None and P is not self._P:
                self.graphs.clear()
            self._P = P
        return self._P

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
        pl.id_emb, pl.x, pl.ln, pl.ln_pos, pl.v, pl.tmp = (f(R, C) for _ in range(6))
        pl.qk, pl.core = f(R, 2 * C), f(R, 2 * C)
        pl.ff, pl.ff2 = f(R, 4 * C), f(R, 4 * C)
        pl.cat = f(R, (L + 1) * C)
        pl.curr_Q, pl.curr_V = [f(R, C) for _ in range(L)], [f(R, C) for _ in range(L)]
        pl.st_K, pl.st_V = [f(R, C) for _ in range(L)], [f(R, C) for _ in range(L)]
        pl.bank_K, pl.bank_V = [f(S * M * N, C) for _ in range(L)], [f(S * M * N, C) for _ in range(L)]
        pl.bank_Kp, pl.bank_Vp = [hz(P.H, S * M * N, 64) for _ in range(L)], [hz(P.H, S * M * N, 64) for _ in range(L)]
        pl.Qp, pl.saKp, pl.saVp = hz(P.H, R, 64), hz(P.H, R, 64), hz(P.H, R, 64)
        pl.part = {}
        pl.gn_ws = ops.groupnorm_workspace(S, 32, dev)
        pl.pos = E._pos_emb_sine(h, w, npf=C // 2).to(dev).repeat(S, 1).contiguous()
        pl.dec = {}
        self._pool, self._N, self._hw, self._geom = pl, N, (h, w), geom

    def _copy_mask(self, b, mask, st):
        m = mask.reshape(mask.shape[-2], mask.shape[-1]) if mask.dim() >= 2 else None
        if m is None or mask.numel() != m.numel() or tuple(m.shape) != self._geom:
            raise ValueError(f"expected a label map of the network input size {self._geom}, got {tuple(mask.shape)}")
        ops.eltwise(ops.EW_COPY, m.float().contiguous(), None, self._pool.mask[b], stream=st)

    def _parts(self, splits, rows):
        """Split-KV partials of `splits` splits over `rows` query rows: views of one allocation per split count, so a graph
        body for any n reads memory that lives as long as the pool."""
        pl, H, C = self._pool, self._P.H, self._P.C
        flat = pl.part.get(splits)
        if flat is None:
            R = self.max_videos * self._N
            flat = pl.part[splits] = torch.empty(splits * R * (C + 2 * H), dtype=torch.float32, device=pl.x.device)
        nO, nM = splits * rows * C, splits * H * rows
        return (flat[:nO].view(splits, rows, C), flat[nO:nO + nM].view(splits, H, rows),
                flat[nO + nM:nO + 2 * nM].view(splits, H, rows))

    def _attention(self, Q, Kp, Vp, kv_stride, n, Tk, Tk_dev, out, splits, st):
        P, N = self._P, self._N
        pl = self._pool
        ops.tc_pack_rows(Q, pl.Qp, 0, div=math.sqrt(P.C // P.H), stream=st)
        exact = E.LT_IMPL == "tc_exact" and self.precision == "fp32"
        ops.lt_attention_tc_batched(pl.Qp, N, Kp, Vp, kv_stride, n, N, Tk=Tk, Tk_dev=Tk_dev, O=out, splits=splits,
                                    exact=exact, part=self._parts(splits, n * N) if splits > 1 else None, stream=st)

    # ------------------------------------------------------------------ batched bodies (rows of slots b .. b + n - 1)
    def _lstt(self, b, n, proj, st, ref, splits=None):
        """AOTEngine._lstt_forward over slots [b, b + n): ref = the reference-frame form (the frame's own K / V as long-term
        memory, short-term memory written), else the propagation form over the slots' banks."""
        P, pl, N = self._P, self._pool, self._N
        C, H = P.C, P.H
        h, w = self._hw
        r = slice(b * N, (b + n) * N)
        R = n * N
        x, ln, ln_pos, qk, v, core, tmp = (t[r] for t in (pl.x, pl.ln, pl.ln_pos, pl.qk, pl.v, pl.core, pl.tmp))
        ff, ff2, cat = pl.ff[r], pl.ff2[r], pl.cat[r]
        ops.eltwise(ops.EW_COPY, proj, None, x, stream=st)
        ops.eltwise(ops.EW_COPY, proj, None, cat[:, :C], stream=st)
        sa_splits = E.lt_splits(R, H, N)
        for li in range(P.L):
            Lw = P.layers[li]
            stK, stV = pl.st_K[li][r], pl.st_V[li][r]
            ops.layernorm(x, Lw.norm1[0], Lw.norm1[1], ln, add=pl.pos[:R], out2=ln_pos, stream=st)
            ops.linear(ln_pos, Lw.sa_qk_w, Lw.sa_qk_b, qk, stream=st)
            ops.linear(ln, Lw.sa_v_w, Lw.sa_v_b, v, stream=st)
            ops.tc_pack_rows(qk[:, C:], pl.saKp, 0, stream=st)
            ops.tc_pack_rows(v, pl.saVp, 0, stream=st)
            self._attention(qk[:, :C], pl.saKp, pl.saVp, N, n, N, None, core[:, :C], sa_splits, st)
            ops.linear(core[:, :C], Lw.sa_proj_w, Lw.sa_proj_b, x, res=x, stream=st)
            cQ, cV = pl.curr_Q[li][r], pl.curr_V[li][r]
            ops.layernorm(x, Lw.norm2[0], Lw.norm2[1], cV, stream=st)
            ops.linear(cV, Lw.linQ_w, Lw.linQ_b, cQ, stream=st)
            if ref:
                ops.eltwise(ops.EW_ADD, cV, pl.id_emb[r], tmp, stream=st)
                ops.linear(tmp, Lw.linV_w, Lw.linV_b, stV, stream=st)
                ops.eltwise(ops.EW_COPY, cQ, None, stK, stream=st)
                ops.tc_pack_rows(stK, pl.saKp, 0, stream=st)
                ops.tc_pack_rows(stV, pl.saVp, 0, stream=st)
                self._attention(cQ, pl.saKp, pl.saVp, N, n, N, None, core[:, :C], sa_splits, st)
            else:
                MN = self.long_term_mem_max * N
                self._attention(cQ, pl.bank_Kp[li], pl.bank_Vp[li], MN, n, 0, pl.tk[b:b + n], core[:, :C], splits, st)
            ops.local_attention_tc_batched(cQ, stK, stV, Lw.relk_w, Lw.relk_b, Lw.relv_t, core[:, C:], h, w, H, n, stream=st)
            ops.linear(core, Lw.lst_proj_w, Lw.lst_proj_b, x, res=x, stream=st)
            ops.layernorm(x, Lw.norm3[0], Lw.norm3[1], ln, stream=st)
            ops.linear(ln, Lw.lin1_w, Lw.lin1_b, ff, stream=st)
            ops.groupnorm(ff.view(n, N, 4 * C), Lw.gn[0], Lw.gn[1], ff.view(n, N, 4 * C), 32, E.A_GELU, pl.gn_ws, stream=st)
            ops.dwconv(ff.view(n, h, w, 4 * C), Lw.dw_w, None, ff2.view(n, h, w, 4 * C), K=5, pad=2, stream=st)
            ops.linear(ff2, Lw.lin2_w, Lw.lin2_b, x, res=x, stream=st)
            ops.layernorm(x, Lw.dec_norm[0], Lw.dec_norm[1], cat[:, (li + 1) * C:(li + 2) * C], stream=st)

    def _fuse(self, b, n, st):
        """AOTEngine._fuse_memories over slots [b, b + n): K = curr_K, V = linear_V(curr_V + id)."""
        P, pl, N = self._P, self._pool, self._N
        r = slice(b * N, (b + n) * N)
        for li in range(P.L):
            Lw = P.layers[li]
            ops.eltwise(ops.EW_ADD, pl.curr_V[li][r], pl.id_emb[r], pl.tmp[r], stream=st)
            ops.linear(pl.tmp[r], Lw.linV_w, Lw.linV_b, pl.st_V[li][r], stream=st)
            ops.eltwise(ops.EW_COPY, pl.curr_Q[li][r], None, pl.st_K[li][r], stream=st)

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

    def _dbuf(self, key, shape):
        t = self._pool.dec.get((key, shape))
        if t is None:
            t = self._pool.dec[(key, shape)] = torch.empty(shape, dtype=torch.float32, device=self._pool.x.device)
        return t

    def _decode(self, n):
        """AOTEngine._decode over the n open videos (B = n) -> their logits [n, h/4, w/4, 11] (NHWC)."""
        P, pl = self._P, self._pool
        D = P.dec
        ac = P.align_corners
        st = E._cur_stream()
        x4, x8, x16 = (t[:n] for t in pl.dec_in)
        h, w = self._hw
        gws = pl.gn_ws

        def conv_gn(x, blk, key, k, pad):
            o = self._dbuf(key, (n, x.shape[1], x.shape[2], blk.cout))
            ops.conv2d(x, blk.w, blk.b, o, KH=k, KW=k, pad=pad, stream=st)
            ov = o.view(n, -1, blk.cout)
            ops.groupnorm(ov, blk.gn[0], blk.gn[1], ov, 8, E.A_RELU, gws, stream=st)
            return o

        x = conv_gn(pl.cat[:n * self._N].view(n, h, w, -1), D.conv_in, "in", 1, 0)
        a = self._dbuf("a16", (n, h, w, D.adapter_16x.cout))
        ops.conv2d(x16, D.adapter_16x.w, D.adapter_16x.b, a, res=x, stream=st)
        x = conv_gn(a, D.conv_16x, "c16", 3, 1)
        for xs, tag, ad, cv in ((x8, "8", D.adapter_8x, D.conv_8x), (x4, "4", D.adapter_4x, D.conv_4x)):
            up = self._dbuf("up" + tag, (n, xs.shape[1], xs.shape[2], x.shape[3]))
            ops.bilinear(x, up, ac, stream=st)
            a = self._dbuf("a" + tag, (n, xs.shape[1], xs.shape[2], ad.cout))
            ops.conv2d(xs, ad.w, ad.b, a, res=up, stream=st)
            x = conv_gn(a, cv, "c" + tag, 3, 1)
        lg = self._dbuf("logit", (n, x.shape[1], x.shape[2], D.conv_out.cout))
        ops.conv2d(x, D.conv_out.w, D.conv_out.b, lg, stream=st)
        return lg
