"""Drop-in eval engines: the reference's protocol, executed by the sm_90a kernels.

Mirrors networks/engines/aot_engine.py (AOTEngine :13-482, AOTInferEngine :485-635) and
networks/engines/deaot_engine.py (DeAOTEngine :9-56, DeAOTInferEngine :59-94): same class and
method names, arguments, state attributes and error behaviour, so networks/managers/evaluator.py
and tools/demo.py drive it unedited.  Differences are internal:

* activations live in NHWC / token-major fp32 buffers allocated once per video;
* the long-term memory is a pre-allocated append buffer (bank) instead of torch.cat'ed tensors
  (new frames are appended, not prepended -- attention is permutation invariant over keys); with long_term_mem_max = M it
  holds the first memory frame and the newest M - 1 in a ring (with long_term_mem_policy="usage", a full bank overwrites
  the least-attended unpinned frame instead of the oldest), so a long clip runs at constant cost;
* every FLOP of the per-frame path runs in libaotb200.so; there is no eager fallback and the
  engines refuse CPU tensors.

Training (AOTEngine.forward, aot_engine.py:33-108) is a "next" row of SURVEY 8(f) and raises.
"""
from __future__ import annotations

import contextlib
import functools
import math

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .plan import get_plan

A_NONE, A_RELU, A_GELU, A_SILU, A_RELU6 = ops.ACT_NONE, ops.ACT_RELU, ops.ACT_GELU, ops.ACT_SILU, ops.ACT_RELU6
A_HSWISH = ops.ACT_HSWISH

# bench.py hook: when set to a list, every long-term attention launch appends
# (start_event, end_event, algorithmic_flops) so the roofline is measured live, per launch.
LT_PROBE = None
# long-term attention implementation for the AOT head shape (8 x 32):
#   "tc_exact" wgmma kernel, split-fp16 operands, fp32-faithful   (lt_attn_tc.cu)
#   "tc_fast"  wgmma kernel, single fp16 pass for Q K^T and P
#   "simt"     fp32 CUDA-core flash kernel                          (attention_simt.cu)
import os as _os
LT_IMPL = _os.environ.get("AOTB_LT_IMPL", "tc_exact")
LOCAL_IMPL = _os.environ.get("AOTB_LOCAL_IMPL", "tc")   # "tc" (tensor cores, AOT heads) | "tile" (halo in smem) | "warp" (generic)
# DeAOT long-term attention (1 head, d_qk 128, d_v 1024): "tc" = fused wgmma flash kernel (gp_attn_tc.cu, default) |
# "gemm" = tensor-core GEMM (Q K^T) -> row softmax -> tensor-core GEMM (P V) over split-fp16 operand copies of the bank
# (deaot_lt.cu) | "simt" = fp32 CUDA-core flash kernel
DEAOT_LT = _os.environ.get("AOTB_DEAOT_LT", "tc")
# exchange step of the sharded long-term bank (BASELINE configs[3]): "nccl" = three all-gathers of the (m, l, O) partials +
# local merge; "p2p" = the partials live in a torch symmetric-memory allocation and every rank's merge kernel reads its
# peers' partials in place over NVLink (aotb_attn_merge_peers_f32) behind one device-side barrier -- no NCCL on the data
# path.  "p2p" was written without multi-GPU access (logic checked on CPU with an in-process stand-in for the allocator).
SHARD_XCHG = _os.environ.get("AOTB_SHARD_XCHG", "nccl")
SHARD_SMAX = 16          # split capacity of the symmetric partial buffers
SUB_ENGINE_STREAMS = _os.environ.get("AOTB_SUB_ENGINE_STREAMS", "1") == "1"   # > 10 objects: sub-engines on concurrent streams
SHARD_GRAPHS = _os.environ.get("AOTB_SHARD_GRAPHS", "1") == "1"   # capture the LSTT call (incl. the exchange) in sharded mode


def _symm_alloc(numel, device, group):
    """-> (handle, rank -> flat fp32 view of that rank's buffer) for a symmetric-memory allocation of `numel` floats."""
    import torch.distributed as dist
    import torch.distributed._symmetric_memory as symm_mem
    t = symm_mem.empty(numel, dtype=torch.float32, device=device)
    hdl = symm_mem.rendezvous(t, group if group is not None else dist.group.WORLD)
    return hdl, (lambda r, sizes, off: hdl.get_buffer(r, sizes, torch.float32, off))


GEMM_GROW_FRAMES = int(_os.environ.get("AOTB_GEMM_GROW_FRAMES", "8"))   # bank growth step of the GEMM path (memory frames)
_LT_NAMES = {"simt": "attn_f32_kernel<32,32> (fp32 SIMT flash attention)",
             "tc_exact": "attn_tc_kernel<1,1> (wgmma fp16x2 exact: 6+8 MMAs per 64-key tile)",
             "tc_fast": "attn_tc_kernel<1,1> (wgmma fp16 fast: 2+4 MMAs per 64-key tile)"}
_DEAOT_LT_NAMES = {"simt": "attn_f32_kernel<128,256> (fp32 SIMT flash attention, DeAOT 1 x 128 / 1024 head)",
                   "gemm": "conv_tc_kernel (Q K^T) -> row_softmax_kernel -> conv_tc_kernel (P V): wgmma GEMMs over split-fp16 "
                           "copies of the bank (deaot_lt.cu)",
                   "tc": "attn_tc_kernel<4,2> (fused wgmma flash attention, 128 queries x 64 value channels per CTA)"}


def deaot_lt_kernel_name():
    """The DeAOT long-term attention implementation actually in use (bench.py's roofline entry names it)."""
    return _DEAOT_LT_NAMES.get(DEAOT_LT, DEAOT_LT)


LT_KERNEL_NAME = _LT_NAMES.get(LT_IMPL, LT_IMPL) + (f", layout '{ops.LT_VARIANT}'" if LT_IMPL.startswith("tc") else "")


# Whole-call CUDA graphs (encoder / LSTT / decoder / memory update are each captured once per video geometry and
# replayed; the live key count and the bank append offset are read from a device counter inside the kernels).
USE_GRAPHS = _os.environ.get("AOTB_GRAPHS", "1") == "1"
# programmatic dependent launch: kernel N+1's prologue (barrier init, descriptor prefetch) overlaps
# kernel N's tail; every kernel waits (griddepcontrol.wait) before reading its inputs
USE_PDL = _os.environ.get("AOTB_PDL", "1") == "1"     # programmatic dependent launch
CONV_TILING = _os.environ.get("AOTB_CONV_TILING", "model")   # "model" (fitted cost model) | "narrow" (old heuristic)
_CONV_TILING_MASK = {"model": 0, "narrow": 1}


def _apply_pdl():
    """Push the launch-policy knobs into the library (cheap; called at the start of every clip)."""
    from ._lib import lib, check
    lib().aotb_set_pdl(1 if USE_PDL else 0)
    check(lib().aotb_set_conv_tiling(_CONV_TILING_MASK[CONV_TILING]), "aotb_set_conv_tiling")
BANK_INIT_FRAMES = int(_os.environ.get("AOTB_BANK_FRAMES", "24"))   # initial long-term bank capacity (memory frames)
# offline_encoder: frames per batched encoder pass (one captured graph per chunk size; DESIGN §8 has the sweep it is chosen from)
OFFLINE_ENC_CHUNK = 16


def _resolve_mem_max(aot_model, long_term_mem_max):
    """The bound M of the long-term bank in memory frames: the keyword, else cfg.TEST_LONG_TERM_MEM_MAX, else None (unbounded)."""
    m = getattr(aot_model.cfg, "TEST_LONG_TERM_MEM_MAX", None) if long_term_mem_max is None else long_term_mem_max
    if m is None:
        return None
    if int(m) != m or m < 2:
        raise ValueError(f"long_term_mem_max must be an integer >= 2 (the first memory frame and at least one recent one), got {m}")
    return int(m)


MEM_POLICIES = ("fifo", "usage")
USAGE_MAX_SLOTS = 32          # aotb_attn_merge_usage_f32 counts at most 32 memory slots


def _resolve_mem_policy(aot_model, policy, mem_max):
    """The eviction policy of the bounded bank: the keyword, else cfg.TEST_LONG_TERM_MEM_POLICY, else "fifo".  "fifo" overwrites
    the oldest unpinned memory frame; "usage" the unpinned frame the propagated frames attended to least on average since it
    was stored (DESIGN §2).  Usage mode counts attention mass in the tensor-core long-term attention's slot-split launch, so
    it refuses the knobs that select another kernel."""
    p = getattr(aot_model.cfg, "TEST_LONG_TERM_MEM_POLICY", None) if policy is None else policy
    if p is None:
        return "fifo"
    if p not in MEM_POLICIES:
        raise ValueError(f"long_term_mem_policy must be one of {MEM_POLICIES}, got {p!r}")
    if p == "usage":
        if mem_max is None:
            raise ValueError("long_term_mem_policy='usage' chooses which frame a full bounded bank evicts; it needs "
                             "long_term_mem_max (or cfg.TEST_LONG_TERM_MEM_MAX)")
        if mem_max > USAGE_MAX_SLOTS:
            raise NotImplementedError(f"long_term_mem_policy='usage' counts at most {USAGE_MAX_SLOTS} memory slots, "
                                      f"got long_term_mem_max={mem_max}")
        if aot_model.cfg.MODEL_VOS == "deaot":
            if DEAOT_LT != "tc":
                raise NotImplementedError(f"long_term_mem_policy='usage' counts attention mass in DeAOT's fused tensor-core "
                                          f"attention; AOTB_DEAOT_LT={DEAOT_LT} selects another path")
        elif LT_IMPL == "simt":
            raise NotImplementedError("long_term_mem_policy='usage' counts attention mass in the tensor-core long-term "
                                      "attention; AOTB_LT_IMPL=simt selects the fp32 CUDA-core kernel")
        elif ops.LT_VARIANT != "tile":
            raise NotImplementedError(f"long_term_mem_policy='usage' runs the default 'tile' layout of the tensor-core "
                                      f"long-term attention; AOTB_LT_VARIANT={ops.LT_VARIANT} selects another")
    return p


def _resolve_precision(aot_model, precision):
    """The engine's precision: the keyword, else cfg.TEST_PRECISION, else "fp32".  "fp16" runs every tensor-core conv and
    linear with operands rounded once to fp16 and the tensor-core attention without its exact (lo) terms; it does not
    follow torch.is_autocast_enabled()."""
    p = getattr(aot_model.cfg, "TEST_PRECISION", None) if precision is None else precision
    if p is None:
        return "fp32"
    if p not in ops.PRECISIONS:
        raise ValueError(f"precision must be one of {ops.PRECISIONS}, got {p!r}")
    if p == "fp16":
        # the fp16 mode is built from the tensor-core kernels only; these knobs select fp32 CUDA-core or split-GEMM paths
        if ops.CONV_IMPL == "simt":
            raise NotImplementedError("precision='fp16' runs the tensor-core conv; AOTB_CONV_IMPL=simt selects the fp32 "
                                      "CUDA-core conv")
        if LT_IMPL == "simt":
            raise NotImplementedError("precision='fp16' runs the tensor-core long-term attention; AOTB_LT_IMPL=simt selects "
                                      "the fp32 CUDA-core kernel")
        if aot_model.cfg.MODEL_VOS == "deaot" and DEAOT_LT in ("gemm", "simt"):
            raise NotImplementedError(f"precision='fp16' runs DeAOT's attention on the fused tensor-core kernel; "
                                      f"AOTB_DEAOT_LT={DEAOT_LT} selects another path")
    return p


def _in_precision(fn):
    """Run an engine method with the tensor-core conv / linear launches it issues (graph captures included) in the
    engine's precision."""
    @functools.wraps(fn)
    def wrapper(self, *args, **kwargs):
        with ops.precision(self.precision):
            return fn(self, *args, **kwargs)
    return wrapper


REPLAYED_KERNELS = [0]      # kernels launched through graph replays (bench.py adds this to the library's eager count)


class GraphCache:
    """key -> [eager_runs, CUDAGraph | None, result, kernels_in_graph]; first call runs eagerly (warm-up: lazy module
    loads, cudaFuncSetAttribute, buffer allocation), second call is captured, later calls replay."""

    def __init__(self):
        self.slots = {}

    def clear(self):
        self.slots.clear()

    def run(self, key, fn, enabled=True):
        if not (enabled and USE_GRAPHS and LT_PROBE is None):
            return fn()
        slot = self.slots.get(key)
        if slot is None:
            slot = self.slots[key] = [0, None, None]
        if slot[1] is not None:
            slot[1].replay()
            REPLAYED_KERNELS[0] += slot[3]
            return slot[2]
        if slot[0] < 1:
            slot[0] += 1
            return fn()
        from ._lib import lib
        n0 = lib().aotb_launch_count()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = fn()
        n_kernels = int(lib().aotb_launch_count() - n0)     # kernels recorded into this graph
        g.replay()                     # capture records only; replay produces this call's results
        slot[1], slot[2] = g, out
        slot.append(n_kernels)
        return out


def _cur_stream():
    return torch.cuda.current_stream().cuda_stream


def fork_join(owner, items, fn):
    """fn(index, item) for every item: item 0 on the current stream, the others concurrently on side streams owned by `owner`
    (created once, kept across calls), forked from and joined to the current stream.  fn may fork again: a nested call forks
    from the side stream it runs on, onto its own owner's streams.  Sequential on the current stream for one item or with
    AOTB_SUB_ENGINE_STREAMS=0."""
    if len(items) == 1 or not SUB_ENGINE_STREAMS:
        return [fn(i, x) for i, x in enumerate(items)]
    cur = torch.cuda.current_stream()
    side = getattr(owner, "_side_streams", [])
    while len(side) < len(items) - 1:
        side.append(torch.cuda.Stream())
    owner._side_streams = side
    side = side[: len(items) - 1]
    for s in side:
        s.wait_stream(cur)                      # fork: everything queued so far (shared encoding, masks) is visible
    outs = [None] * len(items)
    for i in range(1, len(items)):
        with torch.cuda.stream(side[i - 1]):
            outs[i] = fn(i, items[i])
    outs[0] = fn(0, items[0])
    for s in side:
        cur.wait_stream(s)                      # join
    return outs


# CTAs per SM of the tensor-core attention's "tile" layout: its kernel is register-bounded for two (attn_tc_min_blocks in
# csrc/attn_tc.cuh) and asks for the shared-memory carveout that holds two; the "groups" / "ahead" layouts keep one.
# tests/test_gpu_lt_occupancy.py checks that the device keeps this many resident (aotb_lt_attn_tc_occupancy).
LT_TILE_CTAS_PER_SM = 2


def lt_splits(n_queries, heads, tk, sms=132, variant=None):
    """KV-split count for the tensor-core kernel: fill whole waves of CTA slots while keeping >= 2 x 128 keys per split.
    One CTA = 128 queries x 1 head x 1 split at LT_TILE_CTAS_PER_SM CTAs per SM ("tile" layout) or one ("groups" / "ahead"
    layouts), or 64 queries x 1 head x 1 split at two CTAs per SM ("pair" layout)."""
    v = ops.LT_VARIANT if variant is None else variant
    if v == "pair":
        qrows, slots = 64, 2 * sms
    else:
        qrows, slots = 128, (LT_TILE_CTAS_PER_SM if v == "tile" else 1) * sms
    base = ((n_queries + qrows - 1) // qrows) * heads
    tiles = (tk + 127) // 128
    effs = []
    for s in range(1, 17):
        if s > 1 and tiles < 2 * s:
            break
        ctas = base * s
        effs.append((s, ctas / (((ctas + slots - 1) // slots) * slots)))
    top = max(e for _, e in effs)
    return next(s for s, e in effs if e >= top - 0.05)     # fewest splits within 5 % of the best wave fill


def _pos_emb_sine(h, w, npf=128):
    """networks/layers/position.py:49-74 (normalize=True, scale=2*pi, T=1e4), as a host-computed
    constant table [h*w, 2*npf] (computed once per video, aot_engine.py:225-228)."""
    y = torch.arange(h, dtype=torch.float32).view(h, 1).expand(h, w)
    x = torch.arange(w, dtype=torch.float32).view(1, w).expand(h, w)
    eps = 1e-6
    y = y / (y[-1:, :] + eps) * (2 * math.pi)
    x = x / (x[:, -1:] + eps) * (2 * math.pi)
    dim_t = torch.arange(npf, dtype=torch.float32)
    dim_t = 10000 ** (2 * (dim_t // 2) / npf)
    px = x[:, :, None] / dim_t
    py = y[:, :, None] / dim_t
    px = torch.stack((px[..., 0::2].sin(), px[..., 1::2].cos()), dim=3).flatten(2)
    py = torch.stack((py[..., 0::2].sin(), py[..., 1::2].cos()), dim=3).flatten(2)
    return torch.cat((py, px), dim=2).reshape(h * w, 2 * npf).contiguous()


class EncEmbs(list):
    """``curr_enc_embs``: list of NCHW feature views [4x, 8x, 16x, 16x-projected] like the reference
    (aot.py:81-84) plus the NHWC tensors the kernels use (``.nhwc``)."""
    nhwc = None


# =====================================================================================
# image encoder (shared by all sub-engines of an infer engine)
# =====================================================================================
class _Encoder:
    """The image encoder + projection over B frames at once ([B,3,H,W] -> four NHWC [B,h,w,c] maps).  Each batch size has
    its own activation buffers and its own captured graph (one per plan, H, W and B), so alternating B = 1 frames and
    B-frame chunks never re-allocates what a graph points at."""

    def __init__(self, plan, H, W):
        self.plan = plan
        self.H, self.W = H, W
        dev = plan.device
        self.bufs = {}
        self.dev = dev
        self.B = 1
        self._per_b = {1: (self.bufs, None, None)}      # B -> (buffers, GraphCache, graph key)

    def _buf(self, key, shape):
        b = self.bufs.get(key)
        if b is None or tuple(b.shape) != tuple(shape):
            b = torch.empty(shape, dtype=torch.float32, device=self.dev)
            self.bufs[key] = b
        return b

    def keep_batch_sizes(self, keep):
        """Free the activation buffers and captured graph of every batch size not in `keep`; the next call with such a size
        starts over (eager, then captured)."""
        self._per_b[self.B] = (self.bufs, getattr(self, "graphs", None), getattr(self, "_gkey", None))
        drop = [b for b in self._per_b if b not in keep]
        if any(self._per_b[b][1] is not None and self._per_b[b][1].slots for b in drop):
            torch.cuda.current_stream().synchronize()      # no replay of a dropped graph is still reading its buffers
        for b in drop:
            del self._per_b[b]
        if self.B not in keep:
            self.bufs, self.graphs, self._gkey = self._per_b.setdefault(1, ({}, None, None))
            self.B = 1

    def batch_sizes(self):
        """The batch sizes whose buffers (and graph) this encoder holds."""
        return sorted(set(self._per_b) | {self.B})

    def _vec(self, key, n):
        """A per-image vector of n values: [n] for one frame (the one-image form), [B, n] for a batch."""
        return self._buf(key, (n,) if self.B == 1 else (self.B, n))

    def _reduce_ws(self, key, C):
        """Workspace of the deterministic multi-CTA reductions (split attention, squeeze-excite): zero-filled once (launch
        counters), kept for the encoder's lifetime."""
        ws = self.bufs.get(key)
        if ws is None:
            # the one-frame call keeps its two-argument form (the form every caller of splat_workspace had before batching)
            ws = self.bufs[key] = ops.splat_workspace(C, self.dev) if self.B == 1 else ops.splat_workspace(C, self.dev, self.B)
        return ws

    @staticmethod
    def _osz(n, k, s, p, d=1):
        return (n + 2 * p - d * (k - 1) - 1) // s + 1

    def __call__(self, img, st):
        """img [B,3,H,W] -> EncEmbs of [B, ...] maps (the encoder's own buffers: the next call with the same B overwrites
        them)."""
        P = self.plan
        if img.dim() != 4 or img.shape[0] < 1 or img.shape[1] != 3:
            raise ValueError(f"expected an image tensor [B,3,H,W], got {tuple(img.shape)}")
        if P.encoder_name == "swin_base" and (img.shape[2] % 4 or img.shape[3] % 4):
            # PatchEmbed zero-pads right/bottom to a multiple of the 4x4 patch (swin_transformer.py:476-481)
            img = torch.nn.functional.pad(img, (0, -img.shape[3] % 4, 0, -img.shape[2] % 4))
        B, H, W = img.shape[0], img.shape[2], img.shape[3]
        if B != self.B:
            self._per_b[self.B] = (self.bufs, getattr(self, "graphs", None), getattr(self, "_gkey", None))
            self.bufs, self.graphs, self._gkey = self._per_b.get(B, ({}, None, None))
            self.B = B
        if getattr(self, "_gkey", None) != (id(P), H, W):
            self.graphs = GraphCache()
            self._gkey = (id(P), H, W)
        x = self._buf("in", (B, H, W, 4))
        ops.image_to_nhwc4(img.float(), x, stream=st)        # caller's tensor -> static NHWC4 input (eager)
        nhwc = self.graphs.run("enc", lambda: self._body(x))
        out = EncEmbs(t.permute(0, 3, 1, 2) for t in nhwc)
        out.nhwc = nhwc
        return out

    def _body(self, x):
        P = self.plan
        st = _cur_stream()
        if P.encoder_name in ("resnet50", "resnet101"):
            feats = self._resnet(x, st)
        elif P.encoder_name in ("resnest50", "resnest101"):
            feats = self._resnest(x, st)
        elif P.encoder_name == "swin_base":
            feats = self._swin(x, st)
        elif P.encoder_name == "mobilenetv3":
            feats = self._mobilenetv3(x, st)
        else:
            feats = self._mobilenet(x, st)
        f16 = feats[-1]
        proj = self._buf("proj", (self.B, f16.shape[1], f16.shape[2], P.C))
        ops.conv2d(f16, P.proj.w, P.proj.b, proj, stream=st)
        return [feats[0], feats[1], feats[2], proj]

    def _resnet(self, x, st):
        e = self.plan.enc
        H, W = x.shape[1], x.shape[2]
        h1, w1 = self._osz(H, 7, 2, 3), self._osz(W, 7, 2, 3)
        c1 = self._buf("stem", (self.B, h1, w1, 64))
        ops.conv2d(x, e.stem.w, e.stem.b, c1, KH=7, KW=7, stride=2, pad=3, act=A_RELU, stream=st)
        h, w = self._osz(h1, 3, 2, 1), self._osz(w1, 3, 2, 1)
        cur = self._buf("pool", (self.B, h, w, 64))
        ops.maxpool3x3s2(c1, cur, stream=st)
        feats = []
        for si, blocks in enumerate(e.stages):
            for bi, b in enumerate(blocks):
                ho, wo = self._osz(h, 3, b.stride, 1), self._osz(w, 3, b.stride, 1)
                t1 = self._buf(f"s{si}b{bi}t1", (self.B, h, w, b.c1.cout))
                ops.conv2d(cur, b.c1.w, b.c1.b, t1, act=A_RELU, stream=st)
                t2 = self._buf(f"s{si}b{bi}t2", (self.B, ho, wo, b.c2.cout))
                ops.conv2d(t1, b.c2.w, b.c2.b, t2, KH=3, KW=3, stride=b.stride, pad=1, act=A_RELU, stream=st)
                if b.down is not None:
                    res = self._buf(f"s{si}ds", (self.B, ho, wo, b.down.cout))
                    ops.conv2d(cur, b.down.w, b.down.b, res, stride=b.stride, stream=st)
                else:
                    res = cur
                out = self._buf(f"s{si}o{bi % 2}", (self.B, ho, wo, b.c3.cout))
                ops.conv2d(t2, b.c3.w, b.c3.b, out, res=res, act=A_RELU, stream=st)
                cur, h, w = out, ho, wo
            feats.append(cur)
        return feats

    def _resnest(self, x, st):
        """ResNeSt-50 / ResNeSt-101 (resnest/resnet.py:418-435): deep stem, max-pool, then per bottleneck conv1, the radix-2 grouped 3x3 conv
        as one tensor-core launch per group on channel slices (group g reads channels [g gw/2, (g+1) gw/2) of t1 and writes
        [g gw, (g+1) gw) of t2), the split attention (pixel reduction + fc1 / fc2 / radix softmax in one launch), the
        attention-weighted sum of the two splits (with the avd pool fused in the strided first blocks), the avg_down
        downsample (pool + conv) and conv3 with the residual and ReLU fused: 6 launches per block, 8 in a strided first block."""
        e = self.plan.enc
        H, W = x.shape[1], x.shape[2]
        h, w = self._osz(H, 3, 2, 1), self._osz(W, 3, 2, 1)
        s0 = self._buf("stem0", (self.B, h, w, e.stem[0].cout))
        ops.conv2d(x, e.stem[0].w, e.stem[0].b, s0, KH=3, KW=3, stride=2, pad=1, act=A_RELU, stream=st)
        s1 = self._buf("stem1", (self.B, h, w, e.stem[1].cout))
        ops.conv2d(s0, e.stem[1].w, e.stem[1].b, s1, KH=3, KW=3, pad=1, act=A_RELU, stream=st)
        s2 = self._buf("stem2", (self.B, h, w, e.stem[2].cout))
        ops.conv2d(s1, e.stem[2].w, e.stem[2].b, s2, KH=3, KW=3, pad=1, act=A_RELU, stream=st)
        h, w = self._osz(h, 3, 2, 1), self._osz(w, 3, 2, 1)
        cur = self._buf("pool", (self.B, h, w, s2.shape[3]))
        ops.maxpool3x3s2(s2, cur, stream=st)
        ws = self._reduce_ws("splat_ws", max(b.gw for blocks in e.stages for b in blocks))
        feats = []
        for si, blocks in enumerate(e.stages):
            for bi, b in enumerate(blocks):
                gw, s = b.gw, b.stride
                ho, wo = (ops.pool2d_size(h, 3, s, 1), ops.pool2d_size(w, 3, s, 1)) if s > 1 else (h, w)
                t1 = self._buf(f"s{si}b{bi}t1", (self.B, h, w, gw))
                ops.conv2d(cur, b.c1.w, b.c1.b, t1, act=A_RELU, stream=st)
                t2 = self._buf(f"s{si}b{bi}t2", (self.B, h, w, 2 * gw))
                for g, cg in enumerate(b.groups):
                    ops.conv2d(t1[..., g * gw // 2:(g + 1) * gw // 2], cg.w, cg.b, t2[..., g * gw:(g + 1) * gw], KH=3, KW=3,
                               pad=1, act=A_RELU, stream=st)
                att = self._vec(f"s{si}b{bi}att", 2 * gw)
                ops.splat_attention(t2, b.fc1_w, b.fc1_b, b.fc2_w, b.fc2_b, att, ws, stream=st)
                comb = self._buf(f"s{si}b{bi}sum", (self.B, ho, wo, gw))
                ops.splat_combine(t2, att, comb, pool_stride=s if s > 1 else 0, stream=st)
                if b.down is not None:
                    dsrc = cur
                    if s > 1:                                  # AvgPool2d(s, s, ceil_mode=True, count_include_pad=False)
                        dsrc = self._buf(f"s{si}dp", (self.B, ops.pool2d_size(h, s, s, 0, True), ops.pool2d_size(w, s, s, 0, True),
                                                      cur.shape[3]))
                        ops.avgpool(cur, dsrc, s, s, 0, ceil_mode=True, count_include_pad=False, stream=st)
                    res = self._buf(f"s{si}ds", (self.B, ho, wo, b.down.cout))
                    ops.conv2d(dsrc, b.down.w, b.down.b, res, stream=st)
                else:
                    res = cur
                out = self._buf(f"s{si}o{bi % 2}", (self.B, ho, wo, b.c3.cout))
                ops.conv2d(comb, b.c3.w, b.c3.b, out, res=res, act=A_RELU, stream=st)
                cur, h, w = out, ho, wo
            feats.append(cur)
        return feats

    def _swin(self, x4, st):
        """SwinTransformer.forward (swin_transformer.py:684-716) for 'swin_base': tokens stay one [H*W, C] matrix per
        stage (= the NHWC map), every Linear is a tensor-core GEMM with the residual / GELU fused in its finish, the
        window partition / shift / padding / mask live inside window_attn_kernel, and the per-stage output norms
        write the NHWC feature maps the decoder reads."""
        e = self.plan.enc
        B = self.B
        H, W, C = x4.shape[1] // 4, x4.shape[2] // 4, e.embed
        pe = self._buf("pe", (B, H, W, C))
        ops.conv2d(x4, e.patch.w, e.patch.b, pe, KH=4, KW=4, stride=4, pad=0, stream=st)          # PatchEmbed :473-489
        x = self._buf("s0x", (B * H * W, C))
        ops.layernorm(pe.view(B * H * W, C), e.patch_norm[0], e.patch_norm[1], x, stream=st)
        feats = []
        for si, stg in enumerate(e.stages):
            N = B * H * W                               # the B token maps stacked
            ln = self._buf(f"s{si}ln", (N, C))
            qkv = self._buf(f"s{si}qkv", (N, 3 * C))
            att = self._buf(f"s{si}att", (N, C))
            hid = self._buf(f"s{si}hid", (N, 4 * C))
            for b in stg.blocks:                                                            # SwinTransformerBlock :257-323
                ops.layernorm(x, b.norm1[0], b.norm1[1], ln, stream=st)
                ops.linear(ln, b.qkv_w, b.qkv_b, qkv, stream=st)
                if B == 1:        # the one-frame path issues the one-image call exactly as before batching
                    ops.window_attention(qkv, b.qkv_b, b.relb, att, H, W, stg.heads, b.shift, window=e.window, stream=st)
                else:
                    ops.window_attention(qkv, b.qkv_b, b.relb, att, H, W, stg.heads, b.shift, window=e.window, stream=st,
                                         B=B)
                ops.linear(att, b.proj_w, b.proj_b, x, res=x, stream=st)                    # x = shortcut + proj(attn)
                ops.layernorm(x, b.norm2[0], b.norm2[1], ln, stream=st)
                ops.linear(ln, b.fc1_w, b.fc1_b, hid, act=A_GELU, stream=st)
                ops.linear(hid, b.fc2_w, b.fc2_b, x, res=x, stream=st)                      # x = x + mlp(norm2(x))
            f = self._buf(f"s{si}f", (self.B, H, W, C))
            ops.layernorm(x, stg.norm[0], stg.norm[1], f.view(N, C), stream=st)             # norm{i} on the stage output
            feats.append(f)
            if stg.down is not None:                                                        # PatchMerging :339-365
                H2, W2 = (H + 1) // 2, (W + 1) // 2
                mg = self._buf(f"s{si}mg", (B * H2 * W2, 4 * C))
                if B == 1:
                    ops.patch_merge(x, mg, H, W, stream=st)
                else:
                    ops.patch_merge(x, mg, H, W, stream=st, B=B)
                mln = self._buf(f"s{si}mln", (B * H2 * W2, 4 * C))
                ops.layernorm(mg, stg.down.norm[0], stg.down.norm[1], mln, stream=st)
                x = self._buf(f"s{si + 1}x", (B * H2 * W2, 2 * C))
                ops.linear(mln, stg.down.w, stg.down.b, x, stream=st)
                H, W, C = H2, W2, 2 * C
        return feats

    def _mobilenetv3(self, x, st):
        """MobileNetV3-Large (mobilenetv3.py:135-215): the 3x3/2 stem with h_swish, then per InvertedResidual the expand conv
        with the block's activation, the depthwise conv (with the activation when the block has no SE), for SE blocks the gate
        (pixel mean, fc1 + ReLU, fc2 + h_sigmoid in one launch) and gate * x with the activation (the reference applies the
        SE before the activation, :127-129), then the pw-linear conv with the residual fused.  Taps after blocks 3, 6 and 12;
        the last tap is the 1x1 960 conv with h_swish."""
        e = self.plan.enc
        H, W = x.shape[1], x.shape[2]
        h, w = self._osz(H, 3, 2, 1), self._osz(W, 3, 2, 1)
        cur = self._buf("stem", (self.B, h, w, e.stem.cout))
        ops.conv2d(x, e.stem.w, e.stem.b, cur, KH=3, KW=3, stride=2, pad=1, act=A_HSWISH, stream=st)
        ws = self._reduce_ws("se_ws", max(b.dw.cout for b in e.blocks if b.se is not None))
        feats = []
        for i, b in enumerate(e.blocks):
            act = A_HSWISH if b.hs else A_RELU
            y = cur
            if b.expand is not None:
                t = self._buf(f"b{i}e", (self.B, h, w, b.expand.cout))
                ops.conv2d(y, b.expand.w, b.expand.b, t, act=act, stream=st)
                y = t
            pad = (b.k - 1) // 2 * b.dil                                       # mobilenetv3.py:119-125
            ho, wo = self._osz(h, b.k, b.stride, pad, b.dil), self._osz(w, b.k, b.stride, pad, b.dil)
            t = self._buf(f"b{i}d", (self.B, ho, wo, b.dw.cout))
            ops.dwconv(y, b.dw.w, b.dw.b, t, K=b.k, stride=b.stride, pad=pad, dil=b.dil,
                       act=A_NONE if b.se is not None else act, stream=st)
            if b.se is not None:
                gate = self._vec(f"b{i}gate", b.dw.cout)
                ops.se_gate(t, b.se.w1, b.se.b1, b.se.w2, b.se.b2, gate, ws, stream=st)
                g = self._buf(f"b{i}g", (self.B, ho, wo, b.dw.cout))
                ops.gate_scale(t, gate, g, act=act, stream=st)
                t = g
            o = self._buf(f"b{i}o", (self.B, ho, wo, b.pw.cout))
            ops.conv2d(t, b.pw.w, b.pw.b, o, res=cur if b.res else None, stream=st)
            cur, h, w = o, ho, wo
            if b.tap:
                feats.append(cur)
        last = self._buf("last", (self.B, h, w, e.last.cout))
        ops.conv2d(cur, e.last.w, e.last.b, last, act=A_HSWISH, stream=st)
        feats.append(last)
        return feats

    def _mobilenet(self, x, st):
        e = self.plan.enc
        H, W = x.shape[1], x.shape[2]
        h, w = self._osz(H, 3, 2, 1), self._osz(W, 3, 2, 1)
        cur = self._buf("stem", (self.B, h, w, 32))
        ops.conv2d(x, e.stem.w, e.stem.b, cur, KH=3, KW=3, stride=2, pad=1, act=A_RELU6, stream=st)
        feats = []
        for i, b in enumerate(e.blocks):
            y = cur
            if b.expand is not None:
                t = self._buf(f"b{i}e", (self.B, h, w, b.expand.cout))
                ops.conv2d(y, b.expand.w, b.expand.b, t, act=A_RELU6, stream=st)
                y = t
            pad = b.dil  # (3-1)//2*dil, mobilenetv2.py:41-42
            ho, wo = self._osz(h, 3, b.stride, pad, b.dil), self._osz(w, 3, b.stride, pad, b.dil)
            t = self._buf(f"b{i}d", (self.B, ho, wo, b.dw.cout))
            ops.dwconv(y, b.dw.w, b.dw.b, t, K=3, stride=b.stride, pad=pad, dil=b.dil, act=A_RELU6, stream=st)
            o = self._buf(f"b{i}o", (self.B, ho, wo, b.pw.cout))
            ops.conv2d(t, b.pw.w, b.pw.b, o, res=cur if b.res else None, stream=st)
            cur, h, w = o, ho, wo
            if b.tap:
                feats.append(cur)
        last = self._buf("last", (self.B, h, w, e.last.cout))
        ops.conv2d(cur, e.last.w, e.last.b, last, act=A_RELU6, stream=st)
        feats.append(last)
        return feats


# =====================================================================================
# per-frame network body shared by AOTEngine and MultiVideoInferEngine: n maps stacked in the rows of one workspace
# =====================================================================================
@contextlib.contextmanager
def _lt_probe(on, Q, Tk, C):
    """With LT_PROBE set and `on`: CUDA events around the launches of the block and its FLOPs (4 N Tk C) appended."""
    probe = LT_PROBE if on else None
    if probe is None:
        yield
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    yield
    e1.record()
    probe.append((e0, e1, 4.0 * Q.shape[0] * Tk * C))


def _static_buf(bufs, key, shape, device):
    """bufs[(key, shape)], an fp32 buffer allocated on first use and kept: bodies captured for several shapes (one per
    video count n) each keep reading their own."""
    t = bufs.get((key, shape))
    if t is None:
        t = bufs[(key, shape)] = torch.empty(shape, dtype=torch.float32, device=device)
    return t


def _split_partials(bufs, splits, rows, H, dv, device, cap_rows=None):
    """Split-KV partials (O [splits, rows, dv], m [splits, H, rows], l [splits, H, rows]): contiguous views of three
    flat fp32 allocations per split count, kept in bufs and sized for cap_rows (default rows) query rows, so bodies over any
    rows <= cap_rows read memory that lives as long as bufs."""
    views = bufs.get((splits, rows))
    if views is None:
        flat = bufs.get(splits)
        if flat is None:
            cap = cap_rows or rows
            flat = bufs[splits] = [torch.empty(splits * cap * c, dtype=torch.float32, device=device)
                                   for c in (dv, H, H)]
        O, m, l = flat
        nM = splits * H * rows
        views = bufs[(splits, rows)] = (O[:splits * rows * dv].view(splits, rows, dv), m[:nM].view(splits, H, rows),
                                        l[:nM].view(splits, H, rows))
    return views


def _aot_lstt_buffers(rows, C, L, device):
    """The AOT LSTT's fp32 activations over `rows` token rows, by name (curr_Q, curr_V, st_K, st_V: per-layer lists)."""
    f = lambda c: torch.empty((rows, c), dtype=torch.float32, device=device)
    out = {k: f(m * C) for k, m in (("id_emb", 1), ("x", 1), ("ln", 1), ("ln_pos", 1), ("qk", 2), ("v", 1), ("core", 2),
                                    ("tmp", 1), ("ff", 4), ("ff2", 4), ("cat", L + 1))}
    out.update((k, [f(C) for _ in range(L)]) for k in ("curr_Q", "curr_V", "st_K", "st_V"))
    return out


def _fuse_layer(Lw, cQ, cV, id_emb, tmp, K, V, st):
    """fuse_key_value_id (transformer.py:364-367) of one layer: K = curr_K, V = linear_V(curr_V + id)."""
    ops.eltwise(ops.EW_ADD, cV, id_emb, tmp, stream=st)
    ops.linear(tmp, Lw.linV_w, Lw.linV_b, V, stream=st)
    ops.eltwise(ops.EW_COPY, cQ, None, K, stream=st)


def aot_fuse_memories(P, a, id_emb, K, V, st):
    """update_short_term_memory core (aot_engine.py:315-332) over the rows of workspace `a`: the short-term K[li] /
    V[li] of every layer from its curr_Q / curr_V and the ID embedding."""
    for li in range(P.L):
        _fuse_layer(P.layers[li], a.curr_Q[li], a.curr_V[li], id_emb, a.tmp, K[li], V[li], st)


def aot_lstt(P, a, proj, pos, hw, n, st_K, st_V, id_emb, attend_own, attend_bank, local, st):
    """The AOT LSTT (transformer.py:321-359) over n maps of hw = (h, w) tokens stacked in the rows of workspace `a`
    (x, ln, ln_pos, qk, v, core, tmp, ff, ff2, cat, curr_Q, curr_V sliced to those rows, and the groupnorm workspace
    gn_ws for n maps); proj: their projected 16x features, pos: the position table over the same rows.  id_emb None: a
    propagated frame, whose long-term step reads the bank; else a reference frame, whose short-term K / V (st_K, st_V)
    are fused first and are its long-term memory.  The engine's hooks launch the attention steps:
      attend_own(Q, K, V, out, st, long_term)   over the frame's own K / V: the self-attention, and (long_term=True) the
                                                reference frame's long-term step
      attend_bank(li, Q, out, st)               the long-term step over layer li's bank
      local(li, Q, K, V, out, st)               the short-term local attention"""
    C = P.C
    h, w = hw
    x = a.x
    ops.eltwise(ops.EW_COPY, proj, None, x, stream=st)
    ops.eltwise(ops.EW_COPY, proj, None, a.cat[:, :C], stream=st)
    for li in range(P.L):
        Lw = P.layers[li]
        # 1) self-attention (transformer.py:321-326)
        ops.layernorm(x, Lw.norm1[0], Lw.norm1[1], a.ln, add=pos, out2=a.ln_pos, stream=st)
        ops.linear(a.ln_pos, Lw.sa_qk_w, Lw.sa_qk_b, a.qk, stream=st)
        ops.linear(a.ln, Lw.sa_v_w, Lw.sa_v_b, a.v, stream=st)
        attend_own(a.qk[:, :C], a.qk[:, C:], a.v, a.core[:, :C], st, False)
        ops.linear(a.core[:, :C], Lw.sa_proj_w, Lw.sa_proj_b, x, res=x, stream=st)
        # 2) long + short term (transformer.py:329-352)
        cQ, cV = a.curr_Q[li], a.curr_V[li]
        ops.layernorm(x, Lw.norm2[0], Lw.norm2[1], cV, stream=st)
        ops.linear(cV, Lw.linQ_w, Lw.linQ_b, cQ, stream=st)
        if id_emb is not None:
            _fuse_layer(Lw, cQ, cV, id_emb, a.tmp, st_K[li], st_V[li], st)
            attend_own(cQ, st_K[li], st_V[li], a.core[:, :C], st, True)
        else:
            attend_bank(li, cQ, a.core[:, :C], st)
        local(li, cQ, st_K[li], st_V[li], a.core[:, C:], st)
        ops.linear(a.core, Lw.lst_proj_w, Lw.lst_proj_b, x, res=x, stream=st)
        # 3) feed-forward (transformer.py:354-359, basic.py:27-35)
        ops.layernorm(x, Lw.norm3[0], Lw.norm3[1], a.ln, stream=st)
        ops.linear(a.ln, Lw.lin1_w, Lw.lin1_b, a.ff, stream=st)
        ops.groupnorm(a.ff.view(n, h * w, 4 * C), Lw.gn[0], Lw.gn[1], a.ff.view(n, h * w, 4 * C), 32, A_GELU, a.gn_ws,
                      stream=st)
        ops.dwconv(a.ff.view(n, h, w, 4 * C), Lw.dw_w, None, a.ff2.view(n, h, w, 4 * C), K=5, pad=2, stream=st)
        ops.linear(a.ff2, Lw.lin2_w, Lw.lin2_b, x, res=x, stream=st)
        # decoder norms (transformer.py:124-135) written straight into the decoder input
        ops.layernorm(x, Lw.dec_norm[0], Lw.dec_norm[1], a.cat[:, (li + 1) * C:(li + 2) * C], stream=st)


def fpn_decode(P, cat_nhwc, x4, x8, x16, dbuf, gn_ws, st):
    """The FPN decoder (fpn.py:34-58) over B = x4.shape[0] images: cat_nhwc [B, h, w, c] the LSTT output, x4 / x8 / x16
    the encoder maps -> logits [B, h4, w4, 11] (NHWC).  Every intermediate map is a static buffer of the dict dbuf."""
    D = P.dec
    B = x4.shape[0]
    buf = lambda key, x, c: _static_buf(dbuf, key, (B, x.shape[1], x.shape[2], c), x.device)

    def conv_gn(x, blk, key, k, pad):
        o = buf(key, x, blk.cout)
        ops.conv2d(x, blk.w, blk.b, o, KH=k, KW=k, pad=pad, stream=st)
        ov = o.view(B, -1, blk.cout)
        ops.groupnorm(ov, blk.gn[0], blk.gn[1], ov, 8, A_RELU, gn_ws, stream=st)
        return o

    x = conv_gn(cat_nhwc, D.conv_in, "in", 1, 0)
    a = buf("a16", x16, D.adapter_16x.cout)
    ops.conv2d(x16, D.adapter_16x.w, D.adapter_16x.b, a, res=x, stream=st)
    x = conv_gn(a, D.conv_16x, "c16", 3, 1)
    for xs, tag, ad, cv in ((x8, "8", D.adapter_8x, D.conv_8x), (x4, "4", D.adapter_4x, D.conv_4x)):
        up = buf("up" + tag, xs, x.shape[3])
        ops.bilinear(x, up, P.align_corners, stream=st)
        a = buf("a" + tag, xs, ad.cout)
        ops.conv2d(xs, ad.w, ad.b, a, res=up, stream=st)
        x = conv_gn(a, cv, "c" + tag, 3, 1)
    lg = buf("logit", x, D.conv_out.cout)
    ops.conv2d(x, D.conv_out.w, D.conv_out.b, lg, stream=st)
    return lg


# DeAOT: the gated propagation module stack (transformer.py:501-665) over n maps, shared by DeAOTEngine and
# DeAOTMultiVideoInferEngine as aot_lstt is by the AOT engines
def gp_splits(n_queries, C, Tk):
    """KV-split count of the fused DeAOT long-term attention kernel over n_queries query rows (one CTA = 128 queries x 64
    value channels x one split): about two waves of CTAs, at least four 64-key tiles per split."""
    base = ((n_queries + 127) // 128) * (4 * C // 64)
    tiles = (max(Tk, 1) + 63) // 64
    return max(1, min(tiles // 4 if tiles >= 8 else 1, max(1, (2 * 132) // base)))


def _deaot_gpm_buffers(rows, C, L, device):
    """DeAOT's fp32 activations over `rows` token rows, by name (curr_Q, curr_V, curr_IDV, st_K, st_V: per-layer lists;
    curr_IDV[0] is None, layer 0 has no ID stream input), in the one-video engine's allocation order."""
    f = lambda c: torch.empty((rows, c), dtype=torch.float32, device=device)
    d = C // 2
    out = {k: f(m) for k, m in (("id_emb", C), ("xz", 2 * C), ("ln", C), ("qv", d + 2 * C), ("catU", 4 * C),
                                ("idin", 2 * C), ("core", 4 * C), ("gated", 4 * C), ("dw", 8 * C), ("c", 2 * C),
                                ("sa_qk", d), ("sa_v", 4 * C), ("sa_u", 4 * C), ("cat", 2 * C))}
    out["curr_Q"] = [f(d) for _ in range(L)]
    out["curr_V"] = [f(2 * C) for _ in range(L)]
    out["curr_IDV"] = [None] + [f(C) for _ in range(L - 1)]
    out["st_K"] = [f(d) for _ in range(L)]
    out["st_V"] = [f(4 * C) for _ in range(L)]   # cat[V | ID_V] (transformer.py:625-626)
    return out


def _gated_tail(a, core, U, dw_w, out, n, hw, st):
    """(attn @ V) * U -> depthwise 5x5 (attention.py:707-709 / :855-857) over n maps; the projection is fused later."""
    h, w = hw
    C4 = core.shape[1]
    ops.eltwise(ops.EW_MUL, core, U, a.gated, stream=st)
    ops.dwconv(a.gated.view(n, h, w, C4), dw_w, None, out.unflatten(0, (n, h, w)), K=5, pad=2, stream=st)


def _deaot_fuse_id(Lw, a, C, cIDV, id_emb, out, st):
    """GatedPropagationModule.fuse_key_value_id (transformer.py:659-665) of one layer."""
    if cIDV is None:
        ops.linear(id_emb, Lw.idv_w, Lw.idv_b, out, act=A_SILU, stream=st)
    else:
        ops.eltwise(ops.EW_COPY, cIDV, None, a.idin[:, :C], stream=st)
        ops.eltwise(ops.EW_COPY, id_emb, None, a.idin[:, C:], stream=st)
        ops.linear(a.idin, Lw.idv_w, Lw.idv_b, out, act=A_SILU, stream=st)


def deaot_fuse_memories(P, a, id_emb, K, V, st):
    """deaot_engine.py:20-45 over the rows of workspace `a`: the short-term K[li] = curr_Q and V[li] = [curr_V | ID_V] of
    every layer, ID_V = fuse_key_value_id(curr_ID_V, id_emb)."""
    C2 = 2 * P.C
    for li in range(P.L):
        ops.eltwise(ops.EW_COPY, a.curr_Q[li], None, K[li], stream=st)
        ops.eltwise(ops.EW_COPY, a.curr_V[li], None, V[li][:, :C2], stream=st)
        _deaot_fuse_id(P.layers[li], a, P.C, a.curr_IDV[li], id_emb, V[li][:, C2:], st)


def deaot_lstt(P, a, proj, hw, n, st_K, st_V, id_emb, attend_own, attend_bank, local, st):
    """The DeAOT LSTT (GatedPropagationModule stack, transformer.py:590-665, and its final GroupNorm, :197-200) over n maps of
    hw = (h, w) tokens stacked in the rows of workspace `a` (the activations of _deaot_gpm_buffers sliced to those rows, and
    the groupnorm workspace gn_ws for n maps); proj: their projected 16x features.  id_emb None: a propagated frame, whose
    long-term step reads the bank; else a reference frame, whose short-term K / V (st_K, st_V) are fused first and are its
    long-term memory.  The engine's hooks launch the attention steps:
      attend_own(Q, K, V, out, st, long_term)   over the frame's own K / V: the gated self-attention, and (long_term=True)
                                                the reference frame's long-term step
      attend_bank(li, Q, out, st)               the long-term step over layer li's bank
      local(li, Q, K, V, out, st)               the short-term gated local attention"""
    C = P.C
    h, w = hw
    d, C2, C4 = C // 2, 2 * C, 4 * C
    x, z = a.xz[:, :C], a.xz[:, C:]
    ops.eltwise(ops.EW_COPY, proj, None, x, stream=st)
    ops.eltwise(ops.EW_FILL, None, None, z, scalar=0.0, stream=st)        # tgt_id = 0 (transformer.py:603)
    for li in range(P.L):
        Lw = P.layers[li]
        cQ, cV = a.curr_Q[li], a.curr_V[li]
        ops.layernorm(x, Lw.norm1[0], Lw.norm1[1], a.ln, stream=st)
        ops.linear(a.ln, Lw.qv_w, Lw.qv_b, a.qv, stream=st)
        ops.eltwise(ops.EW_COPY, a.qv[:, :d], None, cQ, stream=st)
        ops.eltwise(ops.EW_SILU, a.qv[:, d:], None, cV, stream=st)          # curr_V = silu(.) :599
        ops.linear(a.ln, Lw.u_w, Lw.u_b, a.catU[:, :C2], act=A_SILU, stream=st)
        if li == 0:
            ops.eltwise(ops.EW_FILL, None, None, a.catU[:, C2:], scalar=1.0, stream=st)   # :604-605
            cIDV = None
        else:
            cIDV = a.curr_IDV[li]
            ops.layernorm(z, Lw.id_norm1[0], Lw.id_norm1[1], cIDV, stream=st)
            ops.linear(cIDV, Lw.idu_w, Lw.idu_b, a.catU[:, C2:], act=A_SILU, stream=st)    # :610-611
        if id_emb is not None:
            ops.eltwise(ops.EW_COPY, cQ, None, st_K[li], stream=st)
            ops.eltwise(ops.EW_COPY, cV, None, st_V[li][:, :C2], stream=st)
            _deaot_fuse_id(Lw, a, C, cIDV, id_emb, st_V[li][:, C2:], st)
            attend_own(cQ, st_K[li], st_V[li], a.core, st, True)
        else:
            attend_bank(li, cQ, a.core, st)
        _gated_tail(a, a.core, a.catU, Lw.lt_dw, a.dw[:, :C4], n, hw, st)
        local(li, cQ, st_K[li], st_V[li], a.core, st)
        _gated_tail(a, a.core, a.catU, Lw.st_dw, a.dw[:, C4:], n, hw, st)
        # [tgt | tgt_id] += proj_lt(.) + proj_st(.)   (transformer.py:633-641) as one K = 8C GEMM
        ops.linear(a.dw, Lw.lst_proj_w, Lw.lst_proj_b, a.xz, res=a.xz, stream=st)
        # gated self-attention on both streams (transformer.py:644-653, attention.py:648-669)
        ops.layernorm(x, Lw.norm2[0], Lw.norm2[1], a.c[:, :C], stream=st)
        ops.layernorm(z, Lw.id_norm2[0], Lw.id_norm2[1], a.c[:, C:], stream=st)
        ops.linear(a.c, Lw.sa_qk_w, Lw.sa_qk_b, a.sa_qk, stream=st)
        ops.linear(a.c[:, :C], Lw.sa_v1[0], Lw.sa_v1[1], a.sa_v[:, :C2], act=A_SILU, stream=st)
        ops.linear(a.c[:, C:], Lw.sa_v2[0], Lw.sa_v2[1], a.sa_v[:, C2:], act=A_SILU, stream=st)
        ops.linear(a.c[:, :C], Lw.sa_u1[0], Lw.sa_u1[1], a.sa_u[:, :C2], act=A_SILU, stream=st)
        ops.linear(a.c[:, C:], Lw.sa_u2[0], Lw.sa_u2[1], a.sa_u[:, C2:], act=A_SILU, stream=st)
        attend_own(a.sa_qk, a.sa_qk, a.sa_v, a.core, st, False)
        _gated_tail(a, a.core, a.sa_u, Lw.sa_dw, a.dw[:, :C4], n, hw, st)
        ops.linear(a.dw[:, :C4], Lw.sa_proj_w, Lw.sa_proj_b, a.xz, res=a.xz, stream=st)
    # final GroupNorm1D(2C, groups=2) (transformer.py:197-200,241) -> decoder input
    ops.groupnorm(a.xz.view(n, h * w, C2), P.final_gn[0], P.final_gn[1], a.cat.view(n, h * w, C2), 2, A_NONE, a.gn_ws,
                  stream=st)


# =====================================================================================
# single engine (<= max_obj_num objects)
# =====================================================================================
class AOTEngine(nn.Module):
    def __init__(self, aot_model, gpu_id=0, long_term_mem_gap=9999, short_term_mem_skip=1, long_term_mem_max=None,
                 precision=None, long_term_mem_policy=None):
        """long_term_mem_max = M bounds the long-term bank to M memory frames: the first frame stored after
        restart_engine() stays, the other M - 1 slots hold the newest stored frames (the oldest is overwritten).  None: the
        bound of cfg.TEST_LONG_TERM_MEM_MAX if the config has one, else the reference's ever-growing memory.
        long_term_mem_policy: which frame a full bounded bank overwrites -- "fifo" (default) the oldest, "usage" the one
        with the lowest mean attention mass since it was stored (see long_term_memory_usage).  None: cfg.TEST_LONG_TERM_MEM_POLICY
        if the config has one, else "fifo".
        precision: "fp32" (default; split-fp16 tensor-core operands, fp32-faithful) or "fp16" (operands of every
        tensor-core conv, linear and attention product rounded once to fp16, accumulated in fp32).  None: cfg.TEST_PRECISION
        if the config has one, else "fp32"."""
        super().__init__()
        self.precision = _resolve_precision(aot_model, precision)
        self.cfg = aot_model.cfg
        self.align_corners = aot_model.cfg.MODEL_ALIGN_CORNERS
        self.AOT = aot_model
        self.max_obj_num = aot_model.max_obj_num
        self.gpu_id = gpu_id
        self.long_term_mem_gap = long_term_mem_gap
        self.short_term_mem_skip = short_term_mem_skip
        self.long_term_mem_max = _resolve_mem_max(aot_model, long_term_mem_max)
        self.long_term_mem_policy = _resolve_mem_policy(aot_model, long_term_mem_policy, self.long_term_mem_max)
        self.losses = None
        self._enc = None
        self._ws = None
        self._ws_key = None
        self._P = None
        self.graphs = GraphCache()
        self.tk_dev = None
        self.wr_dev = None            # bounded bank: row offset of the next stored memory frame
        self.kv_shard = None          # (rank, world, process_group) when the long-term bank is sharded over GPUs
        self.restart_engine()

    # ------------------------------------------------------------------ protocol
    def forward(self, *args, **kwargs):
        raise NotImplementedError("training step (BASELINE config 5) is a 'next' row (SURVEY 8f); this engine "
                                  "implements the eval protocol")

    def restart_engine(self, batch_size=1, enable_id_shuffle=False):
        if batch_size != 1 or enable_id_shuffle:
            raise NotImplementedError("batch_size > 1 / id shuffle are training-only (SURVEY 8f)")
        self.batch_size = 1
        self.frame_step = 0
        self.last_mem_step = -1
        self.enable_id_shuffle = False
        self.freeze_id = False
        self.obj_nums = None
        self.pos_emb = None
        self.enc_size_2d = None
        self.enc_hw = None
        self.input_size_2d = None
        self.bank_len = 0
        self._drop_offline_clip()
        self._alloc_pending = False   # offline_encoder sized the engine for a new video; add_reference_frame allocates
        self.curr_enc_embs = None
        self.curr_id_embs = None
        self.pred_id_logits = None
        self._have_lstt = False
        self._mem_frames = 0          # memory frames stored so far (global count, all shards)
        if self.tk_dev is not None:
            self.tk_dev.zero_()
            self.wr_dev.zero_()
        self._zero_usage()

    def _drop_offline_clip(self):
        self.enable_offline_enc = False
        self.offline_enc_embs = None
        self.offline_masks = None
        self.offline_frames = -1
        self.total_offline_frame_num = 0

    def _zero_usage(self):
        if getattr(self._ws, "usage_U", None) is not None:
            self._ws.usage_U.zero_()
            self._ws.usage_A.zero_()

    def _usage(self):
        return self.long_term_mem_policy == "usage" and self.long_term_mem_max is not None

    def enable_kv_sharding(self, rank, world, group=None):
        """BASELINE config 4: shard the long-term bank by memory frame round-robin over `world` ranks.  Every rank
        runs the rest of the network redundantly on identical inputs; rank `f % world` keeps memory frame f; each
        rank's long-term attention produces un-normalised partials (m, l, O) over its shard which are all-gathered
        (one NCCL collective per layer) and merged exactly (log-sum-exp) on every rank."""
        if self.precision == "fp16":
            raise NotImplementedError("a long-term bank sharded over GPUs is not built for precision='fp16'")
        if not (LT_IMPL.startswith("tc") and not self._plan_is_deaot()):
            raise NotImplementedError("sharded long-term attention is implemented for the AOT tensor-core kernel")
        if self.long_term_mem_max is not None:
            raise NotImplementedError("a bounded long-term bank (long_term_mem_max) cannot be sharded over GPUs: each rank "
                                      "would need its own ring")
        self.kv_shard = (int(rank), int(world), group)

    def _plan_is_deaot(self):
        return self.AOT.cfg.MODEL_VOS == "deaot"

    def update_size(self, input_size, enc_size):
        self.input_size_2d = tuple(int(s) for s in input_size)
        self.enc_size_2d = tuple(int(s) for s in enc_size)
        self.enc_hw = self.enc_size_2d[0] * self.enc_size_2d[1]

    # ------------------------------------------------------------------ buffers
    def _plan(self):
        # resolved once per reference frame (get_plan walks every parameter to detect reloads)
        if self._P is None:
            self._P = get_plan(self.AOT)
        return self._P

    def _alloc(self):
        P = self._plan()
        dev = P.device
        N = self.enc_hw
        C = P.C
        L = P.L
        M = self.long_term_mem_max
        if M is not None and P.deaot and DEAOT_LT == "gemm":
            raise NotImplementedError("a bounded long-term bank (long_term_mem_max) is not built for AOTB_DEAOT_LT=gemm: its "
                                      "transposed value copies have no ring store; use the default fused kernel")
        usage = self._usage()
        key = (id(P), N, tuple(self.enc_size_2d), tuple(self.input_size_2d), LT_IMPL, DEAOT_LT, M, usage)
        if self._ws is not None and self._ws_key == key:
            # same geometry and weights as the previous video: keep buffers and captured graphs
            self.bank_len = 0
            self.tk_dev.zero_()
            self.wr_dev.zero_()
            self._zero_usage()
            self._st_ring = []
            return
        self._ws_key = key
        self.graphs.clear()
        self.tk_dev = torch.zeros(1, dtype=torch.int32, device=dev)    # live rows of the long-term bank
        self.wr_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        ws = type("WS", (), {})()
        ws.N = N
        ws.gn_ws = ops.groupnorm_workspace(1, 32, dev)
        if not P.deaot:
            bufs = _aot_lstt_buffers(N, C, L, dev)
            self.st_K, self.st_V = bufs.pop("st_K"), bufs.pop("st_V")     # the live slot: _commit_short_slot moves it
            vars(ws).update(bufs)
            self.curr_Q, self.curr_V = ws.curr_Q, ws.curr_V
            self._kdim, self._vdim = C, C
        else:
            bufs = _deaot_gpm_buffers(N, C, L, dev)
            self.st_K, self.st_V = bufs.pop("st_K"), bufs.pop("st_V")     # the live slot: _commit_short_slot moves it
            vars(ws).update(bufs)
            self.curr_Q, self.curr_V, self.curr_IDV = ws.curr_Q, ws.curr_V, ws.curr_IDV
            self._kdim, self._vdim = C // 2, 4 * C
        ws.mask = f(*self.input_size_2d)                            # static copy of the caller's label map
        self._dec_out = {}
        cap = (min(BANK_INIT_FRAMES, GEMM_GROW_FRAMES) if (P.deaot and DEAOT_LT == "gemm") else BANK_INIT_FRAMES) * N
        if M is not None:
            cap = M * N               # bounded: allocated once, slot s = rows [s N, (s + 1) N), never re-allocated
        self.bank_cap = cap
        self.bank_K = [f(cap, self._kdim) for _ in range(L)]
        self.bank_V = [f(cap, self._vdim) for _ in range(L)]
        self.bank_len = 0
        self._gemm_lt = bool(P.deaot and DEAOT_LT == "gemm")
        if self._gemm_lt:
            self._alloc_gemm_lt(cap, ws=ws)
        self._gp_tc = bool(P.deaot and DEAOT_LT == "tc")
        if self._gp_tc:
            hz = lambda *s: torch.zeros(s, dtype=torch.float16, device=dev)
            ws.gpQp = hz(self._kdim // 32, ((N + 127) // 128) * 128, 64)
            ncap = ((N + 63) // 64) * 64 + 64                      # K / V of the CURRENT frame (self-attention, reference frame)
            ws.gpSaK = hz(self._kdim // 32, ncap, 64)
            ws.gpSaV = hz(self._vdim // 32, ncap, 64)
            self.bank_gpK = [hz(self._kdim // 32, cap, 64) for _ in range(L)]     # split-fp16 rows, one "head" / 32 channels
            self.bank_gpV = [hz(self._vdim // 32, cap, 64) for _ in range(L)]
            ws.gp_part = {}
        self._tc = LT_IMPL.startswith("tc") and (not P.deaot) and (C // P.H == 32)
        if self._tc:
            hz = lambda *s: torch.zeros(s, dtype=torch.float16, device=dev)
            ws.Qp = hz(P.H, ((N + 255) // 256) * 256, 64)
            ws.saKp = hz(P.H, ((N + 127) // 128) * 128, 64)          # self-attention K / V of the current frame
            ws.saVp = hz(P.H, ((N + 127) // 128) * 128, 64)
            self.bank_Kp = [hz(P.H, cap, 64) for _ in range(L)]     # split-fp16 copies read by TMA
            self.bank_Vp = [hz(P.H, cap, 64) for _ in range(L)]
            ws.part = {}
        if usage:
            if not (self._tc or self._gp_tc):
                raise NotImplementedError("long_term_mem_policy='usage' needs the tensor-core long-term attention, which "
                                          f"this model's head shape ({P.H} x {C // P.H}) does not run on")
            # per memory slot: summed mean attention mass U and propagated frames since the store A (restart_engine zeroes
            # both), the merge's CTA sums, and one split of partials per slot
            ws.usage_U = torch.zeros(M, dtype=torch.float32, device=dev)
            ws.usage_A = torch.zeros(M, dtype=torch.int32, device=dev)
            ws.usage_ws = ops.attn_merge_usage_workspace(M, dev)
            H, dv = (1, self._vdim) if P.deaot else (P.H, C)
            ws.usage_part = (f(M, N, dv), f(M, H, N), f(M, H, N))
        self._st_ring = []
        self._ws = ws
        self._dec_bufs = {}

    def _alloc_gemm_lt(self, cap, old_len=0, old=None, ws=None):
        """Split-fp16 operand copies of the DeAOT bank for the GEMM formulation: keys [cap64][d] (weights of Q K^T),
        values transposed [4C][cap64] (weights of P V), zero beyond the live rows, plus the score matrix [N][cap64]."""
        P = self._plan()
        dev = P.device
        capw = ((cap + 63) // 64) * 64
        hz = lambda *s: torch.zeros(s, dtype=torch.float16, device=dev)
        Kh, Kl = [hz(capw, self._kdim) for _ in range(P.L)], [hz(capw, self._kdim) for _ in range(P.L)]
        Vh, Vl = [hz(self._vdim, capw) for _ in range(P.L)], [hz(self._vdim, capw) for _ in range(P.L)]
        if old is not None:
            for new_l, old_l in zip((Kh, Kl), old[:2]):
                for a, b in zip(new_l, old_l):
                    a[:old_len].copy_(b[:old_len])
            for new_l, old_l in zip((Vh, Vl), old[2:]):
                for a, b in zip(new_l, old_l):
                    a[:, :old_len].copy_(b[:, :old_len])
        self.bank_Kh, self.bank_Kl, self.bank_VhT, self.bank_VlT = Kh, Kl, Vh, Vl
        self._capw = capw
        (self._ws if ws is None else ws).S = torch.empty((self.enc_hw, capw), dtype=torch.float32, device=dev)

    def _bank_reserve(self, rows):
        if self.bank_len + rows <= self.bank_cap or self.long_term_mem_max is not None:
            return
        new_cap = max(2 * self.bank_cap, self.bank_len + rows)
        if getattr(self, "_gemm_lt", False):
            # the GEMM formulation of DeAOT's long-term attention costs O(capacity), not O(live keys): grow in steps of
            # GEMM_GROW_FRAMES memory frames (a few graph re-captures per clip) instead of doubling
            new_cap = max(self.bank_cap + GEMM_GROW_FRAMES * self.enc_hw, self.bank_len + rows)
        for lst in (self.bank_K, self.bank_V):
            for i, old in enumerate(lst):
                nb = torch.empty((new_cap, old.shape[1]), dtype=torch.float32, device=old.device)
                nb[: self.bank_len].copy_(old[: self.bank_len])
                lst[i] = nb
        if self._tc:
            for lst in (self.bank_Kp, self.bank_Vp):
                for i, old in enumerate(lst):
                    nb = torch.zeros((old.shape[0], new_cap, 64), dtype=torch.float16, device=old.device)
                    nb[:, : self.bank_len].copy_(old[:, : self.bank_len])
                    lst[i] = nb
        if getattr(self, "_gemm_lt", False):
            self._alloc_gemm_lt(new_cap, self.bank_len, (self.bank_Kh, self.bank_Kl, self.bank_VhT, self.bank_VlT))
        if getattr(self, "_gp_tc", False):
            for lst in (self.bank_gpK, self.bank_gpV):
                for i, old in enumerate(lst):
                    nb = torch.zeros((old.shape[0], new_cap, 64), dtype=torch.float16, device=old.device)
                    nb[:, : self.bank_len].copy_(old[:, : self.bank_len])
                    lst[i] = nb
        self.bank_cap = new_cap
        self.graphs.clear()            # captured launches point at the old bank

    # ------------------------------------------------------------------ reference-shaped views
    @property
    def long_term_memories(self):
        """The live rows of the bank, per layer, in the reference's list-of-lists shape.  Rows are in storage order: the order
        the frames were stored in for the unbounded bank; with long_term_mem_max = M, slot order (slot 0 = the first frame,
        slots 1 .. M - 1 the ring, which is not age order once it has wrapped)."""
        if self.bank_len == 0:
            return None
        P = self._plan()
        n = self.bank_len
        out = []
        for li in range(P.L):
            K = self.bank_K[li][:n].unsqueeze(1)
            V = self.bank_V[li][:n]
            if P.deaot:
                c2 = 2 * P.C
                out.append([K, V[:, :c2].unsqueeze(1), None, V[:, c2:].unsqueeze(1)])
            else:
                out.append([K, V.unsqueeze(1)])
        return out

    @property
    def long_term_memory_usage(self):
        """long_term_mem_policy="usage": (U, A), float32 and int32 [long_term_mem_max], per memory slot (the slot order of
        long_term_memories): U = the summed per-frame mean attention mass the propagated frames put on the slot's keys, A =
        frames propagated since the slot was stored; the bank evicts the unpinned slot with the lowest U / A.  Slot 0 is never
        evicted.  None in FIFO mode or before the first reference frame."""
        if not self._usage() or getattr(self._ws, "usage_U", None) is None:
            return None
        return self._ws.usage_U.clone(), self._ws.usage_A.clone()

    @property
    def short_term_memories(self):
        if not self._have_lstt:
            return None
        P = self._plan()
        h, w = self.enc_size_2d
        to2d = lambda t: t.view(h, w, 1, -1).permute(2, 3, 0, 1)
        out = []
        for li in range(P.L):
            if P.deaot:
                c2 = 2 * P.C
                out.append([to2d(self.st_K[li]), to2d(self.st_V[li][:, :c2]), None, to2d(self.st_V[li][:, c2:])])
            else:
                out.append([to2d(self.st_K[li]), to2d(self.st_V[li])])
        return out

    # ------------------------------------------------------------------ steps
    @_in_precision
    def _encode(self, img, st):
        if self._enc is None:
            self._enc = _Encoder(self._plan(), img.shape[2], img.shape[3])
        self._enc.plan = self._plan()
        return self._enc(img, st)

    def _check_img(self, img):
        if not img.is_cuda:
            raise RuntimeError("aot_benchmark_b200 engines run on CUDA tensors only (there is no CPU path)")

    @_in_precision
    def offline_encoder(self, all_frames, all_masks=None):
        """aot_engine.py:147-166 at batch size 1: encode every frame of a stored clip all_frames [T,3,H,W] (CUDA) and keep each
        frame's features (offline_enc_embs[t], EncEmbs views of the clip's storage; the whole clip stays resident, as in the
        reference).  all_masks [T,1,H,W] label maps, if given, are kept as offline_masks[t].  Until restart_engine(),
        add_reference_frame / match_propogate_one_frame read the stored features of their frame step and ignore an image
        they are handed; add_reference_frame(mask=None) uses the stored mask of its step.  The encoder runs over chunks of
        OFFLINE_ENC_CHUNK frames, each chunk's maps copied straight into the clip's storage.  A clip of at least one chunk
        runs every pass at B = OFFLINE_ENC_CHUNK, the last one over the clip's last chunk of frames (overlapping the pass
        before it; only its new frames are stored), so the encoder keeps one batched set of buffers and one graph whatever
        the clip lengths; a shorter clip runs as one pass of T frames whose buffers are freed when the call returns.
        The stored frames reach the LSTT and decoder through the engine's own copy buffers (see _offline_embs), so the
        offline path has its own graph keys, next to those of the per-frame path."""
        T = self._check_clip(all_frames, all_masks)
        st = torch.cuda.current_stream().cuda_stream
        _apply_pdl()
        self._P = get_plan(self.AOT)
        if self._enc is None:
            self._enc = _Encoder(self._plan(), all_frames.shape[2], all_frames.shape[3])
        self._enc.plan = self._plan()
        B = min(OFFLINE_ENC_CHUNK, T)
        starts = list(range(0, T - B + 1, B))
        if starts[-1] + B < T:
            starts.append(T - B)                       # the tail: the last B frames, of which only the new ones are stored
        store, done = None, 0
        for t0 in starts:
            maps = self._enc(all_frames[t0:t0 + B], st).nhwc
            if store is None:
                store = [torch.empty((T,) + tuple(m.shape[1:]), dtype=torch.float32, device=m.device) for m in maps]
            for m, dst in zip(maps, store):
                c = m.shape[3]
                ops.eltwise(ops.EW_COPY, m[done - t0:].reshape(-1, c), None, dst[done:t0 + B].view(-1, c), stream=st)
            done = t0 + B
        self._enc.keep_batch_sizes((1, OFFLINE_ENC_CHUNK))
        self.enable_offline_enc = True
        self.offline_frames = T
        self.total_offline_frame_num = T
        self.offline_enc_embs = [self._embs_of([m[t:t + 1] for m in store]) for t in range(T)]
        self.offline_masks = None if all_masks is None else [all_masks[t:t + 1] for t in range(T)]
        if self.input_size_2d is None:
            self.update_size(all_frames.shape[2:], tuple(store[-1].shape[1:3]))
            self._alloc_pending = True

    @staticmethod
    def _embs_of(nhwc):
        out = EncEmbs(t.permute(0, 3, 1, 2) for t in nhwc)
        out.nhwc = list(nhwc)
        return out

    def _check_clip(self, all_frames, all_masks):
        if not isinstance(all_frames, torch.Tensor) or all_frames.dim() != 4 or all_frames.shape[0] < 1 \
                or all_frames.shape[1] != 3:
            shape = tuple(all_frames.shape) if isinstance(all_frames, torch.Tensor) else type(all_frames).__name__
            raise ValueError(f"offline_encoder: all_frames must be a [T,3,H,W] tensor with T >= 1, got {shape}")
        self._check_img(all_frames)
        T, _, H, W = all_frames.shape
        if all_masks is not None:
            if not isinstance(all_masks, torch.Tensor) or tuple(all_masks.shape) != (T, 1, H, W):
                shape = tuple(all_masks.shape) if isinstance(all_masks, torch.Tensor) else type(all_masks).__name__
                raise ValueError(f"offline_encoder: all_masks must be [T,1,H,W] = {(T, 1, H, W)} label maps, got {shape}")
            self._check_img(all_masks)
        return T

    def _offline_step(self, step):
        if not 0 <= step < self.total_offline_frame_num:
            raise IndexError(f"frame step {step} is outside the clip stored by offline_encoder "
                             f"({self.total_offline_frame_num} frames: steps 0 .. {self.total_offline_frame_num - 1})")
        return step

    def _offline_embs(self, step, st):
        """Copy stored frame `step` into the engine's offline feature buffers and return them.  They are static across
        frames and videos, so the LSTT and decoder graphs keyed on them are captured once; they are not the per-frame
        encoder's output buffers, so an engine that runs both paths holds one set of those graphs per path."""
        src = self.offline_enc_embs[self._offline_step(step)].nhwc
        key = tuple(tuple(t.shape) for t in src)
        frame = getattr(self, "_offline_frame", None)
        if frame is None or frame[0] != key:
            frame = self._offline_frame = (key, self._embs_of([torch.empty(t.shape, dtype=torch.float32, device=t.device)
                                                               for t in src]))
        dst = frame[1]
        for a, b in zip(src, dst.nhwc):
            ops.eltwise(ops.EW_COPY, a.reshape(-1, a.shape[3]), None, b.view(-1, b.shape[3]), stream=st)
        return dst

    @_in_precision
    def assign_identity_from_mask(self, mask, st):
        """one_hot_mask + get_id_emb (aot_engine.py:168-179) fused as a gather (K4)."""
        P = self._plan()
        ws = self._ws
        if mask.dim() == 4 and mask.shape[1] != 1:
            # probability / one-hot input [1, 11, H, W]: dense conv through the same weight table
            x = torch.empty((1, mask.shape[2], mask.shape[3], mask.shape[1]), dtype=torch.float32, device=mask.device)
            ops.nchw_to_nhwc(mask.float().contiguous(), x, stream=st)
            ops.conv2d(x, P.id_wt, P.id_b, ws.id_emb.view(1, *self.enc_size_2d, P.C), KH=P.id_k, KW=P.id_k,
                       stride=P.id_stride, pad=P.id_pad, stream=st)
            if P.deaot:
                ops.layernorm(ws.id_emb, P.id_norm[0], P.id_norm[1], ws.id_emb, stream=st)
            return ws.id_emb
        m2 = mask.reshape(mask.shape[-2], mask.shape[-1]).float().contiguous()
        if tuple(m2.shape) == tuple(ws.mask.shape):
            ops.eltwise(ops.EW_COPY, m2, None, ws.mask, stream=st)      # static buffer: graph replays read it
            m2 = ws.mask
        self._id_from_static_mask(m2, st)
        return ws.id_emb

    def _id_from_static_mask(self, m2, st):
        P = self._plan()
        if P.C == 256:
            ops.id_embed_runs(m2, P.id_wp, P.id_b, self._ws.id_emb, P.C, P.nid, P.id_k, P.id_stride, P.id_pad,
                              ln_gamma=P.id_norm[0] if P.deaot else None, ln_beta=P.id_norm[1] if P.deaot else None,
                              stream=st)
        else:
            ops.id_embed(m2, P.id_wt, P.id_b, self._ws.id_emb, P.C, P.nid, P.id_k, P.id_stride, P.id_pad,
                         ln_gamma=P.id_norm[0] if P.deaot else None, ln_beta=P.id_norm[1] if P.deaot else None, stream=st)

    @_in_precision
    def add_reference_frame(self, img=None, mask=None, frame_step=-1, obj_nums=None, img_embs=None):
        if self.obj_nums is None and obj_nums is None:
            print('No objects for reference frame!')
            exit()
        elif obj_nums is not None:
            self.obj_nums = obj_nums
        if frame_step == -1:
            frame_step = self.frame_step
        offline = self.enable_offline_enc and img_embs is None
        if offline:
            self._offline_step(frame_step)
            if mask is None and self.offline_masks is not None:
                mask = self.offline_masks[frame_step]
        if img_embs is None and img is None and not offline:
            print('No image for reference frame!')
            exit()
        if mask is None:
            print('No mask for reference frame!')
            exit()
        st = torch.cuda.current_stream().cuda_stream
        _apply_pdl()
        self._P = get_plan(self.AOT)   # picks up load_state_dict / .to() done since the last video
        if offline:
            img_embs = self._offline_embs(frame_step, st)      # the stored frame; an image handed here is ignored
        elif img_embs is None:
            self._check_img(img)
            img_embs = self._encode(img, st)
        if self.input_size_2d is None or self._alloc_pending:
            if self.input_size_2d is None:
                f16 = img_embs.nhwc[-1]
                in_size = img.shape[2:] if img is not None else (f16.shape[1] * 16, f16.shape[2] * 16)
                self.update_size(in_size, (f16.shape[1], f16.shape[2]))
            self._alloc()
            self._alloc_pending = False
        self.curr_enc_embs = img_embs
        if self.pos_emb is None:
            # the table lives in the workspace, i.e. exactly as long as the captured graphs that read it: re-creating it per
            # video left the graphs of the previous video replaying a freed address (same block again only by allocator luck)
            if getattr(self._ws, "pos_emb", None) is None:
                self._ws.pos_emb = _pos_emb_sine(*self.enc_size_2d, npf=self._plan().C // 2).to(self._plan().device)
            self.pos_emb = self._ws.pos_emb
        id_emb = self.assign_identity_from_mask(mask, st)
        self.curr_id_embs = id_emb
        self._lstt_forward(img_embs, id_emb, st)
        # lstt_long_memories of a reference frame = its own fused K/V (transformer.py:337-341)
        if self._claim_memory_frame():
            self._bank_reserve(self.enc_hw)
            self._append_short_to_bank(st)
            self.bank_len = self._bank_len_after_store()
        self.last_mem_step = self.frame_step
        self._have_lstt = True

    @_in_precision
    def match_propogate_one_frame(self, img=None, img_embs=None):
        offline = img_embs is None and self.enable_offline_enc
        if offline:
            self._offline_step(self.frame_step + 1)
        self.frame_step += 1
        st = torch.cuda.current_stream().cuda_stream
        if offline:
            img_embs = self._offline_embs(self.frame_step, st)   # the stored frame; an image handed here is ignored
        elif img_embs is None:
            self._check_img(img)
            img_embs = self._encode(img, st)
        self.curr_enc_embs = img_embs
        splits = lt_splits(self.enc_hw, self._plan().H, max(self.bank_len, 1)) if getattr(self, "_tc", False) else 0
        if getattr(self, "_gp_tc", False):
            splits = self._gp_splits(self.bank_len)       # the fused DeAOT kernel's split count is part of the captured body
        if self._usage():
            splits = "usage"                              # one split per memory slot, whatever the live count
        if self.kv_shard is not None:
            # sharded bank: the captured body also depends on the shard split count (a function of the GLOBAL memory-frame
            # count, identical on every rank) and on whether this rank holds any memory frame yet
            splits = ("shard", self._shard_splits(), self.bank_len > 0, SHARD_XCHG)
        self.graphs.run(("lstt", splits, img_embs.nhwc[-1].data_ptr()),
                        lambda: self._lstt_forward(img_embs, None, _cur_stream()),
                        enabled=self.short_term_mem_skip <= 1 and (self.kv_shard is None or SHARD_GRAPHS))

    @_in_precision
    def update_short_term_memory(self, curr_mask, curr_id_emb=None, skip_long_term_update=False):
        st = torch.cuda.current_stream().cuda_stream
        append = False
        if self.frame_step - self.last_mem_step >= self.long_term_mem_gap:
            append = not skip_long_term_update
            self.last_mem_step = self.frame_step
        append = append and self._claim_memory_frame()       # sharded bank: only the owner rank stores this memory frame
        if append:
            self._bank_reserve(self.enc_hw)          # may re-allocate (and drop graphs) before anything is captured
        ws = self._ws
        label_map = curr_id_emb is None and not (curr_mask.dim() == 4 and curr_mask.shape[1] != 1) and \
            tuple(curr_mask.shape[-2:]) == tuple(ws.mask.shape)
        if label_map and self.short_term_mem_skip <= 1:
            m2 = curr_mask.reshape(ws.mask.shape).float().contiguous()
            ops.eltwise(ops.EW_COPY, m2, None, ws.mask, stream=st)

            def body():
                s2 = _cur_stream()
                self._id_from_static_mask(ws.mask, s2)
                self._fuse_memories(ws.id_emb, s2)
                if append:
                    self._append_short_to_bank(s2)
            self.graphs.run(("upd", append), body)
        else:
            id_emb = self.assign_identity_from_mask(curr_mask, st) if curr_id_emb is None else curr_id_emb
            self._fuse_memories(id_emb, st)
            if append:
                self._append_short_to_bank(st)
        if append:
            self.bank_len = self._bank_len_after_store()

    def _bank_len_after_store(self):
        """Host copy of the live row count: one more frame, saturating at the capacity of a bounded bank."""
        n = self.bank_len + self.enc_hw
        return n if self.long_term_mem_max is None else min(n, self.bank_cap)

    def _claim_memory_frame(self):
        """Count one more memory frame (global count, all shards) and say whether THIS rank stores it: always without
        sharding, rank `f % world` for memory frame f with the bank sharded (SURVEY 8e.2)."""
        f = self._mem_frames
        self._mem_frames += 1
        return self.kv_shard is None or f % self.kv_shard[1] == self.kv_shard[0]

    def _append_short_to_bank(self, st):
        """Append the newest fused K/V of every layer at the device-side row counter, then advance it (kernels only: the
        host-side row count and capacity are the caller's business, so the body can be captured in a graph)."""
        N = self.enc_hw
        K_src, V_src = self._latest_kv()
        if self.long_term_mem_max is not None:
            # bounded: one launch per layer writes the fp32 rows and the packed rows of the selected attention kernel at the
            # ring's write offset, then both counters move (the first frame's slot is never the wrap target)
            packed = (self.bank_Kp, self.bank_Vp) if self._tc else (self.bank_gpK, self.bank_gpV) if self._gp_tc else None
            if self._usage():          # the write offset becomes the next free slot, or the least-attended unpinned one
                ops.ring_select_usage(self.tk_dev, self.wr_dev, self._ws.usage_U, self._ws.usage_A, N, self.bank_cap, N,
                                      stream=st)
            for li in range(self._plan().L):
                ops.bank_ring_store(K_src[li], V_src[li], self.bank_K[li], self.bank_V[li],
                                    packed[0][li] if packed else None, packed[1][li] if packed else None, self.wr_dev, stream=st)
            ops.ring_advance(self.tk_dev, self.wr_dev, N, self.bank_cap, N, stream=st)
            return
        off = self.tk_dev
        for li in range(self._plan().L):
            ops.bank_append(K_src[li], self.bank_K[li], 0, offset_dev=off, stream=st)
            ops.bank_append(V_src[li], self.bank_V[li], 0, offset_dev=off, stream=st)
            if self._tc:
                ops.tc_pack_rows(K_src[li], self.bank_Kp[li], 0, row_off_dev=off, stream=st)
                ops.tc_pack_rows(V_src[li], self.bank_Vp[li], 0, row_off_dev=off, stream=st)
            if self._gemm_lt:
                ops.split_rows(K_src[li], self.bank_Kh[li], self.bank_Kl[li], row_off_dev=off, stream=st)
                ops.split_cols(V_src[li], self.bank_VhT[li], self.bank_VlT[li], col_off_dev=off, stream=st)
            if getattr(self, "_gp_tc", False):
                ops.tc_pack_rows(K_src[li], self.bank_gpK[li], 0, row_off_dev=off, stream=st)
                ops.tc_pack_rows(V_src[li], self.bank_gpV[li], 0, row_off_dev=off, stream=st)
        ops.counter_add(off, N, stream=st)

    def _latest_kv(self):
        return self._new_K, self._new_V

    # ------------------------------------------------------------------ LSTT (AOT)
    def _lstt_forward(self, embs, id_emb, st):
        P = self._plan()
        stK, stV = (self.st_K, self.st_V) if id_emb is None else self._next_short_slot()
        aot_lstt(P, self._ws, embs.nhwc[-1].view(self.enc_hw, P.C), self.pos_emb, self.enc_size_2d, 1, stK, stV, id_emb,
                 self._attend_own, self._attend_bank, self._local_attention, st)
        if id_emb is not None:
            self._commit_short_slot(stK, stV)
        self._have_lstt = True

    def _attend_own(self, Q, K, V, out, st, long_term):
        """softmax(Q K^T / T) V over the frame's own K / V: the self-attention, or (long_term) a reference frame's
        long-term step (transformer.py:337-341), which LT_PROBE times."""
        P = self._plan()
        d = P.C // P.H
        with _lt_probe(long_term, Q, self.enc_hw, P.C):
            if self._tc:
                self._tc_attention(Q, K, V, None, None, self.enc_hw, out, st)
            else:
                ops.attention(Q, K, V, out, P.H, d, d, Tk=self.enc_hw, stream=st)

    def _attend_bank(self, li, Q, out, st):
        """The long-term step of a propagated frame over layer li's bank."""
        P = self._plan()
        d = P.C // P.H
        if self._tc:
            ops.tc_pack_rows(Q, self._ws.Qp, 0, div=math.sqrt(d), stream=st)      # Q / T (attention.py:82)
        elif self.kv_shard is not None:
            raise ops.AotbError("sharded long-term bank needs the tensor-core attention kernel (8 heads x 32); this model's "
                                "head shape runs on the fp32 kernel, which has no partial (m, l, O) outputs")
        with _lt_probe(True, Q, self.bank_len, P.C):
            if not self._tc:
                ops.attention(Q, self.bank_K[li], self.bank_V[li], out, P.H, d, d, Tk=self.bank_len, Tk_dev=self.tk_dev,
                              stream=st)
            elif self.kv_shard is not None:
                self._sharded_attention(li, out, st)
            elif self._usage():
                self._usage_attention(li, self._ws.Qp, self.bank_Kp[li], self.bank_Vp[li], out, st)
            else:
                self._tc_attention(None, None, None, self.bank_Kp[li], self.bank_Vp[li], self.bank_len, out, st,
                                   Tk_dev=self.tk_dev)

    def _local_attention(self, li, Q, K, V, out, st):
        P = self._plan()
        Lw = P.layers[li]
        h, w = self.enc_size_2d
        d = P.C // P.H
        if d == 32 and LOCAL_IMPL in ops.LOCAL_KERNELS:
            with ops.local_kernel(LOCAL_IMPL):
                ops.local_attention_tile(Q, K, V, Lw.relk_w, Lw.relk_b, Lw.relv_t, out, h, w, P.H, stream=st)
        else:
            ops.local_attention(Q, K, V, Lw.relk_w, Lw.relk_b, Lw.relv, out, h, w, P.H, d, d, stream=st)

    def _tc_attention(self, Q, K, V, Kp, Vp, Tk, out, st, Tk_dev=None):
        """softmax(Q K^T / T) V on the tensor-core kernel.  Q/K/V fp32 [rows, C] are packed into the split-fp16
        operand buffers first unless already-packed banks (Kp, Vp) are given (then Q was packed by the caller)."""
        P = self._plan()
        ws = self._ws
        d = P.C // P.H
        N = self.enc_hw
        if Q is not None:
            ops.tc_pack_rows(Q, ws.Qp, 0, div=math.sqrt(d), stream=st)
        if Kp is None:
            ops.tc_pack_rows(K, ws.saKp, 0, stream=st)
            ops.tc_pack_rows(V, ws.saVp, 0, stream=st)
            Kp, Vp = ws.saKp, ws.saVp
        splits = lt_splits(N, P.H, Tk)
        part = _split_partials(ws.part, splits, N, P.H, P.C, out.device) if splits > 1 else None
        exact = LT_IMPL == "tc_exact" and self.precision == "fp32"
        ops.lt_attention_tc(ws.Qp, Kp, Vp, N, Tk, O=out, Tk_dev=Tk_dev, splits=splits, exact=exact, part=part, stream=st)

    def _usage_attention(self, li, Qp, Kp, Vp, out, st):
        """Usage mode: the long-term attention over the bank with one KV split per memory slot (packed Q given), merged by
        the kernel that also adds each slot's attention mass to U; layer 0's merge ticks A for the live slots."""
        P = self._plan()
        ws = self._ws
        M, N = self.long_term_mem_max, self.enc_hw
        if P.deaot:
            H = 1
            ops.gp_attention_tc_slots(Qp, Kp, Vp, N, self.tk_dev, M, N, ws.usage_part, exact=self.precision == "fp32",
                                      stream=st)
        else:
            H = P.H
            ops.lt_attention_tc_slots(Qp, Kp, Vp, N, self.tk_dev, M, N, ws.usage_part,
                                      exact=LT_IMPL == "tc_exact" and self.precision == "fp32", stream=st)
        ops.attn_merge_usage(*ws.usage_part, out, H, out.shape[1] // H, ws.usage_U, ws.usage_A if li == 0 else None,
                             self.tk_dev, N, P.L, ws.usage_ws, stream=st)

    def _shard_splits(self):
        """KV-split count of the per-rank partial attention in sharded mode: a function of the GLOBAL memory-frame count, so it
        is identical on every rank (the exchanged buffers must have the same shape everywhere)."""
        world = self.kv_shard[1]
        frames_per_rank = (self._mem_frames + world - 1) // world
        s = max(2, lt_splits(self.enc_hw, self._plan().H, max(frames_per_rank, 1) * self.enc_hw))
        if s > SHARD_SMAX:
            raise ops.AotbError(f"sharded long-term attention: {s} KV splits exceed the exchange buffer capacity {SHARD_SMAX}")
        return s

    def _sharded_attention(self, li, out, st):
        """Split-KV over ranks (SURVEY 8e.2): local partials -> ONE all-gather of the packed [O | m | l] block -> exact LSE
        merge straight out of the gathered buffer (per-rank slices, no re-layout).  Q was packed by the caller."""
        import torch.distributed as dist
        rank, world, group = self.kv_shard
        P = self._plan()
        ws = self._ws
        N, C, H = self.enc_hw, P.C, P.H
        splits = self._shard_splits()                                            # identical on every rank
        if st != torch.cuda.current_stream().cuda_stream:
            raise ops.AotbError("sharded long-term attention must run on torch's current stream (the collective / the "
                                "symmetric-memory barrier are issued there)")
        if SHARD_XCHG == "p2p":
            return self._sharded_attention_p2p(li, out, st, splits)
        key = ("shard", splits)
        bufs = ws.part.get(key)
        if bufs is None:
            nO, nM = splits * N * C, splits * H * N
            mine = torch.empty(nO + 2 * nM, dtype=torch.float32, device=out.device)
            allr = torch.empty(world * (nO + 2 * nM), dtype=torch.float32, device=out.device)
            sl = lambda t: (t[:nO].view(splits, N, C), t[nO:nO + nM].view(splits, H, N), t[nO + nM:].view(splits, H, N))
            per_rank = [sl(allr[r * (nO + 2 * nM):(r + 1) * (nO + 2 * nM)]) for r in range(world)]
            bufs = ws.part[key] = (mine, allr, sl(mine), per_rank)
        mine, allr, (Op, Mp, Lp), per_rank = bufs
        if self.bank_len > 0:
            ops.lt_attention_tc(ws.Qp, self.bank_Kp[li], self.bank_Vp[li], N, self.bank_len, O=None, Tk_dev=self.tk_dev,
                                splits=splits, exact=(LT_IMPL == "tc_exact"), part=(Op, Mp, Lp), stream=st, merge=False)
        else:                                  # this rank holds no memory frame yet: neutral partial
            ops.eltwise(ops.EW_FILL, None, None, mine[:Op.numel()].view(1, -1), scalar=0.0, stream=st)
            ops.eltwise(ops.EW_FILL, None, None, Mp.view(1, -1), scalar=float("-inf"), stream=st)
            ops.eltwise(ops.EW_FILL, None, None, Lp.view(1, -1), scalar=0.0, stream=st)
        dist.all_gather_into_tensor(allr, mine, group=group)
        ops.attn_merge_peers([v[0] for v in per_rank], [v[1] for v in per_rank], [v[2] for v in per_rank], out, splits, H,
                             C // H, stream=st)

    def _sharded_attention_p2p(self, li, out, st, splits):
        """Exchange over peer memory: the local partials are written into this rank's slice of a symmetric allocation, one
        device-side barrier makes every rank's partials of this layer visible, and the merge kernel reads all ranks'
        partials in place (NVLink P2P loads).  One allocation per layer, so the next write of a buffer (this layer, next
        frame) is separated from its readers by the barriers of the other layers; single-layer models add a second barrier."""
        rank, world, group = self.kv_shard
        P = self._plan()
        ws = self._ws
        N, C, H = self.enc_hw, P.C, P.H
        key = ("p2p", li)
        buf = ws.part.get(key)
        if buf is None:
            nO, nM = SHARD_SMAX * N * C, SHARD_SMAX * H * N
            hdl, view = _symm_alloc(nO + 2 * nM, out.device, group)
            views = [(view(r, (SHARD_SMAX, N, C), 0), view(r, (SHARD_SMAX, H, N), nO), view(r, (SHARD_SMAX, H, N), nO + nM))
                     for r in range(world)]
            buf = ws.part[key] = (hdl, views)
        hdl, views = buf
        Op, Mp, Lp = (t[:splits] for t in views[rank])
        if self.bank_len > 0:
            ops.lt_attention_tc(ws.Qp, self.bank_Kp[li], self.bank_Vp[li], N, self.bank_len, O=None, Tk_dev=self.tk_dev,
                                splits=splits, exact=(LT_IMPL == "tc_exact"), part=(Op, Mp, Lp), stream=st, merge=False)
        else:                                  # this rank holds no memory frame yet: neutral partial
            ops.eltwise(ops.EW_FILL, None, None, Op.reshape(1, -1), scalar=0.0, stream=st)
            ops.eltwise(ops.EW_FILL, None, None, Mp.reshape(1, -1), scalar=float("-inf"), stream=st)
            ops.eltwise(ops.EW_FILL, None, None, Lp.reshape(1, -1), scalar=0.0, stream=st)
        hdl.barrier()
        ops.attn_merge_peers([v[0] for v in views], [v[1] for v in views], [v[2] for v in views], out, splits, H, C // H,
                             stream=st)
        if P.L < 2:
            hdl.barrier()

    # short-term memory slots (TEST_SHORT_TERM_MEM_SKIP ring, aot_engine.py:329-332)
    def _next_short_slot(self):
        if self.short_term_mem_skip <= 1:
            return self.st_K, self.st_V
        K = [torch.empty_like(t) for t in self.st_K]
        V = [torch.empty_like(t) for t in self.st_V]
        return K, V

    def _commit_short_slot(self, K, V, reset=True):
        self._new_K, self._new_V = K, V
        if self.short_term_mem_skip <= 1:
            return
        if reset:
            self._st_ring = [(K, V)]
        else:
            self._st_ring.append((K, V))
            self._st_ring = self._st_ring[-self.short_term_mem_skip:]
        self.st_K, self.st_V = self._st_ring[0]

    def _fuse_memories(self, id_emb, st):
        K, V = self._next_short_slot()
        aot_fuse_memories(self._plan(), self._ws, id_emb, K, V, st)
        self._commit_short_slot(K, V, reset=False)

    def _decode(self, st):
        x4, x8, x16, _ = self.curr_enc_embs.nhwc
        return fpn_decode(self._plan(), self._ws.cat.view(1, *self.enc_size_2d, -1), x4, x8, x16, self._dec_bufs,
                          self._ws.gn_ws, st)

    @_in_precision
    def decode_current_logits(self, output_size=None):
        """aot_engine.py:356-380.  The returned tensor (and ``pred_id_logits``) are per-engine static buffers that
        the next call overwrites -- clone them to keep a frame's logits."""
        P = self._plan()
        size = None if output_size is None else (int(output_size[0]), int(output_size[1]))
        obj = int(self.obj_nums[0])

        def body():
            st = _cur_stream()
            lg = self._decode(st)
            h4, w4, NC = lg.shape[1], lg.shape[2], lg.shape[3]
            bufs = self._dec_out.get(size)
            if bufs is None:
                lo = torch.empty((1, NC, h4, w4), dtype=torch.float32, device=lg.device)
                out = None if size is None else torch.empty((1, NC) + size, dtype=torch.float32, device=lg.device)
                bufs = self._dec_out[size] = (lo, out)
            ops.logits_postproc(lg, bufs[0], bufs[1], obj, P.align_corners, stream=st)
            return bufs

        # keyed on every encoder map the body reads: after restart_engine() a pooled sub-engine can decode the maps of a
        # different encoder, and the allocator may hand back only some of the blocks the captured graph points at
        enc_ptrs = tuple(t.data_ptr() for t in self.curr_enc_embs.nhwc[:3])
        lo, out = self.graphs.run(("dec", size, obj) + enc_ptrs, body)
        self.pred_id_logits = lo
        return lo if out is None else out

    def predict_current_mask(self, output_size=None, return_prob=False):
        """aot_engine.py:382-396 (argmax of the upsampled logits; fused K9 kernel)."""
        if output_size is None:
            output_size = self.input_size_2d
        st = torch.cuda.current_stream().cuda_stream
        oh, ow = int(output_size[0]), int(output_size[1])
        label = torch.empty((1, oh, ow), dtype=torch.float32, device=self.pred_id_logits.device)
        ops.logits_argmax(self.pred_id_logits, label, self._plan().align_corners, stream=st)
        if return_prob:
            raise NotImplementedError("return_prob is used by the training path only (SURVEY 8f)")
        return label.long()


class DeAOTEngine(AOTEngine):
    """networks/engines/deaot_engine.py:9-56 -- GatedPropagationModule stack (transformer.py:501-665)."""

    def __init__(self, aot_model, gpu_id=0, long_term_mem_gap=9999, short_term_mem_skip=1,
                 layer_loss_scaling_ratio=2., long_term_mem_max=None, precision=None, long_term_mem_policy=None):
        super().__init__(aot_model, gpu_id, long_term_mem_gap, short_term_mem_skip, long_term_mem_max=long_term_mem_max,
                         precision=precision, long_term_mem_policy=long_term_mem_policy)
        self.layer_loss_scaling_ratio = layer_loss_scaling_ratio

    def _lstt_forward(self, embs, id_emb, st):
        P = self._plan()
        stK, stV = (self.st_K, self.st_V) if id_emb is None else self._next_short_slot()
        deaot_lstt(P, self._ws, embs.nhwc[-1].view(self.enc_hw, P.C), self.enc_size_2d, 1, stK, stV, id_emb,
                   self._attend_own, self._attend_bank, self._local_attention, st)
        if id_emb is not None:
            self._commit_short_slot(stK, stV)
        self._have_lstt = True

    def _attend_own(self, Q, K, V, out, st, long_term):
        """softmax(Q K^T / T) V over the frame's own K / V: the gated self-attention, or (long_term) a reference frame's
        long-term step (transformer.py:614-616)."""
        if self._gp_tc:
            self._gp_attention(Q, K, V, None, None, self.enc_hw, None, out, st)
        else:
            ops.attention(Q, K, V, out, 1, self._kdim, self._vdim, Tk=self.enc_hw, stream=st)

    def _attend_bank(self, li, Q, out, st):
        """The long-term step of a propagated frame over layer li's bank, which LT_PROBE times."""
        ws = self._ws
        Tk = self.bank_len
        probe = LT_PROBE
        if probe is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        if self._gp_tc and self._usage():
            ops.tc_pack_rows(Q, ws.gpQp, 0, div=math.sqrt(self._kdim), stream=st)
            self._usage_attention(li, ws.gpQp, self.bank_gpK[li], self.bank_gpV[li], out, st)
        elif self._gp_tc:
            # fused wgmma kernel (gp_attn_tc.cu): 128 queries x 64 value channels per CTA, KV splits to fill the GPU
            self._gp_attention(Q, None, None, self.bank_gpK[li], self.bank_gpV[li], Tk, self.tk_dev, out, st)
        elif self._gemm_lt:
            # S = Q K^T -> softmax(S / T) over the live keys -> P V, all on the tensor-core GEMM (deaot_lt.cu)
            ops.linear_tc(Q, self.bank_Kh[li], self.bank_Kl[li], None, ws.S, stream=st)
            ops.row_softmax(ws.S, self._capw, Tk, 1.0 / math.sqrt(self._kdim), Tk_dev=self.tk_dev, stream=st)
            ops.linear_tc(ws.S, self.bank_VhT[li], self.bank_VlT[li], None, out, stream=st)
        else:
            ops.attention(Q, self.bank_K[li], self.bank_V[li], out, 1, self._kdim, self._vdim, Tk=Tk, Tk_dev=self.tk_dev,
                          stream=st)
        if probe is not None:
            e1.record()
            probe.append((e0, e1, 2.0 * self.enc_hw * Tk * (self._kdim + self._vdim)))   # FLOPs = 2*N*Tk*(d_qk + d_v), SURVEY 8d

    def _local_attention(self, li, Q, K, V, out, st):
        Lw = self._plan().layers[li]
        h, w = self.enc_size_2d
        if LOCAL_IMPL != "warp" and self._kdim == 128 and self._vdim == 1024:
            ops.local_gated_tile(Q, K, V, Lw.relk_w, Lw.relk_b, out, h, w, stream=st)
        else:
            ops.local_attention(Q, K, V, Lw.relk_w, Lw.relk_b, None, out, h, w, 1, self._kdim, self._vdim, stream=st)

    def _gp_attention(self, Q, K, V, Kp, Vp, Tk, Tk_dev, out, st):
        """softmax(Q K^T / T) V for the DeAOT head shape (1 x 128 / 1024) on the fused wgmma kernel.  Q fp32 [N, 128] is
        packed (with the 1/T of attention.py:672) here; K / V fp32 of the current frame are packed unless already-packed
        bank copies (Kp, Vp) are given."""
        ws = self._ws
        N = self.enc_hw
        ops.tc_pack_rows(Q, ws.gpQp, 0, div=math.sqrt(self._kdim), stream=st)
        if Kp is None:
            ops.tc_pack_rows(K, ws.gpSaK, 0, stream=st)
            ops.tc_pack_rows(V, ws.gpSaV, 0, stream=st)
            Kp, Vp = ws.gpSaK, ws.gpSaV
        splits = self._gp_splits(Tk)
        part = _split_partials(ws.gp_part, splits, N, 1, out.shape[1], out.device) if splits > 1 else None
        ops.gp_attention_tc(ws.gpQp, Kp, Vp, N, Tk, O=out, Tk_dev=Tk_dev, splits=splits, exact=self.precision == "fp32",
                            part=part, stream=st)

    def _gp_splits(self, Tk):
        """gp_splits over this engine's query rows."""
        return gp_splits(self.enc_hw, self._plan().C, Tk)

    def _fuse_memories(self, id_emb, st):
        """deaot_engine.py:20-45: K, V unchanged; ID_V = fuse_key_value_id(None, curr_ID_V, id_emb)."""
        K, V = self._next_short_slot()
        deaot_fuse_memories(self._plan(), self._ws, id_emb, K, V, st)
        self._commit_short_slot(K, V, reset=False)


# =====================================================================================
# multi-object facade (aot_engine.py:485-635)
# =====================================================================================
class AOTInferEngine(nn.Module):
    _engine_cls = AOTEngine

    def __init__(self, aot_model, gpu_id=0, long_term_mem_gap=9999, short_term_mem_skip=1, max_aot_obj_num=None,
                 long_term_mem_max=None, precision=None, long_term_mem_policy=None):
        """long_term_mem_max: bound of every sub-engine's long-term bank in memory frames; precision: "fp32" | "fp16" and
        long_term_mem_policy: "fifo" | "usage" of every sub-engine (see AOTEngine for all three)."""
        super().__init__()
        self.precision = _resolve_precision(aot_model, precision)
        self.cfg = aot_model.cfg
        self.AOT = aot_model
        if max_aot_obj_num is None or max_aot_obj_num > aot_model.max_obj_num:
            self.max_aot_obj_num = aot_model.max_obj_num
        else:
            self.max_aot_obj_num = max_aot_obj_num
        self.gpu_id = gpu_id
        self.long_term_mem_gap = long_term_mem_gap
        self.short_term_mem_skip = short_term_mem_skip
        self.long_term_mem_max = _resolve_mem_max(aot_model, long_term_mem_max)
        self.long_term_mem_policy = _resolve_mem_policy(aot_model, long_term_mem_policy, self.long_term_mem_max)
        self.aot_engines = []
        self._kv_shard = None
        self.restart_engine()

    def enable_kv_sharding(self, rank, world, group=None):
        """Shard the long-term memory bank over `world` ranks (see AOTEngine.enable_kv_sharding)."""
        if self.precision == "fp16":
            raise NotImplementedError("a long-term bank sharded over GPUs is not built for precision='fp16'")
        if self.long_term_mem_max is not None:
            raise NotImplementedError("a bounded long-term bank (long_term_mem_max) cannot be sharded over GPUs: each rank "
                                      "would need its own ring")
        self._kv_shard = (rank, world, group)
        for e in self.aot_engines:
            e.enable_kv_sharding(rank, world, group)

    def restart_engine(self):
        # keep the engines (and their device buffers) across videos; just reset their state
        for e in self.aot_engines:
            e._drop_offline_clip()         # a pooled engine does not keep the previous video's stored clip alive
        self._pool = getattr(self, "_pool", []) + list(self.aot_engines)
        self.aot_engines = []
        self.obj_nums = None
        self.enable_offline_enc = False
        self.offline_frames = -1
        self.total_offline_frame_num = 0

    # ------------------------------------------------------------------ > max_aot_obj_num objects (SURVEY 8 f.2)
    # ceil(objects / 10) sub-engines share one encoder pass.  Their LSTT / decoder / memory-update work is independent, so
    # every sub-engine after the first runs on its own side stream (forked from and joined to the caller's stream inside
    # each protocol call) and the small per-engine kernels overlap on the GPU instead of queueing behind one another as in
    # the reference's Python loop (aot_engine.py:584-630); mask separation and logit aggregation are one kernel each.
    def _run_engines(self, fn):
        """fn(index, engine) for every sub-engine; engine 0 on the current stream, the others concurrently on side streams."""
        return fork_join(self, self.aot_engines, fn)

    def separate_mask(self, mask, obj_nums):
        """aot_engine.py:515-545 -> (per-engine masks, per-engine object counts).  Label maps go through one kernel
        (ids [10e+1, 10e+10] -> 1..10 for engine e); the probability form ([K, ...] foreground stack) slices channels."""
        n = len(self.aot_engines)
        if mask is None:
            return [None] * n
        if n == 1:
            return [mask], [obj_nums]
        per = self.max_aot_obj_num
        counts = [per] * n
        if obj_nums % per > 0:
            counts[-1] = obj_nums % per
        if mask.dim() == 3 or mask.shape[0] == 1:
            m = mask.float().contiguous()
            out = torch.empty((n,) + tuple(m.shape), dtype=torch.float32, device=m.device)
            ops.separate_labels(m, out, per)
            return [out[e] for e in range(n)], counts
        probs = []
        for e in range(n):
            fg = mask[e * per + 1:(e + 1) * per + 1]
            probs.append(torch.cat([1. - fg.sum(dim=1, keepdim=True), fg], dim=1))
        return probs, counts

    def soft_logit_aggregation(self, all_logits):
        """aot_engine.py:565-582: identity for one engine, otherwise the fused aggregation kernel."""
        if len(all_logits) == 1:
            return all_logits[0]
        per = self.max_aot_obj_num
        first = all_logits[0]
        key = (len(all_logits), tuple(first.shape[-2:]))
        buf = getattr(self, "_agg_out", None)
        if buf is None or buf[0] != key:
            buf = self._agg_out = (key, torch.empty((1, 1 + len(all_logits) * per) + tuple(first.shape[-2:]),
                                                    dtype=torch.float32, device=first.device))
        return ops.soft_logit_aggregation([t if t.is_contiguous() else t.contiguous() for t in all_logits], buf[1], per)

    def _ensure_engines(self, want):
        """At least `want` sub-engines, from the pool first, each restarted for the new video."""
        while len(self.aot_engines) < want:
            eng = self._pool.pop(0) if self._pool else self._engine_cls(self.AOT, self.gpu_id, self.long_term_mem_gap,
                                                                       self.short_term_mem_skip,
                                                                       long_term_mem_max=self.long_term_mem_max,
                                                                       precision=self.precision,
                                                                       long_term_mem_policy=self.long_term_mem_policy)
            eng.long_term_mem_max = self.long_term_mem_max      # pooled engines too: part of their workspace key
            eng.long_term_mem_policy = self.long_term_mem_policy
            eng.restart_engine()
            eng.eval()
            if self._kv_shard is not None:
                eng.enable_kv_sharding(*self._kv_shard)
            self.aot_engines.append(eng)

    def offline_encoder(self, all_frames, all_masks=None):
        """Encode a stored clip once for every sub-engine (see AOTEngine.offline_encoder): sub-engine 0 holds the features
        and the stored label maps, the others are handed its features frame by frame (as in the per-frame path), and
        add_reference_frame(mask=None) separates the stored mask of its step among the sub-engines."""
        self._ensure_engines(1)
        first = self.aot_engines[0]
        first.offline_encoder(all_frames, all_masks)
        self.enable_offline_enc = True
        self.offline_frames = first.offline_frames
        self.total_offline_frame_num = first.total_offline_frame_num

    def add_reference_frame(self, img=None, mask=None, obj_nums=None, frame_step=-1):
        if isinstance(obj_nums, list):
            obj_nums = obj_nums[0]
        self.obj_nums = obj_nums
        want = max(-(-int(obj_nums) // self.max_aot_obj_num), 1)          # ceil(objects / max_aot_obj_num), at least one
        self._ensure_engines(want)
        first = self.aot_engines[0]
        if mask is None and first.enable_offline_enc and first.offline_masks is not None:
            mask = first.offline_masks[first._offline_step(first.frame_step if frame_step == -1 else frame_step)]
        masks, counts = self.separate_mask(mask, obj_nums)
        # engine 0 encodes the frame (or copies out its stored features); the others reuse its feature maps
        # (aot_engine.py:596-607)
        first.add_reference_frame(img, masks[0], obj_nums=[counts[0]], frame_step=frame_step)
        embs = first.curr_enc_embs
        if len(self.aot_engines) > 1:
            self._run_engines(lambda i, e: None if i == 0 else e.add_reference_frame(
                img, masks[i], obj_nums=[counts[i]], frame_step=frame_step, img_embs=embs))
        self.update_size()

    def match_propogate_one_frame(self, img=None):
        first = self.aot_engines[0]
        if len(self.aot_engines) == 1:
            return first.match_propogate_one_frame(img)
        st = torch.cuda.current_stream().cuda_stream
        if first.enable_offline_enc:
            embs = first._offline_embs(first.frame_step + 1, st)               # the stored frame, shared by all sub-engines
        else:
            first._check_img(img)
            embs = first._encode(img, st)       # shared by all sub-engines
        self._run_engines(lambda i, e: e.match_propogate_one_frame(img, img_embs=embs))

    def decode_current_logits(self, output_size=None):
        all_logits = self._run_engines(lambda i, e: e.decode_current_logits(output_size))
        return self.soft_logit_aggregation(all_logits)

    def update_memory(self, curr_mask, skip_long_term_update=False):
        masks, _ = self.separate_mask(curr_mask, self.obj_nums)
        self._run_engines(lambda i, e: e.update_short_term_memory(masks[i], skip_long_term_update=skip_long_term_update))

    # BASELINE.json's north_star names this method; the reference's real name is update_memory
    update_short_long_term_memory = update_memory

    def update_size(self):
        self.input_size_2d = self.aot_engines[0].input_size_2d
        self.enc_size_2d = self.aot_engines[0].enc_size_2d
        self.enc_hw = self.aot_engines[0].enc_hw

    @property
    def pred_id_logits(self):
        return self.aot_engines[0].pred_id_logits if self.aot_engines else None

    @property
    def long_term_memory_usage(self):
        """Every sub-engine's long_term_memory_usage (see AOTEngine), in sub-engine order."""
        return [e.long_term_memory_usage for e in self.aot_engines]


class DeAOTInferEngine(AOTInferEngine):
    _engine_cls = DeAOTEngine


_ENGINES = {("aotengine", "train"): AOTEngine, ("aotengine", "eval"): AOTInferEngine,
            ("deaotengine", "train"): DeAOTEngine, ("deaotengine", "eval"): DeAOTInferEngine}


def build_engine(name, phase='train', **kwargs):
    """networks/engines/__init__.py:5-21: same names, same keyword arguments, NotImplementedError for anything else."""
    cls = _ENGINES.get((name, phase))
    if cls is None:
        raise NotImplementedError
    return cls(**kwargs)
