"""TEST INFRASTRUCTURE ONLY: CPU emulations of the entry points that run DeAOT's gated propagation for several independent
videos in one launch (include/aotb200.h: aotb_gp_attn_tc_batched_f16x2, aotb_local_gated_tile_batched_f32).  Their
contract is that video b's rows equal the one-video entry point on video b's rows, so each emulation runs the one-video
emulation (tests/emu_ops.py) video by video.  Nothing under aot_benchmark_b200/ imports this module."""
import torch

import emu_multi_video
import emu_ops


def gp_attention_tc_batched(Qp, q_stride, Kp, Vp, kv_stride, n, N, Tk=0, Tk_dev=None, O=None, splits=1, exact=True,
                            part=None, stream=None):
    for b in range(n):
        q = Qp[:, b * q_stride:b * q_stride + N]
        k, v = Kp[:, b * kv_stride:(b + 1) * kv_stride], Vp[:, b * kv_stride:(b + 1) * kv_stride]
        tk = Tk_dev[b:b + 1] if Tk_dev is not None else None
        pb = None
        if splits > 1:
            pb = (torch.empty(splits, N, O.shape[1]), torch.empty(splits, 1, N), torch.empty(splits, 1, N))
        emu_ops.gp_attention_tc(q, k, v, N, Tk, O=O[b * N:(b + 1) * N], Tk_dev=tk, splits=splits, exact=exact, part=pb)
    return O


def local_gated_tile_batched(q, k, v, relk_w, relk_b, out, h, w, n, stream=None):
    m = h * w
    for b in range(n):
        r = slice(b * m, (b + 1) * m)
        emu_ops.local_gated_tile(q[r], k[r], v[r], relk_w, relk_b, out[r], h, w)
    return out


EMULATED = ("gp_attention_tc_batched", "local_gated_tile_batched")


def install_engine(monkeypatch):
    """emu_multi_video.install_engine and the two DeAOT multi-video entry points."""
    from aot_benchmark_b200 import ops
    emu_multi_video.install_engine(monkeypatch)
    for name in EMULATED:
        monkeypatch.setattr(ops, name, globals()[name])
