"""TEST INFRASTRUCTURE ONLY: CPU emulations of the entry points that run several independent videos in one launch
(include/aotb200.h: aotb_lt_attn_tc_batched_f16x2, aotb_local_attention_tc_batched_f32, aotb_id_embed_runs_batched_f32,
aotb_bank_ring_store_batched, aotb_ring_advance_batched).  Their contract is that video b's rows equal the one-video entry
point on video b's rows, so each emulation runs the one-video emulation (tests/emu_ops.py, tests/bounded_bank_support.py)
video by video.  Nothing under aot_benchmark_b200/ imports this module."""
import torch

import bounded_bank_support
import emu_batched
import emu_ops


def lt_attention_tc_batched(Qp, q_stride, Kp, Vp, kv_stride, n, N, Tk=0, Tk_dev=None, O=None, splits=1, exact=True,
                            part=None, stream=None):
    for b in range(n):
        q = Qp[:, b * q_stride:b * q_stride + N]
        k, v = Kp[:, b * kv_stride:(b + 1) * kv_stride], Vp[:, b * kv_stride:(b + 1) * kv_stride]
        tk = Tk_dev[b:b + 1] if Tk_dev is not None else None
        pb = None
        if splits > 1:
            pb = tuple(torch.empty_like(t[:, :N] if t.dim() == 3 and t.shape[1] == n * N else t[..., :N]) for t in part)
        emu_ops.lt_attention_tc(q, k, v, N, Tk, O=O[b * N:(b + 1) * N], Tk_dev=tk, splits=splits, exact=exact, part=pb)
    return O


def local_attention_tc_batched(q, k, v, relk_w, relk_b, relv_t, out, h, w, H, n, stream=None):
    m = h * w
    for b in range(n):
        r = slice(b * m, (b + 1) * m)
        emu_ops.local_attention_tile(q[r], k[r], v[r], relk_w, relk_b, relv_t, out[r], h, w, H)
    return out


def id_embed_runs_batched(masks, wp, bias, out, C, nid, ksize, stride, pad, ln_gamma=None, ln_beta=None, stream=None):
    n = masks.shape[0]
    m = out.shape[0] // n
    for b in range(n):
        emu_ops.id_embed_runs(masks[b], wp, bias, out[b * m:(b + 1) * m], C, nid, ksize, stride, pad, ln_gamma, ln_beta)
    return out


def bank_ring_store_batched(k_src, v_src, k_bank, v_bank, k_packed, v_packed, write_dev, store_dev, n, cap_rows, stream=None):
    rows = k_src.shape[0] // n
    for b in range(n):
        if int(store_dev[b]):
            c = slice(b * cap_rows, (b + 1) * cap_rows)
            bounded_bank_support.bank_ring_store(k_src[b * rows:(b + 1) * rows], v_src[b * rows:(b + 1) * rows], k_bank[c],
                                                 v_bank[c], k_packed[:, c], v_packed[:, c], write_dev[b:b + 1])


def ring_advance_batched(live_dev, write_dev, store_dev, n, rows, cap_rows, pinned_rows, stream=None):
    for b in range(n):
        if int(store_dev[b]):
            bounded_bank_support.ring_advance(live_dev[b:b + 1], write_dev[b:b + 1], rows, cap_rows, pinned_rows)


EMULATED = ("lt_attention_tc_batched", "local_attention_tc_batched", "id_embed_runs_batched", "bank_ring_store_batched",
            "ring_advance_batched")


def install_engine(monkeypatch):
    """bounded_bank_support.install_engine, the batched encoder emulations and the five multi-video entry points."""
    from aot_benchmark_b200 import ops
    bounded_bank_support.install_engine(monkeypatch)
    emu_batched.install(monkeypatch)
    for name in EMULATED:
        monkeypatch.setattr(ops, name, globals()[name])
