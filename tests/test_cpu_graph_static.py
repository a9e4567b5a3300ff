"""CPU: what a captured CUDA graph takes for granted, checked without a GPU.

A graph replays the launches of ONE execution of a body with the addresses, shapes and strides that execution saw.  The engine is
therefore only correct if every body it hands to `GraphCache.run` issues the same entry points over the same memory every time the
same key comes up -- across frames, bank growth, `restart_engine()` and a second video.  Here `GraphCache` is replaced by a tracer with
the same slot policy (first call eager, second call "captured", later calls "replayed"): capture records the sequence of
(entry point, tensor address / shape / stride) the body issued through the emulated C-ABI (tests/emu_ops.py), every replay runs the
body again and must reproduce that sequence exactly.  A tensor re-created outside the workspace (round 2: the position table, rebuilt
per video while the first video's graphs kept its old address) or launch arguments derived from host state that is not part of the key
fail here; on the GPU they would silently read stale memory."""
import functools

import pytest
import torch

from oracle import aot_oracle as O
from oracle import weights as OW

TRACE = None          # list being recorded, or None outside a body


def _sig(x):
    if isinstance(x, torch.Tensor):
        return ("T", x.data_ptr(), tuple(x.shape), tuple(x.stride()))
    if isinstance(x, (list, tuple)):
        return tuple(_sig(v) for v in x)
    return None        # scalars may legitimately differ between capture and replay (e.g. the host copy of a device counter)


def _traced(name, fn):
    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        if TRACE is not None:
            TRACE.append((name, tuple(_sig(a) for a in args), tuple((k, _sig(v)) for k, v in sorted(kwargs.items()))))
        return fn(*args, **kwargs)
    return wrapper


class TracingGraphCache:
    replays = 0

    def __init__(self):
        self.slots = {}

    def clear(self):
        self.slots.clear()

    def run(self, key, fn, enabled=True):
        global TRACE
        if not enabled:
            return fn()
        slot = self.slots.setdefault(key, [0, None])
        if slot[0] < 1:                       # warm-up call, eager
            slot[0] += 1
            return fn()
        assert TRACE is None, "graph bodies do not nest"
        TRACE = []
        try:
            out = fn()
            trace = TRACE
        finally:
            TRACE = None
        if slot[1] is None:
            slot[1] = trace                   # "capture"
        else:                                 # "replay": the launches must be the captured ones
            TracingGraphCache.replays += 1
            cap = slot[1]
            assert len(trace) == len(cap), f"graph {key}: {len(cap)} launches captured, this call issues {len(trace)}"
            for i, (a, b) in enumerate(zip(cap, trace)):
                assert a == b, f"graph {key}: launch {i} ({a[0]}) differs from the captured one:\n  captured {a}\n  now      {b}"
        return out


def _install(monkeypatch):
    import emu_ops
    from aot_benchmark_b200 import engine, ops
    emu_ops.install_engine(monkeypatch)
    for name in emu_ops.EMULATED:
        monkeypatch.setattr(ops, name, _traced(name, getattr(ops, name)))
    for name in ("separate_labels", "soft_logit_aggregation", "local_gated_tile"):
        if hasattr(emu_ops, name):
            monkeypatch.setattr(ops, name, _traced(name, getattr(emu_ops, name)))
    monkeypatch.setattr(engine, "GraphCache", TracingGraphCache)
    TracingGraphCache.replays = 0


def _engine(model_name, sd, gap):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", model_name)
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    model.load_state_dict(sd, strict=True)
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                       short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP)
    eng.eval()
    return eng


@pytest.mark.parametrize("model_name,lt_impl,deaot_lt,H,W,objs", [
    ("aott", "tc_exact", "tc", 97, 129, 3), ("aott", "simt", "tc", 97, 129, 3), ("aott", "tc_exact", "tc", 97, 129, 14),
    ("deaott", "tc_exact", "tc", 97, 129, 3), ("deaott", "tc_exact", "gemm", 97, 129, 3), ("deaott", "tc_exact", "simt", 97, 129, 12),
    ("r50_aotl", "tc_exact", "tc", 97, 129, 5), ("r50_deaotl", "tc_exact", "tc", 97, 129, 5), ("swinb_aotl", "tc_exact", "tc", 96, 128, 2)])
def test_captured_bodies_are_static_across_frames_bank_growth_and_videos(monkeypatch, model_name, lt_impl, deaot_lt, H, W, objs):
    from aot_benchmark_b200 import engine
    _install(monkeypatch)
    monkeypatch.setattr(engine, "LT_IMPL", lt_impl)
    monkeypatch.setattr(engine, "DEAOT_LT", deaot_lt)
    monkeypatch.setattr(engine, "BANK_INIT_FRAMES", 2)            # the bank is re-allocated mid-clip (graphs dropped, re-captured)
    sd = OW.build_state_dict(model_name, seed=4)
    eng = _engine(model_name, sd, 2)
    outs = []
    big = model_name.startswith(("r50", "swinb"))
    for video in range(2 if big else 3):                          # same geometry: buffers and "graphs" are kept
        frames, mask = O.synthetic_video(6 if big else 8, H, W, objs, seed=31)
        with torch.no_grad():
            lo, labels = O.run_video(eng, frames, mask, objs, (H, W))
        outs.append(lo)
    assert len(eng.aot_engines) == (objs + 9) // 10
    assert TracingGraphCache.replays > (8 if big else 20)
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    for a, b in zip(outs[0], outs[-1]):
        assert torch.equal(a, b)
    # a different geometry on the same engine: new workspace, new graphs, no stale trace
    frames, mask = O.synthetic_video(4, H - 16, W - 16, 2, seed=32)
    with torch.no_grad():
        O.run_video(eng, frames, mask, 2, (H - 16, W - 16))


def _sub_engine_logits(eng, frames, mask, objs, out_size):
    """run_video, keeping the merged logits and every sub-engine's pred_id_logits of every frame."""
    subs = []
    on_frame = lambda t, logit, label: subs.append([logit.clone()] + [e.pred_id_logits.clone() for e in eng.aot_engines])
    with torch.no_grad():
        O.run_video(eng, frames, mask, objs, out_size, on_frame=on_frame)
    return subs


@pytest.mark.parametrize("model_name", ["aott", "deaott"])
def test_sub_engine_reuse_across_videos_with_a_recycled_encoder_block(monkeypatch, model_name):
    """restart_engine() pools the sub-engines and the next video pops them in order, so in (A, 20 objects) -> (B, 3) ->
    (A, 20) the first video's follower owns the encoder in the third one, with a fresh _Encoder but its old workspace
    and graphs (same geometry, and 10 objects in both roles, so its decode graph's key can match).  Stand-in for the
    allocator handing back SOME of the freed blocks: the new encoder gets the old 4x feature tensor back and fresh 8x /
    16x ones.  Every graph the new owner replays must then read the new encoder's maps, and every video must equal a
    fresh engine running it alone."""
    from aot_benchmark_b200 import engine
    _install(monkeypatch)
    sd = OW.build_state_dict(model_name, seed=4)
    A, B = (97, 129), (129, 177)
    seq = [(A, 20), (B, 3), (A, 20), (A, 3), (B, 14)]
    clips = [O.synthetic_video(5, h, w, objs, seed=50 + i) for i, ((h, w), objs) in enumerate(seq)]
    eng = _engine(model_name, sd, 2)
    got = [_sub_engine_logits(eng, *clips[0], 20, A)]
    owner, follower = eng.aot_engines
    old_enc, old_x4 = owner._enc, owner.curr_enc_embs.nhwc[0]
    x4_key = next(k for k, v in old_enc.bufs.items() if v is old_x4)
    alloc = engine._Encoder._buf

    def recycled_buf(self, key, shape):
        if self is not old_enc and key == x4_key and key not in self.bufs and tuple(shape) == tuple(old_x4.shape):
            self.bufs[key] = old_x4                 # the freed 4x block comes back; 8x / 16x are new addresses
        return alloc(self, key, shape)
    monkeypatch.setattr(engine._Encoder, "_buf", recycled_buf)
    for i in range(1, len(seq)):
        (h, w), objs = seq[i]
        got.append(_sub_engine_logits(eng, *clips[i], objs, (h, w)))
        if i == 2:
            assert eng.aot_engines[0] is follower and follower._enc is not old_enc
            assert follower.curr_enc_embs.nhwc[0] is old_x4 and follower._ws_key is not None
    assert TracingGraphCache.replays > 20
    for i, ((h, w), objs) in enumerate(seq):
        alone = _sub_engine_logits(_engine(model_name, sd, 2), *clips[i], objs, (h, w))
        assert len(alone) == len(got[i])
        for f, (a, b) in enumerate(zip(got[i], alone)):
            assert len(a) == len(b) == 1 + (objs + 9) // 10
            for j, (x, y) in enumerate(zip(a, b)):
                assert torch.equal(x, y), f"video {i + 1}, frame {f + 1}, {'merged' if j == 0 else f'sub-engine {j - 1}'}"


def test_tracer_catches_a_per_video_tensor(monkeypatch):
    """The tracer itself: re-creating the position table per video (the round-2 bug) must be reported."""
    from aot_benchmark_b200 import engine
    _install(monkeypatch)
    sd = OW.build_state_dict("aott", seed=4)
    eng = _engine("aott", sd, 2)
    frames, mask = O.synthetic_video(4, 97, 129, 3, seed=31)
    keep = []
    with torch.no_grad():
        O.run_video(eng, frames, mask, 3, (97, 129))
        e0 = eng.aot_engines[0]
        keep.append(e0._ws.pos_emb)
        e0._ws.pos_emb = e0._ws.pos_emb.clone()                   # what restart_engine() + add_reference_frame() used to do
        with pytest.raises(AssertionError, match="differs from the captured one"):
            O.run_video(eng, frames, mask, 3, (97, 129))
