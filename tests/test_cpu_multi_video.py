"""CPU: MultiVideoInferEngine driven through the emulated entry points (tests/emu_multi_video.py): videos of different
lengths that open and close at different steps, a new object mid-video, per-video long-term gaps and a close that compacts a
middle slot, against the bounded oracle of each video and one bounded AOTInferEngine per video (bank rows and counters); a
tracer showing the captured bodies are static across frames, stores, opens, closes and videos; and the refused
combinations."""
import pytest
import torch

import bounded_bank_support as BB
import emu_multi_video as EMU
import test_cpu_graph_static as GS
from oracle import aot_oracle as O
from oracle import weights as OW

H, W, M = 65, 81, 3
# video: (step it opens at, frames, objects, gap, local frame where one more object appears)
SCHEDULE = {0: (0, 9, 2, 2, 4), 1: (1, 5, 3, 1, None), 2: (2, 6, 1, 3, None), 3: (6, 4, 2, 2, 2)}


def _model(name, sd, **cfg_kw):
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    cfg = EngineConfig("t", name)
    for k, v in cfg_kw.items():
        setattr(cfg, k, v)
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    model.load_state_dict(sd, strict=True)
    return model


def _drive(eng, schedule, refs_for=None, on_step=None):
    """Run `schedule` through eng.  refs_for(v) -> per-video reference engines driven in lockstep (the first one's argmax is
    fed back to every engine); on_step(step, vids, local, refs, got) checks after each frame's memory update.  Returns the
    multi-video logits of every (step, video)."""
    clips = {v: O.synthetic_video(n, H, W, objs, seed=11 + v) for v, (_, n, objs, _, _) in schedule.items()}
    vids, local, refs, objs, trace = {}, {}, {}, {}, []
    with torch.no_grad():
        for step in range(20):
            for v, (t0, n, o, gap, _) in schedule.items():
                if step == t0:
                    frames, mask = clips[v]
                    vids[v] = eng.open_video(frames[0], mask, o, long_term_mem_gap=gap)
                    refs[v] = refs_for(v, gap) if refs_for else []
                    for r in refs[v]:
                        r.add_reference_frame(frames[0], mask, obj_nums=[o], frame_step=0)
                    local[v], objs[v] = 0, o
            for v in [v for v in vids if local[v] + 1 >= schedule[v][1]]:
                eng.close_video(vids.pop(v))               # its last frame was the previous step
            if not vids and step > max(t0 for t0, *_ in schedule.values()):
                break
            if not vids:
                continue
            live = list(vids)
            for v in live:
                local[v] += 1
            eng.propagate({vids[v]: clips[v][0][local[v]] for v in live})
            for v in live:
                for r in refs[v]:
                    r.match_propogate_one_frame(clips[v][0][local[v]])
            got = eng.decode_current_logits((H, W))
            trace.append({v: got[vids[v]].clone() for v in live})
            labels = {}
            for v in live:
                want = [r.decode_current_logits((H, W)) for r in refs[v]]
                src = want[0] if want else got[vids[v]]
                labels[v] = torch.argmax(src[:, :objs[v] + 1], dim=1, keepdim=True).float()
                if on_step:
                    on_step("logits", v, got[vids[v]], want, objs[v])
            lab = eng.decode_labels((H, W))
            if refs_for is None:
                for v in live:
                    assert torch.equal(lab[vids[v]], labels[v][:, 0].long())
            for v in [v for v in live if schedule[v][4] == local[v]]:      # one more object appears in this video
                objs[v] += 1
                m = labels[v].clone()
                m[..., 5:15, 5:15] = objs[v]
                eng.add_reference_frame(vids[v], clips[v][0][local[v]], m, objs[v])
                for r in refs[v]:
                    r.add_reference_frame(clips[v][0][local[v]], m, obj_nums=[objs[v]], frame_step=local[v])
                got_v = eng.decode_current_logits((H, W))[vids[v]]
                if on_step:
                    on_step("logits", v, got_v, [r.decode_current_logits((H, W)) for r in refs[v]], objs[v])
            eng.update_memory({vids[v]: labels[v] for v in live})
            for v in live:
                for r in refs[v]:
                    r.update_memory(labels[v])
            if on_step:
                on_step("memory", eng, vids, refs, None)
    return trace


def test_engine_matches_the_bounded_oracle_and_one_engine_per_video(monkeypatch):
    from aot_benchmark_b200.engine import AOTInferEngine
    from aot_benchmark_b200.multi_video import MultiVideoInferEngine
    EMU.install_engine(monkeypatch)
    sd = OW.build_state_dict("aott", seed=5)
    model = _model("aott", sd)
    eng = MultiVideoInferEngine(model, max_videos=3, long_term_mem_max=M, long_term_mem_gap=2)
    worst = [0.0, 0.0]

    def refs_for(v, gap):
        return [BB.BoundedOracleEngine(sd, O.OracleConfig("aott"), long_term_mem_gap=gap, dtype=torch.float64,
                                       long_term_mem_max=M),
                AOTInferEngine(model, long_term_mem_gap=gap, long_term_mem_max=M)]

    def on_step(kind, a, b, c, objs):
        if kind == "logits":
            got, (oracle, single) = b, c
            k = objs + 1
            worst[0] = max(worst[0], (got[:, :k].double() - oracle[:, :k]).abs().max().item())
            worst[1] = max(worst[1], (got[:, :k] - single[:, :k]).abs().max().item())
            return
        eng_, vids, refs = a, b, c
        mem = eng_.long_term_memories
        for slot, vid in enumerate(eng_.videos):
            v = next(k for k, x in vids.items() if x == vid)
            e = refs[v][1].aot_engines[0]
            assert int(eng_._pool.tk[slot]) == int(e.tk_dev.item()) == e.bank_len
            assert int(eng_._pool.wr[slot]) == int(e.wr_dev.item())
            for li, (K, V) in enumerate(mem[vid]):
                assert torch.allclose(K, e.bank_K[li][:e.bank_len], atol=1e-5)
                assert torch.allclose(V, e.bank_V[li][:e.bank_len], atol=1e-5)
    _drive(eng, SCHEDULE, refs_for, on_step)
    assert worst[0] < 2e-4, f"max |dlogit| vs the float64 bounded oracle = {worst[0]}"
    assert worst[1] < 1e-4, f"max |dlogit| vs one bounded AOTInferEngine per video = {worst[1]}"


def test_captured_bodies_are_static_across_frames_stores_opens_closes_and_videos(monkeypatch):
    """The LSTT, decoder and memory-update bodies, run through a tracer with GraphCache's slot policy, issue the captured
    launches over the captured memory at every replay."""
    import emu_batched  # noqa: F401  (installed by EMU.install_engine)
    import emu_ops
    from aot_benchmark_b200 import engine, ops
    from aot_benchmark_b200.multi_video import MultiVideoInferEngine
    EMU.install_engine(monkeypatch)
    names = set(emu_ops.EMULATED) | set(BB.EMULATED) | set(EMU.EMULATED)
    for name in names:
        monkeypatch.setattr(ops, name, GS._traced(name, getattr(ops, name)))
    monkeypatch.setattr(engine, "GraphCache", GS.TracingGraphCache)
    GS.TracingGraphCache.replays = 0
    sd = OW.build_state_dict("aott", seed=6)
    eng = MultiVideoInferEngine(_model("aott", sd), max_videos=3, long_term_mem_max=M, long_term_mem_gap=2)
    first = _drive(eng, SCHEDULE)
    keys = {k[0] for k in eng.graphs.slots}
    assert keys == {"lstt", "dec", "upd"}
    replays = GS.TracingGraphCache.replays
    assert replays > 20
    second = _drive(eng, SCHEDULE)                         # the same videos again on the same engine: same results
    assert GS.TracingGraphCache.replays > 2 * replays
    for a, b in zip(first, second):
        assert a.keys() == b.keys() and all(torch.equal(a[v], b[v]) for v in a)


def test_close_then_decode_reads_the_moved_video(monkeypatch):
    """propagate -> close_video(a middle video) -> decode: the video moved into the freed slot decodes its own features."""
    from aot_benchmark_b200.multi_video import MultiVideoInferEngine
    EMU.install_engine(monkeypatch)
    eng = MultiVideoInferEngine(_model("aott", OW.build_state_dict("aott", seed=7)), max_videos=3, long_term_mem_max=M)
    clips = [O.synthetic_video(2, H, W, 2, seed=40 + i) for i in range(3)]
    with torch.no_grad():
        vids = [eng.open_video(f[0], m, 2) for f, m in clips]
        eng.propagate({v: f[1] for v, (f, _) in zip(vids, clips)})
        before = {v: t.clone() for v, t in eng.decode_current_logits((H, W)).items()}
        eng.close_video(vids[1])
        after = eng.decode_current_logits((H, W))
    assert set(after) == {vids[0], vids[2]}
    for v in after:
        assert torch.equal(after[v], before[v]), v


def test_refusals(monkeypatch):
    from aot_benchmark_b200 import engine, ops
    from aot_benchmark_b200.multi_video import MultiVideoInferEngine
    EMU.install_engine(monkeypatch)
    sd = OW.build_state_dict("aott", seed=5)
    model = _model("aott", sd)
    with pytest.raises(ValueError, match="long_term_mem_max"):
        MultiVideoInferEngine(model, max_videos=2)
    with pytest.raises(NotImplementedError, match="DeAOT"):
        MultiVideoInferEngine(_model("deaott", OW.build_state_dict("deaott", seed=5)), long_term_mem_max=M)
    with pytest.raises(NotImplementedError, match="usage"):
        MultiVideoInferEngine(_model("aott", sd, TEST_LONG_TERM_MEM_POLICY="usage"), long_term_mem_max=M)
    with pytest.raises(NotImplementedError, match="usage"):
        MultiVideoInferEngine(model, long_term_mem_max=M, long_term_mem_policy="usage")
    with pytest.raises(ValueError, match="long_term_mem_policy"):
        MultiVideoInferEngine(model, long_term_mem_max=M, long_term_mem_policy="lru")
    MultiVideoInferEngine(model, long_term_mem_max=M, long_term_mem_policy="fifo")
    for mod, knob, val, word in ((engine, "LT_IMPL", "simt", "AOTB_LT_IMPL=simt"),
                                 (ops, "CONV_IMPL", "simt", "AOTB_CONV_IMPL=simt")):
        with monkeypatch.context() as m:
            m.setattr(mod, knob, val)
            with pytest.raises(NotImplementedError, match=word):
                MultiVideoInferEngine(model, long_term_mem_max=M)
    eng = MultiVideoInferEngine(model, max_videos=1, long_term_mem_max=M)
    with pytest.raises(NotImplementedError, match="sharded"):
        eng.enable_kv_sharding(0, 2)
    frames, mask = O.synthetic_video(2, H, W, 2, seed=1)
    with pytest.raises(NotImplementedError, match="at most 10 objects"):
        eng.open_video(frames[0], mask, 11)
    with torch.no_grad():
        vid = eng.open_video(frames[0], mask, 2)
        with pytest.raises(ValueError, match="max_videos"):
            eng.open_video(frames[0], mask, 2)
        with pytest.raises(ValueError, match="exactly the open videos"):
            eng.propagate({vid + 1: frames[1]})
        with pytest.raises(ValueError, match="network input size"):
            eng.propagate({vid: torch.zeros(1, 3, H + 16, W)})
        eng.close_video(vid)
        with pytest.raises(KeyError):
            eng.close_video(vid)
