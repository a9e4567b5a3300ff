"""CPU: the multi-video engines with more than 10 objects per video, driven through the emulated entry points
(tests/emu_multi_video_objects.py): videos of 1, 2 and 3 ID-bank lanes that open, close and gain lanes mid-video, against
one bounded AOTInferEngine / DeAOTInferEngine per video (logits, every lane's bank rows and ring counters); closes between
propagate and update that move lanes of several-lane videos; a tracer showing the captured bodies stay static; the one-lane
path issuing none of the lane entry points; and the refusals."""
import pytest
import torch

import emu_multi_video_objects as EMO
import test_cpu_graph_static as GS
import test_cpu_multi_video as MV
from oracle import aot_oracle as O
from oracle import weights as OW

H, W, M = MV.H, MV.W, MV.M
# video: (step it opens at, frames, objects, gap, (local frame, new object count) or None)
SCHEDULE = {0: (0, 7, 4, 2, (3, 11)), 1: (0, 5, 14, 1, None), 2: (1, 6, 23, 2, None), 3: (4, 4, 3, 1, (2, 12))}


def _clip(v, n, objs):
    return O.synthetic_video(n, H, W, objs, seed=70 + v)


def _drive(eng, schedule, refs_for=None, on_step=None):
    """MV._drive for videos of several lanes: a new object count may open a lane; labels fed back are the first reference
    engine's argmax (or the engine's own labels without references).  Returns the logits of every (step, video)."""
    total = {v: max(o, ev[1] if ev else 0) for v, (_, _, o, _, ev) in schedule.items()}
    clips = {v: _clip(v, n, total[v]) for v, (_, n, _, _, _) in schedule.items()}
    vids, local, refs, objs, trace = {}, {}, {}, {}, []
    with torch.no_grad():
        for step in range(20):
            for v, (t0, n, o, gap, _) in schedule.items():
                if step == t0:
                    frames, full = clips[v]
                    mask = torch.where(full <= o, full, torch.zeros_like(full))
                    vids[v] = eng.open_video(frames[0], mask, o, long_term_mem_gap=gap)
                    refs[v] = refs_for(gap) if refs_for else None
                    if refs[v] is not None:
                        refs[v].add_reference_frame(frames[0], mask, obj_nums=[o], frame_step=0)
                    local[v], objs[v] = 0, o
            for v in [v for v in vids if local[v] + 1 >= schedule[v][1]]:
                eng.close_video(vids.pop(v))
            if not vids and step > max(t0 for t0, *_ in schedule.values()):
                break
            if not vids:
                continue
            live = list(vids)
            for v in live:
                local[v] += 1
            eng.propagate({vids[v]: clips[v][0][local[v]] for v in live})
            for v in live:
                if refs[v] is not None:
                    refs[v].match_propogate_one_frame(clips[v][0][local[v]])
            got = eng.decode_current_logits((H, W))
            trace.append({v: got[vids[v]].clone() for v in live})
            lab = eng.decode_labels((H, W))
            labels = {}
            for v in live:
                g = got[vids[v]]
                assert g.shape[1] == (11 if objs[v] <= 10 else 1 + 10 * len(eng.video_lanes(vids[v])))
                assert torch.equal(lab[vids[v]], g.argmax(1)), v
                src = g
                if refs[v] is not None:
                    src = refs[v].decode_current_logits((H, W))
                    if on_step:
                        on_step("logits", v, g, src, objs[v])
                labels[v] = torch.argmax(src[:, :objs[v] + 1], dim=1, keepdim=True).float()
            for v in [v for v in live if schedule[v][4] and schedule[v][4][0] == local[v]]:
                objs[v] = schedule[v][4][1]
                m = labels[v].clone()
                full = clips[v][1]
                m = torch.where(full > schedule[v][2], full, m)         # the new ids keep their annotation
                eng.add_reference_frame(vids[v], clips[v][0][local[v]], m, objs[v])
                if refs[v] is not None:
                    refs[v].add_reference_frame(clips[v][0][local[v]], m, obj_nums=[objs[v]], frame_step=local[v])
                    if on_step:
                        on_step("logits", v, eng.decode_current_logits((H, W))[vids[v]],
                                refs[v].decode_current_logits((H, W)), objs[v])
            eng.update_memory({vids[v]: labels[v] for v in live})
            for v in live:
                if refs[v] is not None:
                    refs[v].update_memory(labels[v])
            if on_step:
                on_step("memory", eng, vids, refs, None)
    return trace


def _check_banks(eng, vids, refs):
    """Every lane's ring counters and bank rows equal its sub-engine's."""
    for v, vid in vids.items():
        lanes = eng.video_lanes(vid)
        assert len(lanes) == len(refs[v].aot_engines)
        mems = eng.lane_long_term_memories(vid)
        assert all(a is b or torch.equal(a, b) for a, b in zip(eng.long_term_memories[vid][0], mems[0][0]))
        for l, e, mem in zip(lanes, refs[v].aot_engines, mems):
            assert int(eng._pool.tk[l]) == int(e.tk_dev.item()) == e.bank_len
            assert int(eng._pool.wr[l]) == int(e.wr_dev.item())
            for li, (K, V) in enumerate(mem):
                assert torch.allclose(K, e.bank_K[li][:e.bank_len], atol=1e-5)
                assert torch.allclose(V, e.bank_V[li][:e.bank_len], atol=1e-5)


@pytest.mark.parametrize("family", ["aott", "deaott"])
def test_schedule_matches_one_engine_per_video(monkeypatch, family):
    from aot_benchmark_b200.engine import AOTInferEngine, DeAOTInferEngine
    from aot_benchmark_b200.multi_video import DeAOTMultiVideoInferEngine, MultiVideoInferEngine
    deaot = family == "deaott"
    EMO.install_engine(monkeypatch, deaot=deaot)
    model = MV._model(family, OW.build_state_dict(family, seed=5))
    cls, ref_cls = (DeAOTMultiVideoInferEngine, DeAOTInferEngine) if deaot else (MultiVideoInferEngine, AOTInferEngine)
    eng = cls(model, max_videos=4, long_term_mem_max=M, max_lanes=8)
    worst, lanes_seen = [0.0], set()

    def on_step(kind, a, b, c, objs):
        if kind == "logits":
            k = objs + 1
            worst[0] = max(worst[0], (b[:, :k] - c[:, :k]).abs().max().item())
            return
        _check_banks(a, b, c)
        lanes_seen.update(len(a.video_lanes(vid)) for vid in b.values())
    _drive(eng, SCHEDULE, lambda gap: ref_cls(model, long_term_mem_gap=gap, long_term_mem_max=M), on_step)
    assert lanes_seen == {1, 2, 3}
    assert worst[0] < 1e-4, f"max |dlogit| vs one bounded {ref_cls.__name__} per video = {worst[0]}"


def test_close_between_propagate_and_update_moves_lanes(monkeypatch):
    """A one-lane video closes between propagate and update and its lane is refilled by the last lane of a three-lane
    video; then a two-lane video closes the same way: the remaining videos decode, store and propagate as their own
    engines."""
    from aot_benchmark_b200.engine import AOTInferEngine
    from aot_benchmark_b200.multi_video import MultiVideoInferEngine
    EMO.install_engine(monkeypatch)
    model = MV._model("aott", OW.build_state_dict("aott", seed=7))
    eng = MultiVideoInferEngine(model, max_videos=3, long_term_mem_max=M, long_term_mem_gap=1, max_lanes=6)
    objs = [3, 14, 23]
    clips = [_clip(i, 4, o) for i, o in enumerate(objs)]
    refs = [AOTInferEngine(model, long_term_mem_gap=1, long_term_mem_max=M) for _ in objs]
    with torch.no_grad():
        vids = [eng.open_video(f[0], m, o) for (f, m), o in zip(clips, objs)]
        for r, (f, m), o in zip(refs, clips, objs):
            r.add_reference_frame(f[0], m, obj_nums=[o], frame_step=0)
        assert [eng.video_lanes(v) for v in vids] == [[0], [1, 2], [3, 4, 5]]
        live = [0, 1, 2]
        for t, closing in ((1, 0), (2, 1), (3, None)):
            eng.propagate({vids[i]: clips[i][0][t] for i in live})
            if closing is not None:
                eng.close_video(vids[closing])
                live.remove(closing)
            got = eng.decode_current_logits((H, W))
            labels = {}
            for i in live:
                refs[i].match_propogate_one_frame(clips[i][0][t])
                want = refs[i].decode_current_logits((H, W))
                d = (got[vids[i]][:, :objs[i] + 1] - want[:, :objs[i] + 1]).abs().max().item()
                assert d < 1e-4, (t, i, d)
                labels[i] = torch.argmax(want[:, :objs[i] + 1], dim=1, keepdim=True).float()
            if closing == 0:
                assert eng.video_lanes(vids[2]) == [3, 4, 0] and eng.videos == [vids[1], vids[2]]
            if closing == 1:
                assert eng.video_lanes(vids[2]) == [2, 1, 0] and eng.videos == [vids[2]]
            eng.update_memory({vids[i]: labels[i] for i in live})
            for i in live:
                refs[i].update_memory(labels[i])
            _check_banks(eng, {i: vids[i] for i in live}, {i: refs[i] for i in live})


def test_captured_bodies_are_static_with_lanes(monkeypatch):
    """The tracer of test_cpu_multi_video over the lane schedule: the LSTT, decoder and memory-update bodies (the gather
    reading the device lane table included) issue the captured launches over the captured memory at every replay."""
    import bounded_bank_support as BB
    import emu_multi_video as EMU
    import emu_ops
    from aot_benchmark_b200 import engine, ops
    from aot_benchmark_b200.multi_video import MultiVideoInferEngine
    EMO.install_engine(monkeypatch)
    names = set(emu_ops.EMULATED) | set(BB.EMULATED) | set(EMU.EMULATED) | set(EMO.EMULATED)
    for name in names:
        monkeypatch.setattr(ops, name, GS._traced(name, getattr(ops, name)))
    monkeypatch.setattr(engine, "GraphCache", GS.TracingGraphCache)
    GS.TracingGraphCache.replays = 0
    eng = MultiVideoInferEngine(MV._model("aott", OW.build_state_dict("aott", seed=6)), max_videos=4,
                                long_term_mem_max=M, long_term_mem_gap=2, max_lanes=8)
    first = _drive(eng, SCHEDULE)
    assert {k[0] for k in eng.graphs.slots} == {"lstt", "dec", "upd"}
    replays = GS.TracingGraphCache.replays
    assert replays > 10
    second = _drive(eng, SCHEDULE)
    assert GS.TracingGraphCache.replays > 2 * replays
    for a, b in zip(first, second):
        assert a.keys() == b.keys() and all(torch.equal(a[v], b[v]) for v in a)


def test_one_lane_path_calls_no_lane_entry_point(monkeypatch):
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200.multi_video import MultiVideoInferEngine
    EMO.install_engine(monkeypatch)

    def refuse(*a, **k):
        raise AssertionError("a lane entry point ran on the one-lane path")
    for name in EMO.EMULATED:
        monkeypatch.setattr(ops, name, refuse)
    eng = MultiVideoInferEngine(MV._model("aott", OW.build_state_dict("aott", seed=5)), max_videos=3,
                                long_term_mem_max=M, long_term_mem_gap=2, max_lanes=6)
    MV._drive(eng, MV.SCHEDULE)
    assert eng._pool.x16 is None


def test_refusals(monkeypatch):
    from aot_benchmark_b200.multi_video import DeAOTMultiVideoInferEngine, MultiVideoInferEngine
    EMO.install_engine(monkeypatch)
    model = MV._model("aott", OW.build_state_dict("aott", seed=5))
    for bad in (1, 2.5, "4"):
        with pytest.raises(ValueError, match="max_lanes"):
            MultiVideoInferEngine(model, max_videos=2, long_term_mem_max=M, max_lanes=bad)
    with pytest.raises(ValueError, match="max_lanes"):
        DeAOTMultiVideoInferEngine(MV._model("deaott", OW.build_state_dict("deaott", seed=5)), max_videos=3,
                                   long_term_mem_max=M, max_lanes=2)
    assert MultiVideoInferEngine(model, max_videos=2, long_term_mem_max=M).max_lanes == 2
    eng = MultiVideoInferEngine(model, max_videos=2, long_term_mem_max=M, max_lanes=3)
    frames, full = _clip(0, 3, 30)
    sub = lambda k: torch.where(full <= k, full, torch.zeros_like(full))
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="at most 80 objects"):
            MultiVideoInferEngine(model, max_videos=1, long_term_mem_max=M, max_lanes=9).open_video(frames[0], full, 81)
        with pytest.raises(NotImplementedError, match="at most 30 objects.*max_lanes=3"):
            eng.open_video(frames[0], full, 31)
        assert eng.videos == [] and eng._lanes == []                     # a failed open leaves no lane behind
        a = eng.open_video(frames[0], sub(14), 14)
        with pytest.raises(NotImplementedError, match="at most 10 objects"):
            eng.open_video(frames[0], sub(11), 11)
        assert eng.videos == [a] and len(eng._lanes) == 2
        b = eng.open_video(frames[0], sub(5), 5)
        with pytest.raises(NotImplementedError, match="at most 20 objects"):
            eng.add_reference_frame(a, frames[1], sub(21), 21)
        with pytest.raises(NotImplementedError, match="at most 10 objects"):
            eng.add_reference_frame(b, frames[1], sub(11), 11)
        assert eng.video_lanes(a) == [0, 1] and eng.video_lanes(b) == [2]
        eng.close_video(b)
        eng.add_reference_frame(a, frames[0], sub(30), 30)
        assert eng.video_lanes(a) == [0, 1, 2] and len(eng.lane_long_term_memories(a)) == 3
