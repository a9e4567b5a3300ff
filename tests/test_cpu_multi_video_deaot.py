"""CPU: DeAOTMultiVideoInferEngine driven through the emulated entry points (tests/emu_multi_video_deaot.py) on the
four-video schedule of test_cpu_multi_video, against the float64 bounded oracle of each video (logits) and one bounded
DeAOTInferEngine per video (logits, bank rows and counters); a close between propagate and update_memory; a tracer showing
the captured bodies are static across frames, stores, opens, closes and videos; and the refused combinations."""
import pytest
import torch

import bounded_bank_support as BB
import emu_multi_video as EMU
import emu_multi_video_deaot as EMUD
import test_cpu_graph_static as GS
import test_cpu_multi_video as MV
from oracle import aot_oracle as O
from oracle import weights as OW

H, W, M = MV.H, MV.W, MV.M


def test_engine_matches_the_bounded_oracle_and_one_engine_per_video(monkeypatch):
    from aot_benchmark_b200.engine import DeAOTInferEngine
    from aot_benchmark_b200.multi_video import DeAOTMultiVideoInferEngine
    EMUD.install_engine(monkeypatch)
    sd = OW.build_state_dict("deaott", seed=5)
    model = MV._model("deaott", sd)
    eng = DeAOTMultiVideoInferEngine(model, max_videos=3, long_term_mem_max=M, long_term_mem_gap=2)
    worst = [0.0, 0.0]
    stores = [0]

    def refs_for(v, gap):
        return [BB.BoundedOracleEngine(sd, O.OracleConfig("deaott"), long_term_mem_gap=gap, dtype=torch.float64,
                                       long_term_mem_max=M),
                DeAOTInferEngine(model, long_term_mem_gap=gap, long_term_mem_max=M)]

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
            stores[0] = max(stores[0], e.bank_len // eng_._N)
            assert len(mem[vid]) == eng_._P.L
            for li, (K, V) in enumerate(mem[vid]):
                assert K.shape == (e.bank_len, 128) and V.shape == (e.bank_len, 1024)
                assert torch.allclose(K, e.bank_K[li][:e.bank_len], atol=1e-5)
                assert torch.allclose(V, e.bank_V[li][:e.bank_len], atol=1e-5)
    MV._drive(eng, MV.SCHEDULE, refs_for, on_step)
    assert stores[0] == M                                  # some bank filled up and wrapped
    assert worst[0] < 2e-4, f"max |dlogit| vs the float64 bounded oracle = {worst[0]}"
    assert worst[1] < 1e-4, f"max |dlogit| vs one bounded DeAOTInferEngine per video = {worst[1]}"


def test_close_between_propagate_and_update_moves_the_carried_state(monkeypatch):
    """propagate -> close_video(the middle video) -> update_memory: the video moved into the freed slot stores its own
    curr_Q / curr_V / curr_IDV, so its next frame still equals its own DeAOTInferEngine.  DeAOTS: two layers, so layer 1
    carries a curr_IDV."""
    from aot_benchmark_b200.engine import DeAOTInferEngine
    from aot_benchmark_b200.multi_video import DeAOTMultiVideoInferEngine
    EMUD.install_engine(monkeypatch)
    model = MV._model("deaots", OW.build_state_dict("deaots", seed=7))
    eng = DeAOTMultiVideoInferEngine(model, max_videos=3, long_term_mem_max=M, long_term_mem_gap=1)
    clips = [O.synthetic_video(3, H, W, 2 + i, seed=60 + i) for i in range(3)]
    refs = [DeAOTInferEngine(model, long_term_mem_gap=1, long_term_mem_max=M) for _ in clips]
    with torch.no_grad():
        vids = [eng.open_video(f[0], m, 2 + i) for i, (f, m) in enumerate(clips)]
        for i, (r, (f, m)) in enumerate(zip(refs, clips)):
            r.add_reference_frame(f[0], m, obj_nums=[2 + i], frame_step=0)
        eng.propagate({v: f[1] for v, (f, _) in zip(vids, clips)})
        eng.close_video(vids[1])
        labels = {}
        for i in (0, 2):
            refs[i].match_propogate_one_frame(clips[i][0][1])
            labels[i] = torch.argmax(refs[i].decode_current_logits((H, W))[:, :3 + i], dim=1, keepdim=True).float()
        assert eng.videos == [vids[0], vids[2]]
        eng.update_memory({vids[i]: labels[i] for i in (0, 2)})
        for i in (0, 2):
            refs[i].update_memory(labels[i])
            refs[i].match_propogate_one_frame(clips[i][0][2])
        eng.propagate({vids[i]: clips[i][0][2] for i in (0, 2)})
        got = eng.decode_current_logits((H, W))
        for i in (0, 2):
            want = refs[i].decode_current_logits((H, W))
            d = (got[vids[i]][:, :3 + i] - want[:, :3 + i]).abs().max().item()
            assert d < 1e-4, (i, d)


def test_captured_bodies_are_static_across_frames_stores_opens_closes_and_videos(monkeypatch):
    """The LSTT, decoder and memory-update bodies, run through a tracer with GraphCache's slot policy, issue the captured
    launches over the captured memory at every replay."""
    import emu_ops
    from aot_benchmark_b200 import engine, ops
    from aot_benchmark_b200.multi_video import DeAOTMultiVideoInferEngine
    EMUD.install_engine(monkeypatch)
    names = set(emu_ops.EMULATED) | set(BB.EMULATED) | set(EMU.EMULATED) | set(EMUD.EMULATED)
    for name in names:
        monkeypatch.setattr(ops, name, GS._traced(name, getattr(ops, name)))
    monkeypatch.setattr(engine, "GraphCache", GS.TracingGraphCache)
    GS.TracingGraphCache.replays = 0
    sd = OW.build_state_dict("deaott", seed=6)
    eng = DeAOTMultiVideoInferEngine(MV._model("deaott", sd), max_videos=3, long_term_mem_max=M, long_term_mem_gap=2)
    first = MV._drive(eng, MV.SCHEDULE)
    keys = {k[0] for k in eng.graphs.slots}
    assert keys == {"lstt", "dec", "upd"}
    replays = GS.TracingGraphCache.replays
    assert replays > 20
    second = MV._drive(eng, MV.SCHEDULE)                   # the same videos again on the same engine: same results
    assert GS.TracingGraphCache.replays > 2 * replays
    for a, b in zip(first, second):
        assert a.keys() == b.keys() and all(torch.equal(a[v], b[v]) for v in a)


def test_refusals(monkeypatch):
    from aot_benchmark_b200 import engine, ops
    from aot_benchmark_b200.multi_video import DeAOTMultiVideoInferEngine, MultiVideoInferEngine
    EMUD.install_engine(monkeypatch)
    sd = OW.build_state_dict("deaott", seed=5)
    model = MV._model("deaott", sd)
    with pytest.raises(NotImplementedError, match="DeAOTMultiVideoInferEngine"):
        MultiVideoInferEngine(model, long_term_mem_max=M)
    with pytest.raises(NotImplementedError, match="MultiVideoInferEngine"):
        DeAOTMultiVideoInferEngine(MV._model("aott", OW.build_state_dict("aott", seed=5)), long_term_mem_max=M)
    with pytest.raises(ValueError, match="long_term_mem_max"):
        DeAOTMultiVideoInferEngine(model, max_videos=2)
    with pytest.raises(NotImplementedError, match="usage"):
        DeAOTMultiVideoInferEngine(MV._model("deaott", sd, TEST_LONG_TERM_MEM_POLICY="usage"), long_term_mem_max=M)
    with pytest.raises(NotImplementedError, match="usage"):
        DeAOTMultiVideoInferEngine(model, long_term_mem_max=M, long_term_mem_policy="usage")
    with pytest.raises(NotImplementedError, match="short_term_mem_skip"):
        DeAOTMultiVideoInferEngine(model, long_term_mem_max=M, short_term_mem_skip=2)
    DeAOTMultiVideoInferEngine(model, long_term_mem_max=M, long_term_mem_policy="fifo")
    for mod, knob, val, word in ((ops, "CONV_IMPL", "simt", "AOTB_CONV_IMPL=simt"),
                                 (engine, "DEAOT_LT", "gemm", "AOTB_DEAOT_LT=gemm"),
                                 (engine, "DEAOT_LT", "simt", "AOTB_DEAOT_LT=simt"),
                                 (engine, "LOCAL_IMPL", "warp", "AOTB_LOCAL_IMPL=warp")):
        with monkeypatch.context() as m:
            m.setattr(mod, knob, val)
            with pytest.raises(NotImplementedError, match=word):
                DeAOTMultiVideoInferEngine(model, long_term_mem_max=M)
    # the AOT engine's own kernel knobs do not concern the DeAOT engine
    for mod, knob, val in ((engine, "LT_IMPL", "simt"), (ops, "LT_VARIANT", "groups"), (engine, "LOCAL_IMPL", "tile")):
        with monkeypatch.context() as m:
            m.setattr(mod, knob, val)
            DeAOTMultiVideoInferEngine(model, long_term_mem_max=M)
    eng = DeAOTMultiVideoInferEngine(model, max_videos=1, long_term_mem_max=M)
    with pytest.raises(NotImplementedError, match="sharded"):
        eng.enable_kv_sharding(0, 2)
    frames, mask = O.synthetic_video(2, H, W, 2, seed=1)
    with pytest.raises(NotImplementedError, match="at most 10 objects"):
        eng.open_video(frames[0], mask, 11)
    with torch.no_grad():
        vid = eng.open_video(frames[0], mask, 2)
        with pytest.raises(NotImplementedError, match="at most 10 objects"):
            eng.add_reference_frame(vid, frames[1], mask, 11)
        with pytest.raises(ValueError, match="max_videos"):
            eng.open_video(frames[0], mask, 2)
        with pytest.raises(ValueError, match="exactly the open videos"):
            eng.propagate({vid + 1: frames[1]})
        eng.close_video(vid)
        with pytest.raises(KeyError):
            eng.close_video(vid)
