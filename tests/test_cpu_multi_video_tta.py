"""CPU: MultiVideoTTAInferEngine driven through the emulated entry points (tests/multi_video_tta_support.py): several copies
of the reference's TTA clips opened at different steps against the reference goldens (teacher-forced), a schedule with
evictions, per-video gaps, opens and closes at different steps and a new object against one bounded TTAInferEngine per video
(AOT and DeAOT), a tracer showing the pools' captured bodies are static, and the refused combinations."""
import pytest
import torch
import torch.nn.functional as F

import multi_video_tta_support as MT
import test_cpu_graph_static as GS
import test_cpu_tta_host as TH
import tta_support as S
from oracle import aot_oracle as O
from oracle import weights as OW

GOLDEN_CASES = ["aott_flip_ms", "r50_aotl_flip_ms3", "swinb_aotl_flip_ms"]


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_engine_vs_reference_golden(monkeypatch, golden_dir, name):
    """Three copies of the golden clip opened at steps 0, 1 and 2, the middle one closed two frames early, each teacher-forced
    with the reference's per-augmentation labels: every copy's ensemble, probabilities and per-augmentation labels pass
    test_cpu_tta_host's criteria."""
    from aot_benchmark_b200 import MultiVideoTTAInferEngine
    MT.install_engine(monkeypatch)
    g, sd, frames, first, new = S.load(golden_dir, name)
    T, H, W, flips = TH._frames(g), g["H"], g["W"], g["flips"]
    imgs = S.aug_images(g, frames[:T])
    ac = O.OracleConfig(g["model"]).MODEL_ALIGN_CORNERS
    mem = T                                                # >= the clip's memory frames: no eviction
    eng = MultiVideoTTAInferEngine(S.model(g["model"], sd), max_videos=3, long_term_mem_max=mem,
                                   long_term_mem_gap=g["gap"], flip=True, multi_scale=g["scales"])
    starts, ends = {0: 0, 1: 1, 2: 2}, {0: T, 1: T - 2, 2: T}
    vids, local = {}, {}
    bad_ens = bad_aug = checked = 0
    with torch.no_grad():
        for step in range(T + 2):
            for c in [c for c in vids if local[c] + 1 >= ends[c]]:
                eng.close_video(vids.pop(c))
            for c, t0 in starts.items():
                if step == t0:
                    vids[c] = eng.open_video(imgs[0], first, g["first_objs"])
                    local[c] = 0
            if not vids:
                break
            for c in vids:
                local[c] += 1
            nl = {vids[c]: new[local[c]] for c in vids if local[c] in new}
            forced = {vids[c]: [g["aug"][local[c] - 1, e] for e in range(len(flips))] for c in vids}
            objs = {vid: eng._video(vid)["obj"] for vid in vids.values()}           # the count the frame is decoded at
            out = eng.propagate({vids[c]: imgs[local[c]] for c in vids}, (H, W), new_labels=nl, keep_prob=True,
                                forced_labels=forced)
            for c, vid in vids.items():
                t, n_t = local[c], nl.get(vid)
                prob = eng.pred_prob[vid]
                bad_ens += S.outside_band(out[vid], g["ens"][t - 1], prob, new=n_t)
                if t in g["prob"]:
                    ref = g["prob"][t]
                    assert (prob[0, :ref.shape[0]] - ref).abs().max().item() < S.PROB_TOL
                    assert float(prob[0, ref.shape[0]:].abs().sum()) < 1e-6
                for e, f in enumerate(flips):
                    lo = MT.lowres(eng.aug_logits[vid][e], 0, objs[vid])
                    own, p = S.own_label(lo, (H, W), f, ac, new=n_t)
                    bad_aug += S.outside_band(own, g["aug"][t - 1, e], p, new=n_t)
                checked += 1
    assert checked == 2 * (T - 1) + max(T - 3, 1)
    assert bad_ens == 0 and bad_aug == 0, (bad_ens, bad_aug)


SH, SW, M = 49, 65, 2
SCALES = [1.0, 0.7]
# video: (step it opens at, frames, objects, gap, local frame where one more object appears)
SCHEDULE = {0: (0, 7, 2, 2, 3), 1: (1, 3, 3, 1, None), 2: (2, 6, 1, 3, None)}


def _aug(frame, scale, flip):
    h, w = round(SH * scale), round(SW * scale)
    x = frame if (h, w) == (SH, SW) else F.interpolate(frame, size=(h, w), mode="bilinear", align_corners=False)
    return torch.flip(x, dims=[3]) if flip else x


def _drive(eng, model, refs, seed=11, on_frame=None):
    """Run SCHEDULE through eng (and, when refs is a dict, one TTAInferEngine per video in refs) -> every frame's labels."""
    clips = {v: O.synthetic_video(n, SH, SW, objs, seed=seed + v) for v, (_, n, objs, _, _) in SCHEDULE.items()}
    aug = lambda f: [_aug(f, s, fl) for s in SCALES for fl in (False, True)]
    vids, local, objs, trace = {}, {}, {}, []
    with torch.no_grad():
        for step in range(20):
            for v in [v for v in vids if local[v] + 1 >= SCHEDULE[v][1]]:
                eng.close_video(vids.pop(v))
            for v, (t0, n, o, gap, _) in SCHEDULE.items():
                if step == t0:
                    frames, mask = clips[v]
                    vids[v] = eng.open_video(aug(frames[0]), mask, o, long_term_mem_gap=gap)
                    if refs is not None:
                        refs[v] = refs["make"](gap)
                        refs[v].add_reference_frame(aug(frames[0]), mask, obj_nums=[o], frame_step=0)
                    local[v], objs[v] = 0, o
            if not vids:
                break
            for v in vids:
                local[v] += 1
            nl = {}
            for v in vids:
                if SCHEDULE[v][4] == local[v]:
                    objs[v] += 1
                    m = torch.zeros(1, 1, SH, SW)
                    m[..., 5:15, 5:25] = objs[v]
                    nl[v] = m
            out = eng.propagate({vids[v]: aug(clips[v][0][local[v]]) for v in vids}, (SH, SW),
                                new_labels={vids[v]: m for v, m in nl.items()}, keep_prob=True)
            trace.append({v: (out[vids[v]].clone(), eng.pred_prob[vids[v]].clone()) for v in vids})
            if on_frame:
                on_frame(eng, vids, local, nl, out)
    return trace


@pytest.mark.parametrize("model_name", ["aott", "deaott"])
def test_engine_matches_one_bounded_tta_engine_per_video(monkeypatch, model_name):
    from aot_benchmark_b200 import MultiVideoTTAInferEngine, TTAInferEngine
    MT.install_engine(monkeypatch)
    model = S.model(model_name, OW.build_state_dict(model_name, seed=5))
    eng = MultiVideoTTAInferEngine(model, max_videos=3, long_term_mem_max=M, long_term_mem_gap=2, flip=True,
                                   multi_scale=SCALES)
    refs = {"make": lambda gap: TTAInferEngine(model, long_term_mem_gap=gap, long_term_mem_max=M, flip=True,
                                               multi_scale=SCALES)}
    worst, mism, frames = [0.0], [0], [0]

    def on_frame(eng_, vids, local, nl, out):
        clips = {v: O.synthetic_video(SCHEDULE[v][1], SH, SW, SCHEDULE[v][2], seed=11 + v) for v in vids}
        for v, vid in vids.items():
            f = clips[v][0][local[v]]
            k = refs[v].obj_nums + 1                                          # the count the frame is decoded at
            want = refs[v].propagate([_aug(f, s, fl) for s in SCALES for fl in (False, True)], (SH, SW),
                                     new_label=nl.get(v), keep_prob=True)
            for e in range(4):
                got = MT.lowres(eng_.aug_logits[vid][e], 0, 10)[:, :k]
                worst[0] = max(worst[0], (got - refs[v].aug_logits[e][:, :k]).abs().max().item())
            mism[0] += int((out[vid] != want).sum())
            assert eng_._video(vid)["obj"] == refs[v].obj_nums
            frames[0] += 1
    _drive(eng, model, refs, on_frame=on_frame)
    assert frames[0] == sum(n - 1 for _, n, _, _, _ in SCHEDULE.values())
    assert worst[0] < 1e-4, f"max |dlogit| vs one bounded TTAInferEngine per video = {worst[0]}"
    assert mism[0] == 0


def test_captured_bodies_are_static_across_frames_stores_opens_closes_and_events(monkeypatch):
    import emu_multi_video as EMU
    import emu_ops
    import bounded_bank_support as BB
    from aot_benchmark_b200 import MultiVideoTTAInferEngine, engine, ops
    MT.install_engine(monkeypatch)
    names = set(emu_ops.EMULATED) | set(BB.EMULATED) | set(EMU.EMULATED)
    for name in names:
        monkeypatch.setattr(ops, name, GS._traced(name, getattr(ops, name)))
    monkeypatch.setattr(engine, "GraphCache", GS.TracingGraphCache)
    # the encoder trim on open / close waits for the stream before dropping a batch size's graph
    monkeypatch.setattr(emu_ops._FakeStream, "synchronize", lambda self: None, raising=False)
    GS.TracingGraphCache.replays = 0
    model = S.model("aott", OW.build_state_dict("aott", seed=6))
    eng = MultiVideoTTAInferEngine(model, max_videos=3, long_term_mem_max=M, long_term_mem_gap=2, flip=True,
                                   multi_scale=SCALES)
    seen = [set() for _ in eng.pools]

    def keys(eng_, *_):
        for s, p in zip(seen, eng_.pools):
            s.update(k[0] for k in p.graphs.slots)
    first = _drive(eng, model, None, on_frame=keys)
    assert all(s == {"lstt", "dec", "upd"} for s in seen)
    # every video closed: the pools' encoders keep one frame, and the LSTT graphs over the dropped lane counts are gone
    assert all(k[0] != "lstt" for p in eng.pools for k in p.graphs.slots)
    replays = GS.TracingGraphCache.replays
    assert replays > 20
    second = _drive(eng, model, None)                      # the same videos again on the same engine: same results
    assert GS.TracingGraphCache.replays > 2 * replays
    for a, b in zip(first, second):
        assert a.keys() == b.keys()
        for v in a:
            assert torch.equal(a[v][0], b[v][0]) and torch.equal(a[v][1], b[v][1])


def test_refusals(monkeypatch):
    from aot_benchmark_b200 import MultiVideoTTAInferEngine, engine, ops
    MT.install_engine(monkeypatch)
    sd = OW.build_state_dict("aott", seed=5)
    model = S.model("aott", sd)
    mk = lambda m=model, **kw: MultiVideoTTAInferEngine(m, **{"long_term_mem_max": M, "flip": True,
                                                              "multi_scale": [1.0], **kw})
    with pytest.raises(ValueError, match="1 to 8 augmentations"):
        mk(multi_scale=[0.75, 1.0, 1.25, 1.5, 1.75])
    assert len(mk(multi_scale=[0.75, 1.0, 1.25, 1.5]).flips) == 8
    with pytest.raises(ValueError, match="long_term_mem_max"):
        MultiVideoTTAInferEngine(model, flip=True, multi_scale=[1.0])
    with pytest.raises(NotImplementedError, match="usage"):
        mk(long_term_mem_policy="usage")
    with pytest.raises(NotImplementedError, match="short_term_mem_skip"):
        mk(short_term_mem_skip=2)
    for mod, knob, val, word in ((engine, "LT_IMPL", "simt", "AOTB_LT_IMPL=simt"),
                                 (ops, "CONV_IMPL", "simt", "AOTB_CONV_IMPL=simt")):
        with monkeypatch.context() as m:
            m.setattr(mod, knob, val)
            with pytest.raises(NotImplementedError, match=word):
                mk()
    model.cfg.MODEL_USE_PREV_PROB = True
    with pytest.raises(NotImplementedError, match="evaluator.py:438"):
        mk()
    model.cfg.MODEL_USE_PREV_PROB = False
    eng = mk(max_videos=1)
    with pytest.raises(NotImplementedError, match="sharded"):
        eng.enable_kv_sharding(0, 2)
    frames, mask = O.synthetic_video(2, SH, SW, 2, seed=1)
    two = lambda f: [f, torch.flip(f, dims=[3])]
    with pytest.raises(NotImplementedError, match="at most 10 objects"):
        eng.open_video(two(frames[0]), mask, 11)
    with pytest.raises(ValueError, match="augmented images"):
        eng.open_video([frames[0]], mask, 2)
    # checked before any lane opens, also while the pools are empty: a flipped image of another size, a bad shape
    with pytest.raises(ValueError, match="unflipped image of its scale"):
        eng.open_video([frames[0], torch.zeros(1, 3, SH + 16, SW)], mask, 2)
    with pytest.raises(ValueError, match=r"\[1,3,h,w\]"):
        eng.open_video([frames[0], torch.zeros(3, SH, SW)], mask, 2)
    assert eng.videos == [] and all(p.videos == [] for p in eng.pools)
    # a failure inside a pool's open leaves no lane behind
    with monkeypatch.context() as m:
        m.setattr(type(eng.pools[0]), "_reference_pass",
                  lambda self, b, img, mask: (_ for _ in ()).throw(RuntimeError("reference pass failed")) if b == 1 else None)
        with pytest.raises(RuntimeError, match="reference pass failed"):
            eng.open_video(two(frames[0]), mask, 2)
    assert eng.videos == [] and all(p.videos == [] for p in eng.pools)
    with torch.no_grad():
        vid = eng.open_video(two(frames[0]), mask, 2)
        with pytest.raises(ValueError, match="max_videos"):
            eng.open_video(two(frames[0]), mask, 2)
        with pytest.raises(ValueError, match="exactly the open videos"):
            eng.propagate({vid + 1: two(frames[1])}, (SH, SW))
        with pytest.raises(ValueError, match="augmented images"):
            eng.propagate({vid: [frames[1]]}, (SH, SW))
        with pytest.raises(ValueError, match="original frame size"):
            eng.propagate({vid: two(frames[1])}, (SH + 16, SW))
        big = torch.zeros(1, 1, SH, SW)
        big[..., :4, :4] = 11
        with pytest.raises(NotImplementedError, match="at most 10 objects"):
            eng.propagate({vid: two(frames[1])}, (SH, SW), new_labels={vid: big})
        assert eng.frame_step(vid) == 0
        eng.propagate({vid: two(frames[1])}, (SH, SW))
        assert eng.frame_step(vid) == 1
        eng.close_video(vid)
        with pytest.raises(KeyError):
            eng.close_video(vid)
        eng2 = mk(max_videos=2)
        eng2.open_video(two(frames[0]), mask, 2)
        with pytest.raises(ValueError, match="original frame size"):
            eng2.open_video(two(frames[0]), torch.zeros(1, 1, SH + 16, SW), 2)
    deaot = S.model("deaott", OW.build_state_dict("deaott", seed=5))
    assert type(mk(deaot).pools[0]).__name__ == "DeAOTMultiVideoInferEngine"
    assert type(mk().pools[0]).__name__ == "MultiVideoInferEngine"
