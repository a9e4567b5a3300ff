"""GPU: videos of more than 10 objects in the multi-video engines.  The three lane entry points against the one-video launches
(bit for bit: lane gather against copies, batched separation against separate_labels, batched aggregation against
logits_postproc per lane + soft_logit_aggregation); the engines against the real reference's 14-object golden, against one
bounded AOTInferEngine / DeAOTInferEngine per video, graphs against eager, and closes that move lanes."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import aot_oracle as O
from oracle import weights as OW

pytestmark = pytest.mark.gpu
dev = "cuda"


def test_lane_gather_equals_copies():
    from aot_benchmark_b200 import ops
    g = torch.Generator(device=dev).manual_seed(3)
    nv, shapes = 3, [(17, 23, 24), (9, 12, 64), (5, 6, 256), (5, 6, 256)]
    src = [torch.randn((nv,) + s, device=dev, generator=g) for s in shapes]
    table = [2, 0, 2, 1, 0, 0]                        # repeated and out-of-order videos
    dst = [torch.full((8,) + s, -7.0, device=dev) for s in shapes]
    lanes = torch.tensor(table + [5, -1], dtype=torch.int32, device=dev)      # entries past n_lanes are not read
    ops.lane_gather(src, dst, lanes, len(table))
    for s, d in zip(src, dst):
        for l, v in enumerate(table):
            assert torch.equal(d[l], s[v]), (l, v)
        assert bool((d[len(table):] == -7.0).all())
    ops.lane_gather(src[:1], dst[:1], torch.tensor([1, 7], dtype=torch.int32, device=dev), 2)   # 7: no such video
    assert torch.equal(dst[0][0], src[0][1]) and torch.equal(dst[0][1], src[0][0])


def test_separate_labels_batched_equals_separate_labels():
    from aot_benchmark_b200 import ops
    g = torch.Generator(device=dev).manual_seed(4)
    H, W = 37, 53
    labels = [torch.randint(0, 81, (H, W), device=dev, generator=g).float() for _ in range(3)]
    labels[1][:3, :3] = torch.tensor([0., 10., 11.]).to(dev)          # the edges of a part
    entries = [(1, 3), (0, 7), (2, 0), (1, 0), (0, 1), (2, 7), (1, 1)] * 6      # more than one launch of 32
    out = [torch.full((H, W), -1.0, device=dev) for _ in entries]
    ops.separate_labels_batched([labels[v] for v, _ in entries], [p for _, p in entries], out)
    for (v, p), o in zip(entries, out):
        want = torch.empty(8, H, W, device=dev)
        ops.separate_labels(labels[v], want, 10)
        assert torch.equal(o, want[p]), (v, p)


def _aggregate_reference(lg, lanes, objs, size, align):
    """logits_postproc on each lane (at size) + soft_logit_aggregation (one engine: the aggregation of one map)."""
    from aot_benchmark_b200 import ops
    _, h, w, NC = lg.shape
    maps = []
    for l, obj in zip(lanes, objs):
        lo = torch.empty(1, NC, h, w, device=dev)
        up = None if size == (h, w) else torch.empty((1, NC) + size, device=dev)
        ops.logits_postproc(lg[l:l + 1], lo, up, obj, align)
        maps.append(lo if up is None else up)
    out = torch.empty((1, 1 + 10 * len(lanes)) + size, device=dev)
    ops.soft_logit_aggregation(maps, out, 10)
    return out


def _counts(obj):
    k = max(-(-obj // 10), 1)
    return [obj] if k == 1 else [10] * (k - 1) + [obj % 10 or 10]


@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("size", [None, (97, 131)])
@pytest.mark.parametrize("n_videos", [5, 37])
def test_soft_logit_aggregation_batched_equals_postproc_and_aggregation(align, size, n_videos):
    from aot_benchmark_b200 import ops
    g = torch.Generator(device=dev).manual_seed(n_videos)
    h, w = 25, 33
    size = size or (h, w)
    objs = [[7, 11, 14, 20, 21, 80, 30][b % 7] for b in range(n_videos)]   # 1, 2, 2, 2, 3, 8 and 3 lanes
    counts = [_counts(o) for o in objs]
    n_lanes = sum(len(c) for c in counts)
    perm = torch.randperm(n_lanes, generator=torch.Generator().manual_seed(n_videos)).tolist()   # lanes interleaved
    lanes, k = [], 0
    for c in counts:
        lanes.append(perm[k:k + len(c)])
        k += len(c)
    lg = torch.randn(n_lanes, h, w, 11, device=dev, generator=g) * 4
    tie = lanes[2]                                    # a 14-object video: part 1 a copy of part 0 ties channels 1-10 and 11-20
    lg[tie[1]] = lg[tie[0]]
    counts[2] = [10, 10]
    out = [torch.empty((1, 1 + 10 * len(r)) + size, device=dev) for r in lanes]
    labels = [torch.empty((1,) + size, device=dev) for _ in lanes]
    ops.soft_logit_aggregation_batched(lg, lanes, counts, align, out=out, labels=labels)
    only = [torch.empty((1,) + size, device=dev) for _ in lanes]
    ops.soft_logit_aggregation_batched(lg, lanes, counts, align, labels=only)
    for b in range(n_videos):
        want = _aggregate_reference(lg, lanes[b], counts[b], size, align)
        assert torch.equal(out[b], want), b
        first = want.argmax(1).float()
        assert torch.equal(labels[b], first) and torch.equal(only[b], first), b
    assert bool((labels[2] >= 11).any() == False)     # noqa: E712  (the tie goes to part 0's channel)


def _model(name, sd):
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    cfg = EngineConfig("t", name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd)
    return model.cuda().eval()


def _engine_cls(model):
    from aot_benchmark_b200.multi_video import DeAOTMultiVideoInferEngine, MultiVideoInferEngine
    return DeAOTMultiVideoInferEngine if model.cfg.MODEL_VOS == "deaot" else MultiVideoInferEngine


@pytest.mark.parametrize("case", ["aott_multi14_events", "deaott_multi14_events"])
def test_golden_video_next_to_other_videos_vs_reference(golden_dir, case):
    """The 14-object golden video (ids 9-14 first at frame 2: a second lane mid-video) in a multi-video engine next to a
    23-object video that closes after frame 3 and a 6-object video that opens at frame 2, fed the golden's forced masks: its
    live channels within 1e-3 of the reference on every frame (M = 8 is not reached)."""
    g = torch.load(os.path.join(golden_dir, f"events_{case}.pt"))
    sd = OW.build_state_dict(g["model"], seed=g["seed"])
    model = _model(g["model"], sd)
    frames, full = O.synthetic_video(g["frames"], g["H"], g["W"], 14, seed=g["video_seed"])
    first = torch.where(full <= g["first_objs"], full, torch.zeros_like(full))
    others = {6: O.synthetic_video(g["frames"], g["H"], g["W"], 6, seed=91),
              23: O.synthetic_video(g["frames"], g["H"], g["W"], 23, seed=92)}
    eng = _engine_cls(model)(model, max_videos=3, long_term_mem_max=8, long_term_mem_gap=g["gap"], max_lanes=6)
    out_size = tuple(g["out_size"])
    with torch.no_grad():
        big = eng.open_video(others[23][0][0].cuda(), others[23][1].cuda(), 23, long_term_mem_gap=1)
        vid = eng.open_video(frames[0].cuda(), first.cuda(), g["first_objs"])
        other, obj = None, g["first_objs"]
        for t in range(1, g["frames"]):
            if t == 2:                                 # a third video opens while the golden one gains its second lane
                other = eng.open_video(others[6][0][0].cuda(), others[6][1].cuda(), 6, long_term_mem_gap=2)
            feed = {vid: frames[t].cuda()}
            if big is not None:
                feed[big] = others[23][0][t].cuda()
            if other is not None:
                feed[other] = others[6][0][t - 1].cuda()
            eng.propagate(feed)
            logit = eng.decode_current_logits(out_size)[vid]
            label = g["ref_labels"][t - 1].float().cuda()
            if t == g["event_frame"]:
                obj = max(obj, int(g["new_label"].max()))
                fb = F.interpolate(label, size=(g["H"], g["W"]), mode="nearest")
                eng.add_reference_frame(vid, frames[t].cuda(), fb, obj)
                logit = eng.decode_current_logits(out_size)[vid]
            n = g["live_channels"][t - 1]
            d = (logit.cpu()[:, :n] - g["ref_logits"][t - 1]).abs().max().item()
            assert d < 1e-3, f"frame {t}: max |dlogit| vs reference = {d}"
            assert len(eng.video_lanes(vid)) == (2 if t >= g["event_frame"] else 1)
            own = {v: l.argmax(1, keepdim=True).float() for v, l in eng.decode_current_logits(None).items()}
            labels = {v: F.interpolate(own[v], size=(g["H"], g["W"]), mode="nearest") for v in own}
            labels[vid] = F.interpolate(label, size=(g["H"], g["W"]), mode="nearest")
            eng.update_memory(labels)
            if big is not None and t == 3:
                eng.close_video(big)
                big = None


def _run(model, precision, graphs, monkeypatch, Hh=129, Ww=193, M=3):
    """Videos of 4, 14 and 23 objects (the 4-object one gains objects 5-11 at frame 3, taking a second lane; the 14-object
    one closes between propagate and update at frame 5, after the one-lane video 3 closed and its lane was refilled), run
    for more than M memory frames through the multi-video engine and through one bounded one-video engine each ->
    (max |dlogit|, labels disagreeing where the reference's top two are apart, logits per step)."""
    from aot_benchmark_b200 import engine
    from aot_benchmark_b200.engine import AOTInferEngine, DeAOTInferEngine
    monkeypatch.setattr(engine, "USE_GRAPHS", graphs)
    ref_cls = DeAOTInferEngine if model.cfg.MODEL_VOS == "deaot" else AOTInferEngine
    tol = 2e-3 if precision == "fp32" else 5e-2
    eng = _engine_cls(model)(model, max_videos=4, long_term_mem_max=M, long_term_mem_gap=1, precision=precision,
                             max_lanes=8)
    lens, objs, t0 = [8, 6, 8, 3], [4, 14, 23, 2], [0, 0, 1, 0]
    clips = [O.synthetic_video(n, Hh, Ww, max(o, 11), seed=30 + i) for i, (n, o) in enumerate(zip(lens, objs))]
    vids, local, refs = {}, {}, {}
    dmax, bad, trace = 0.0, 0, []
    with torch.no_grad():
        for step in range(9):
            for i in range(4):
                if step == t0[i]:
                    f, full = clips[i]
                    m = torch.where(full <= objs[i], full, torch.zeros_like(full)).cuda()
                    vids[i] = eng.open_video(f[0].cuda(), m, objs[i])
                    refs[i] = ref_cls(model, long_term_mem_gap=1, long_term_mem_max=M, precision=precision)
                    refs[i].add_reference_frame(f[0].cuda(), m, obj_nums=[objs[i]], frame_step=0)
                    local[i] = 0
            for i in [i for i in vids if local[i] + 1 >= lens[i]]:
                eng.close_video(vids.pop(i))
            if not vids:
                break
            live = list(vids)
            for i in live:
                local[i] += 1
            eng.propagate({vids[i]: clips[i][0][local[i]].cuda() for i in live})
            if 1 in live and local[1] == 5:              # close between propagate and update
                eng.close_video(vids.pop(1))
                live.remove(1)
            got = eng.decode_current_logits((Hh, Ww))
            labs = eng.decode_labels((Hh, Ww))
            trace.append({i: got[vids[i]].clone() for i in live})
            labels = {}
            for i in live:
                refs[i].match_propogate_one_frame(clips[i][0][local[i]].cuda())
                want = refs[i].decode_current_logits((Hh, Ww))
                k = objs[i] + 1
                dmax = max(dmax, (got[vids[i]][:, :k] - want[:, :k]).abs().max().item())
                top2 = want.topk(2, dim=1).values
                clear = (top2[:, 0] - top2[:, 1]) > tol
                bad += int(((labs[vids[i]] != want.argmax(1)) & clear).sum())
                labels[i] = torch.argmax(want[:, :k], dim=1, keepdim=True).float()
            if 0 in live and local[0] == 3:
                objs[0] = 11
                m = torch.where(clips[0][1].cuda() > 4, clips[0][1].cuda(), labels[0])
                eng.add_reference_frame(vids[0], clips[0][0][3].cuda(), m, 11)
                refs[0].add_reference_frame(clips[0][0][3].cuda(), m, obj_nums=[11], frame_step=3)
                got0 = eng.decode_current_logits((Hh, Ww))[vids[0]]
                want0 = refs[0].decode_current_logits((Hh, Ww))
                dmax = max(dmax, (got0[:, :12] - want0[:, :12]).abs().max().item())
                assert len(eng.video_lanes(vids[0])) == 2
            eng.update_memory({vids[i]: labels[i] for i in live})
            for i in live:
                refs[i].update_memory(labels[i])
    torch.cuda.synchronize()
    return dmax, bad, trace


@pytest.mark.parametrize("name,precision,tol", [("r50_aotl", "fp32", 2e-3), ("r50_aotl", "fp16", 5e-2),
                                                ("r50_deaotl", "fp32", 2e-3)])
def test_engine_matches_one_engine_per_video(monkeypatch, name, precision, tol):
    model = _model(name, OW.build_state_dict(name, seed=0))
    dmax, bad, _ = _run(model, precision, True, monkeypatch)
    assert dmax < tol, dmax
    assert bad == 0, bad


def test_graphs_equal_eager(monkeypatch):
    model = _model("aott", OW.build_state_dict("aott", seed=1))
    _, _, eager = _run(model, "fp32", False, monkeypatch)
    _, _, graph = _run(model, "fp32", True, monkeypatch)
    assert len(eager) == len(graph)
    for a, b in zip(eager, graph):
        assert a.keys() == b.keys()
        for i in a:
            assert torch.equal(a[i], b[i]), i
