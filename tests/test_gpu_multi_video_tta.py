"""GPU: the batched TTA entry points (aotb_tta_merge_batched_f32 / aotb_tta_feedback_batched_f32) against logits_postproc +
the one-video TTA kernels on every video / lane, bitwise (labels, probabilities, feedback maps, near-ties included), and
MultiVideoTTAInferEngine against the reference's TTA goldens, against one bounded TTAInferEngine per video, and across
streams, graphs and a second pass."""
import random

import pytest
import torch

import tta_support as S
from oracle import aot_oracle as O

pytestmark = pytest.mark.gpu


def _pools(sizes, lanes, NC, seed, tie=False):
    """One NHWC decoder output [lanes, h, w, NC] per distinct low-res size, logits spread over +-8.  tie: channels 1 and 2
    lead every tap by about 20 and are one ulp apart there, so the labels turn on the last bit of each bilinear blend."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = {}
    for s in dict.fromkeys(sizes):
        t = torch.randn((lanes,) + s + (NC,), generator=g) * 8
        if tie:
            t[..., 1] = t[..., 1] * 0.25 + 28
            t[..., 2] = torch.nextafter(t[..., 1], torch.tensor(float("inf")))
        out[s] = t.cuda()
    return out


def _postproc(lg, lane, obj):
    from aot_benchmark_b200 import ops
    h, w, NC = lg.shape[1:]
    lo = torch.empty((1, NC, h, w), device="cuda")
    ops.logits_postproc(lg[lane:lane + 1], lo, None, obj, True)
    return lo


# (E, low-res sizes per augmentation, output size): E = 6 has a downscaled augmentation (0.75), E = 8 four scales
MERGE_CASES = [(1, [(13, 17)], (49, 65)), (2, [(13, 17)] * 2, (49, 65)),
               (4, [(13, 17)] * 2 + [(17, 22)] * 2, (49, 65)),
               (6, [(10, 13)] * 2 + [(13, 17)] * 2 + [(17, 22)] * 2, (49, 65)),
               (8, [(10, 13)] * 2 + [(13, 17)] * 2 + [(17, 22)] * 2 + [(20, 26)] * 2, (50, 66))]


@pytest.mark.parametrize("n", [1, 2, 3, 5, 33])
@pytest.mark.parametrize("E,sizes,out", MERGE_CASES)
@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("tie", [False, True])
def test_merge_batched_equals_postproc_and_one_video_merges(n, E, sizes, out, align, tie):
    """n = 33 takes two launches (32 videos per launch)."""
    from aot_benchmark_b200 import ops
    NC, H, W = 11, out[0], out[1]
    rnd = random.Random(n * 100 + E)
    flips = [bool(e % 2) for e in range(E)]
    L = 2 * n + 1                                            # lanes per map; videos take scattered lanes
    pools = _pools(sizes, L, NC, seed=E * 7 + n, tie=tie)
    maps = [pools[s] for s in sizes]
    lanes = [[rnd.randrange(L) for _ in range(E)] for _ in range(n)]
    objs = [rnd.randint(2 if tie else 1, 10) for _ in range(n)]
    for with_new, with_prob in ((False, False), (True, True), (False, True)):
        news = [None] * n
        if with_new:
            for b in range(0, n, 2):
                t = torch.zeros(H, W, device="cuda")
                t[3:9, 4:20] = objs[b] + 1
                news[b] = t
        label = torch.full((n, 1, H, W), -7.0, device="cuda")
        prob = torch.full((n, NC, H, W), -7.0, device="cuda") if with_prob else None
        ops.tta_merge_batched(maps, flips, lanes, objs, label, align, new_labels=news, prob=prob)
        for b in range(n):
            lo = [_postproc(maps[e], lanes[b][e], objs[b]) for e in range(E)]
            want_l = torch.empty((1, 1, H, W), device="cuda")
            want_p = torch.empty((1, NC, H, W), device="cuda")
            ops.tta_merge(lo, flips, want_l, align, new_label=news[b], prob=want_p if with_prob else None)
            assert torch.equal(label[b:b + 1], want_l), (b, with_new)
            if with_prob:
                assert torch.equal(prob[b:b + 1], want_p), b


@pytest.mark.parametrize("n_lanes", [1, 2, 3, 5, 40])
@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("form", ["logits", "logits_new", "no_logits", "tie"])
def test_feedback_batched_equals_postproc_and_one_lane_feedbacks(n_lanes, align, form):
    from aot_benchmark_b200 import ops
    NC, (h, w), (H, W), (Hi, Wi) = 11, (17, 22), (65, 85), (68, 88)
    rnd = random.Random(n_lanes)
    lg = _pools([(h, w)], n_lanes, NC, seed=n_lanes, tie=form == "tie")[(h, w)]
    objs = [rnd.randint(2 if form == "tie" else 1, 10) for _ in range(n_lanes)]
    flips = [bool(rnd.randint(0, 1)) for _ in range(n_lanes)]
    news = [None] * n_lanes
    if form in ("logits_new", "no_logits"):
        for k in range(n_lanes):
            if form == "no_logits" or k % 2:
                t = torch.zeros(H, W, device="cuda")
                t[5:30, 2:40] = rnd.randint(1, 10)
                news[k] = t
    out = torch.full((n_lanes + 1, Hi, Wi), -7.0, device="cuda")
    src = None if form == "no_logits" else lg
    ops.tta_feedback_batched(src, out, None if src is None else objs, flips, (H, W), align, new_labels=news)
    assert bool((out[n_lanes] == -7.0).all())                  # nothing past the last lane
    for k in range(n_lanes):
        want = torch.empty((1, 1, Hi, Wi), device="cuda")
        ops.tta_feedback(None if src is None else _postproc(lg, k, objs[k]), want, (H, W), align, flips[k],
                         new_label=news[k])
        assert torch.equal(out[k], want[0, 0]), k


# ----------------------------------------------------------------------------------------------------- the engine
def _engine(g, sd, M, **kw):
    from aot_benchmark_b200 import MultiVideoTTAInferEngine
    return MultiVideoTTAInferEngine(S.model(g["model"], sd, "cuda"), max_videos=3, long_term_mem_max=M,
                                    long_term_mem_gap=g["gap"], flip=True, multi_scale=g["scales"], **kw)


def _run_copies(eng, g, imgs, first, new, forced=True):
    """Three copies of the clip opened at steps 0, 1 and 2, the middle one closed two frames early -> {copy: [(label, prob,
    per-augmentation own labels)] per frame}."""
    T, H, W = len(imgs), g["H"], g["W"]
    ac = O.OracleConfig(g["model"]).MODEL_ALIGN_CORNERS
    starts, ends = {0: 0, 1: 1, 2: 2}, {0: T, 1: T - 2, 2: T}
    vids, local, res = {}, {}, {c: [] for c in starts}
    with torch.no_grad():
        for step in range(T + 2):
            for c in [c for c in vids if local[c] + 1 >= ends[c]]:
                eng.close_video(vids.pop(c))
            for c, t0 in starts.items():
                if step == t0:
                    vids[c] = eng.open_video(imgs[0], first.cuda(), g["first_objs"])
                    local[c] = 0
            if not vids:
                break
            for c in vids:
                local[c] += 1
            nl = {vids[c]: new[local[c]].cuda() for c in vids if local[c] in new}
            fl = {vids[c]: [g["aug"][local[c] - 1, e].cuda() for e in range(len(g["flips"]))] for c in vids} \
                if forced else None
            objs = {vid: eng._video(vid)["obj"] for vid in vids.values()}
            out = eng.propagate({vids[c]: imgs[local[c]] for c in vids}, (H, W), new_labels=nl, keep_prob=True,
                                forced_labels=fl)
            for c, vid in vids.items():
                own = []
                if forced:
                    for e, f in enumerate(g["flips"]):
                        lo = eng.aug_logits[vid][e][0].permute(2, 0, 1).clone()
                        lo[objs[vid] + 1:] = -1e10
                        own.append(S.own_label(lo, (H, W), f, ac, new=None if vid not in nl else nl[vid].cpu()))
                res[c].append((out[vid].clone(), eng.pred_prob[vid].clone(), own))
    torch.cuda.synchronize()
    return res


GOLDEN_CASES = ["aott_flip_ms", "r50_aotl_flip_ms3", "swinb_aotl_flip_ms"]


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_engine_vs_reference_golden(golden_dir, name):
    g, sd, frames, first, new = S.load(golden_dir, name)
    imgs = S.aug_images(g, frames, "cuda")
    res = _run_copies(_engine(g, sd, M=len(imgs)), g, imgs, first, new)
    assert [len(r) for r in res.values()] == [len(imgs) - 1, max(len(imgs) - 3, 1), len(imgs) - 1]
    bad = bad_aug = 0
    for c, frames_c in res.items():
        for i, (lab, prob, own) in enumerate(frames_c):
            t = i + 1
            if t in g["prob"]:
                p = g["prob"][t]
                assert (prob[0, :p.shape[0]].cpu() - p).abs().max().item() < S.PROB_TOL
            bad += S.outside_band(lab, g["ens"][t - 1], prob, new=new.get(t))
            bad_aug += sum(S.outside_band(ol, g["aug"][t - 1, e], p, new=new.get(t)) for e, (ol, p) in enumerate(own))
    assert bad == 0 and bad_aug == 0, (bad, bad_aug)


SH, SW, M = 129, 193, 3
SCALES = [1.0, 1.3]
SCHEDULE = {0: (0, 8, 5, 2, 4), 1: (1, 5, 3, 1, None), 2: (2, 7, 2, 3, None)}


def _aug_clip(seed, n, objs):
    from aot_benchmark_b200.io_side import FramePreprocessor
    from oracle.tta_oracle import synthetic_frames_u8
    prep = FramePreprocessor(None, 1040, True, SCALES, True)
    frames = [prep(f) for f in synthetic_frames_u8(n, SH, SW, seed=seed)]
    _, mask = O.synthetic_video(1, SH, SW, objs, seed=seed)
    return [[i.cuda() for i in f] for f in frames], mask.cuda()


def _drive(eng, refs_make=None):
    """SCHEDULE through eng and, with refs_make, one TTAInferEngine per video -> (labels, probs, worst low-res logit
    difference, label pixels outside the tie band)."""
    clips = {v: _aug_clip(40 + v, n, o) for v, (_, n, o, _, _) in SCHEDULE.items()}
    vids, local, objs, refs, trace = {}, {}, {}, {}, []
    worst, bad = 0.0, 0
    with torch.no_grad():
        for step in range(20):
            for v in [v for v in vids if local[v] + 1 >= SCHEDULE[v][1]]:
                eng.close_video(vids.pop(v))
            for v, (t0, n, o, gap, _) in SCHEDULE.items():
                if step == t0:
                    imgs, mask = clips[v]
                    vids[v] = eng.open_video(imgs[0], mask, o, long_term_mem_gap=gap)
                    if refs_make:
                        refs[v] = refs_make(gap)
                        refs[v].add_reference_frame(imgs[0], mask, obj_nums=[o], frame_step=0)
                    local[v], objs[v] = 0, o
            if not vids:
                break
            nl = {}
            for v in vids:
                local[v] += 1
                if SCHEDULE[v][4] == local[v]:
                    objs[v] += 1
                    m = torch.zeros(1, 1, SH, SW, device="cuda")
                    m[..., 10:30, 20:60] = objs[v]
                    nl[v] = m
            pre = {v: objs[v] - (v in nl) for v in vids}
            out = eng.propagate({vids[v]: clips[v][0][local[v]] for v in vids}, (SH, SW),
                                new_labels={vids[v]: m for v, m in nl.items()}, keep_prob=True)
            trace.append({v: (out[vids[v]].clone(), eng.pred_prob[vids[v]].clone()) for v in vids})
            for v in vids if refs_make else ():
                want = refs[v].propagate(clips[v][0][local[v]], (SH, SW), new_label=nl.get(v), keep_prob=True)
                k = pre[v] + 1
                for e in range(len(eng.flips)):
                    got = eng.aug_logits[vids[v]][e][0].permute(2, 0, 1)[:k]
                    worst = max(worst, (got - refs[v].aug_logits[e][0, :k]).abs().max().item())
                bad += S.outside_band(out[vids[v]], want.cpu().reshape(SH, SW), refs[v].pred_prob,
                                      new=None if v not in nl else nl[v].cpu())
    torch.cuda.synchronize()
    return trace, worst, bad


def _model(name, precision=None):
    from oracle import weights as OW
    return S.model(name, OW.build_state_dict(name, seed=3, flavour="calibrated"), "cuda")


@pytest.mark.parametrize("name", ["r50_aotl", "r50_deaotl"])
@pytest.mark.parametrize("precision,tol", [("fp32", 2e-3), ("fp16", 5e-2)])
def test_engine_matches_one_bounded_tta_engine_per_video(name, precision, tol):
    from aot_benchmark_b200 import MultiVideoTTAInferEngine, TTAInferEngine
    model = _model(name)
    eng = MultiVideoTTAInferEngine(model, max_videos=3, long_term_mem_max=M, long_term_mem_gap=2, flip=True,
                                   multi_scale=SCALES, precision=precision)
    _, worst, bad = _drive(eng, lambda gap: TTAInferEngine(model, long_term_mem_gap=gap, long_term_mem_max=M, flip=True,
                                                           multi_scale=SCALES, precision=precision))
    print(f"{name} {precision}: max |dlogit| = {worst:.3e}, label pixels outside the band = {bad}")
    assert worst < tol
    assert bad == 0


def test_engine_invariances(monkeypatch):
    from aot_benchmark_b200 import MultiVideoTTAInferEngine
    from aot_benchmark_b200 import engine as E
    model = _model("r50_aotl")
    mk = lambda: MultiVideoTTAInferEngine(model, max_videos=3, long_term_mem_max=M, long_term_mem_gap=2, flip=True,
                                          multi_scale=SCALES)
    eng = mk()
    base, _, _ = _drive(eng)
    for streams, graphs in ((False, True), (True, False)):
        monkeypatch.setattr(E, "SUB_ENGINE_STREAMS", streams)
        monkeypatch.setattr(E, "USE_GRAPHS", graphs)
        other, _, _ = _drive(mk())
        for a, b in zip(base, other):
            assert a.keys() == b.keys()
            assert all(torch.equal(a[v][0], b[v][0]) and torch.equal(a[v][1], b[v][1]) for v in a), (streams, graphs)
    monkeypatch.undo()
    again, _, _ = _drive(eng)                              # the same videos again on the same engine
    for a, b in zip(base, again):
        assert all(torch.equal(a[v][0], b[v][0]) and torch.equal(a[v][1], b[v][1]) for v in a)
