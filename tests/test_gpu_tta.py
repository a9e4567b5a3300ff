"""GPU: test-time augmentation -- the ensemble and feedback kernels (aotb_tta_merge_f32 / aotb_tta_feedback_f32) against a
float64 restatement, TTAInferEngine and the evaluator's own TTA loop over the drop-in engines against the real reference
(tests/golden/tta_*.pt), and the engine's invariances (streams, graphs, one augmentation, a second video, the bounded bank).

Error bound of the merge (stated as test_gpu_mask_logit_envelope.py states its bounds), eps = 2^-23, L = max |live logit|:
  * source coordinates and bilinear weights are fp32 (bl_src); the restatement uses them as float64 values, but the kernel may
    round src once more or less (fma contraction): a weight error of up to ulp(S), S = largest source coordinate, on a
    neighbour difference of up to 2L;
  * the fp32 bilinear sum of four weighted logits adds <= 4 eps L;
    so every upsampled logit is within delta = 4 eps L + 2 ulp(S) L of the float64 one;
  * softmax: |dp_c| <= p_c (|dv_c| + sum_j p_j |dv_j|) <= 2 delta p_c, plus (NC + 6) eps p_c for expf, the sum and the
    division; the mean over augmentations is a convex combination (+ eps).
  => |dp| <= 2 delta + (NC + 7) eps.  A label may differ only where the float64 top-2 margin is below twice that bound.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tta_support as S
from oracle import aot_oracle as O
from oracle import tta_oracle as TO

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -23


def _bl_src(out_sz, in_sz, align):
    """bl_src of csrc/idbank.cu in float32 arithmetic -> (i0, i1, l1) per output index."""
    d = np.arange(out_sz, dtype=np.float32)
    if align:
        scale = np.float32(in_sz - 1) / np.float32(out_sz - 1) if out_sz > 1 else np.float32(0)
        src = (scale * d).astype(np.float32)
    else:
        scale = np.float32(in_sz) / np.float32(out_sz)
        src = np.maximum((scale * (d + np.float32(0.5))).astype(np.float32) - np.float32(0.5), np.float32(0))
    i0 = np.minimum(src.astype(np.int64), in_sz - 1)
    i1 = i0 + (i0 < in_sz - 1)
    return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy((src - i0).astype(np.float64)), float(src.max())


def _up64(lo, H, W, align, flip):
    """[NC, h, w] -> [NC, H, W] in float64 with the kernel's coordinates; flip reads column W-1-x."""
    lo = lo.double().cpu()
    NC, h, w = lo.shape
    y0, y1, ly, sy = _bl_src(H, h, align)
    x0, x1, lx, sx = _bl_src(W, w, align)
    if flip:
        x0, x1, lx = x0.flip(0), x1.flip(0), lx.flip(0)
    ly, lx = ly.view(1, H, 1), lx.view(1, 1, W)
    g = lambda yy, xx: lo[:, yy][:, :, xx]
    up = (1 - ly) * ((1 - lx) * g(y0, x0) + lx * g(y0, x1)) + ly * ((1 - lx) * g(y1, x0) + lx * g(y1, x1))
    return up, max(sy, sx)


def _ulp(x):
    return 2.0 ** (math.floor(math.log2(max(x, 1.0))) - 23)


def _merge64(maps, flips, H, W, align):
    probs, smax = [], 0.0
    for m, f in zip(maps, flips):
        up, s = _up64(m, H, W, align, f)
        smax = max(smax, s)
        probs.append(torch.softmax(up, dim=0))
    return torch.stack(probs).mean(0), smax


def _bound(L, smax, NC):
    delta = 4 * EPS * L + 2 * _ulp(smax) * L
    return 2 * delta + (NC + 7) * EPS


# (E, NC, low-res sizes or None for maps at the output size, output size, align, flips)
MERGE_GRID = [
    (1, 11, [(13, 17)], (49, 65), True, [False]),
    (2, 11, [(13, 17), (17, 21)], (97, 129), True, [False, True]),
    (4, 21, [(25, 33), (25, 33), (33, 41), (33, 41)], (97, 129), True, [False, True, False, True]),
    (6, 11, [(29, 45), (29, 45), (41, 61), (41, 61), (49, 77), (49, 77)], (161, 241), True, [False, True] * 3),
    (8, 41, [(7, 9), (7, 9), (11, 13), (11, 13), (9, 17), (9, 17), (5, 5), (5, 5)], (31, 47), False, [False, True] * 4),
    (4, 11, [(36, 52), (36, 52), (48, 68), (48, 68)], (144, 208), False, [False, True, False, True]),
    (2, 21, None, (53, 71), True, [False, True]),                          # aggregated maps at the output size: identity
    (3, 41, None, (37, 45), False, [True, False, True]),
    (4, 11, [(121, 214), (121, 214), (157, 277), (157, 277)], (480, 854), True, [False, True, False, True]),
]


def _maps(E, NC, sizes, H, W, live, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for e in range(E):
        h, w = (H, W) if sizes is None else sizes[e]
        m = (torch.rand(NC, h, w, generator=g) * 2 - 1) * 50
        m[live:] = -1e10                                                     # ids above the object count (aot_engine.py:371-374)
        out.append(m.cuda().contiguous())
    return out


@pytest.mark.parametrize("E,NC,sizes,out,align,flips", MERGE_GRID)
def test_merge_kernel_vs_float64(E, NC, sizes, out, align, flips):
    from aot_benchmark_b200 import ops
    H, W = out
    live = NC - 3
    maps = _maps(E, NC, sizes, H, W, live, seed=E * 100 + NC)
    label = torch.empty(1, 1, H, W, device="cuda")
    prob = torch.empty(1, NC, H, W, device="cuda")
    ops.tta_merge(maps, flips, label, align, prob=prob)
    p64, smax = _merge64(maps, flips, H, W, align)
    bound = _bound(50.0, smax if sizes is not None else 0.0, NC)
    err = (prob[0].cpu().double() - p64).abs().max().item()
    assert err <= bound, (err, bound)
    top2 = p64.topk(2, dim=0).values
    band = (top2[0] - top2[1]) < 2 * bound
    ref = p64.argmax(0).float()
    bad = (label[0, 0].cpu() != ref) & ~band
    assert int(bad.sum()) == 0
    if sizes is None:                                              # at the output size bl_src is the identity, exactly
        assert err <= (NC + 7) * EPS
    # without prob, the same labels; with a new-object label, its ids where nonzero
    new = torch.zeros(H, W, device="cuda")
    new[H // 3:H // 2, W // 4:W // 2] = NC + 2
    lab2 = torch.empty(1, 1, H, W, device="cuda")
    ops.tta_merge(maps, flips, lab2, align, new_label=new)
    assert torch.equal(lab2[0, 0], torch.where(new != 0, new, label[0, 0]))


@pytest.mark.parametrize("align", [True, False])
def test_merge_kernel_exact_ties_take_the_first_index(align):
    from aot_benchmark_b200 import ops
    H, W, NC = 41, 57, 11
    maps = _maps(4, NC, [(11, 15), (11, 15), (15, 19), (15, 19)], H, W, NC, seed=3)
    for m in maps:
        m[2] = 50.0
        m[5] = 50.0                                               # ids 2 and 5 tie exactly everywhere, in every map
    label = torch.empty(1, 1, H, W, device="cuda")
    ops.tta_merge(maps, [False, True, False, True], label, align)
    assert bool((label == 2).all())


def _feedback_ref(lo, size, in_size, align, flip, new):
    """F.interpolate(nearest) of the mirrored overlay of the softmax argmax (evaluator.py:346-422), in float64 -> (label, margin)."""
    H, W = size
    if lo is None:
        lab = torch.zeros(1, 1, H, W, dtype=torch.float64)
        margin = torch.full((1, 1, H, W), float("inf"), dtype=torch.float64)
        smax = 0.0
    else:
        up, smax = _up64(lo, H, W, align, False)
        p = torch.softmax(up, dim=0)
        lab = p.argmax(0).double().view(1, 1, H, W)
        top2 = p.topk(2, dim=0).values
        margin = (top2[0] - top2[1]).view(1, 1, H, W)
        if flip:                                                   # original orientation, as the evaluator holds it
            lab, margin = lab.flip(3), margin.flip(3)
    if new is not None:
        n = new.double().cpu().view(1, 1, H, W)
        lab = torch.where(n != 0, n, lab)
        margin = torch.where(n != 0, torch.full_like(margin, float("inf")), margin)
    if flip:
        lab, margin = lab.flip(3), margin.flip(3)
    near = lambda t: F.interpolate(t, size=in_size, mode="nearest")[0, 0]
    return near(lab), near(margin), smax


@pytest.mark.parametrize("form", ["first_frame", "steady", "new_objects"])
@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("align,lowres,size,in_size", [(True, (25, 33), (97, 129), (129, 161)),
                                                       (True, (29, 45), (161, 241), (113, 177)),
                                                       (False, (48, 68), (144, 208), (192, 272)),
                                                       (True, None, (61, 83), (81, 97))])
def test_feedback_kernel_vs_interpolate(form, flip, align, lowres, size, in_size):
    from aot_benchmark_b200 import ops
    H, W = size
    NC = 21 if lowres is None else 11
    lo = None if form == "first_frame" else _maps(1, NC, None if lowres is None else [lowres], H, W, NC - 2, seed=11)[0]
    new = None
    if form != "steady":
        g = torch.Generator().manual_seed(5)
        new = torch.zeros(H, W)
        new[H // 5:H // 2, W // 7:W // 3] = 12
        new[H // 2:H - 3, W // 2:W - 2] = (torch.rand(H - 3 - H // 2, W - 2 - W // 2, generator=g) * 3).floor() * 13
        new = new.cuda()
    out = torch.empty(1, 1, *in_size, device="cuda")
    ops.tta_feedback(lo, out, size, align, flip, new_label=new)
    ref, margin, smax = _feedback_ref(lo, size, in_size, align, flip, new)
    ok = margin > 2 * _bound(50.0, smax, NC)
    assert torch.equal(out[0, 0].cpu().double()[ok], ref[ok])
    if lo is None:
        assert bool(ok.all())


# ---------------------------------------------------------------------------------------------------------------- engines
def _tta(g, sd, **kw):
    from aot_benchmark_b200 import TTAInferEngine
    return TTAInferEngine(S.model(g["model"], sd, "cuda"), long_term_mem_gap=g["gap"], flip=True, multi_scale=g["scales"], **kw)


def _run_tta(eng, g, imgs, first, new, forced=True):
    H, W = g["H"], g["W"]
    labels, probs, own = [], [], []
    ac = O.OracleConfig(g["model"]).MODEL_ALIGN_CORNERS
    with torch.no_grad():
        eng.restart_engine()
        eng.add_reference_frame(imgs[0], first.cuda(), obj_nums=g["first_objs"], frame_step=0)
        for t in range(1, len(imgs)):
            nl = new.get(t)
            fl = [g["aug"][t - 1, e].cuda() for e in range(len(g["flips"]))] if forced else None
            lab = eng.propagate(imgs[t], (H, W), new_label=None if nl is None else nl.cuda(), keep_prob=True, forced_labels=fl)
            labels.append(lab.clone())
            probs.append(eng.pred_prob.clone())
            own.append([S.own_label(m, (H, W), f, ac, new=nl) for m, f in zip(eng.aug_logits, eng.flips)])
    torch.cuda.synchronize()
    return labels, probs, own


@pytest.mark.parametrize("name", S.CASES)
def test_tta_engine_vs_reference_golden(golden_dir, name):
    g, sd, frames, first, new = S.load(golden_dir, name)
    imgs = S.aug_images(g, frames, "cuda")
    eng = _tta(g, sd)
    labels, probs, own = _run_tta(eng, g, imgs, first, new)
    for t, p in g["prob"].items():
        n = p.shape[0]
        assert (probs[t - 1][0, :n].cpu() - p).abs().max().item() < S.PROB_TOL
    bad = sum(S.outside_band(l, g["ens"][t], p, new=new.get(t + 1)) for t, (l, p) in enumerate(zip(labels, probs)))
    bad_aug = sum(S.outside_band(lab, g["aug"][t, e], p, new=new.get(t + 1))
                  for t, per in enumerate(own) for e, (lab, p) in enumerate(per))
    assert bad == 0 and bad_aug == 0, (bad, bad_aug)
    assert [len(e.aot_engines) for e in eng.aug_engines] == g["sub_engines"]
    if name == "deaott_multi14":
        assert all(len(e.aot_engines) == 2 for e in eng.aug_engines)


@pytest.mark.parametrize("name", S.CASES)
def test_evaluator_tta_loop_over_drop_in_engines(golden_dir, name):
    """The unedited evaluator's TTA loop (restated by run_video_tta) over AOTInferEngines from build_engine."""
    from aot_benchmark_b200 import EngineConfig, build_engine
    g, sd, frames, first, new = S.load(golden_dir, name)
    imgs = S.aug_images(g, frames, "cuda")
    m = S.model(g["model"], sd, "cuda")
    cfg = EngineConfig("t", g["model"])
    engines = [build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=m, gpu_id=0, long_term_mem_gap=g["gap"]).eval()
               for _ in g["flips"]]
    T = g["frames"]
    forced = [[g["aug"][t, e].reshape(1, 1, g["H"], g["W"]).cuda() for e in range(len(g["flips"]))] for t in range(T - 1)]
    with torch.no_grad():
        ens, _, probs = TO.run_video_tta(engines, imgs, g["flips"], first.cuda(), g["first_objs"], (g["H"], g["W"]),
                                         new_objects={t: v.cuda() for t, v in new.items()}, forced_labels=forced,
                                         prob_frames=range(1, T))
    for t, p in g["prob"].items():
        assert (probs[t][0, :p.shape[0]].cpu() - p).abs().max().item() < S.PROB_TOL
    bad = sum(S.outside_band(l, g["ens"][t - 1], probs[t], new=new.get(t)) for t, l in enumerate(ens, start=1))
    assert bad == 0


def test_tta_engine_invariances(golden_dir, monkeypatch):
    from aot_benchmark_b200 import engine as E
    g, sd, frames, first, new = S.load(golden_dir, "deaott_multi14")        # nested forks: 2 sub-engines per augmentation
    imgs = S.aug_images(g, frames, "cuda")
    eng = _tta(g, sd)
    base_l, base_p, _ = _run_tta(eng, g, imgs, first, new, forced=False)
    for streams, graphs in ((False, True), (True, False)):
        monkeypatch.setattr(E, "SUB_ENGINE_STREAMS", streams)
        monkeypatch.setattr(E, "USE_GRAPHS", graphs)
        l, p, _ = _run_tta(_tta(g, sd), g, imgs, first, new, forced=False)
        assert all(torch.equal(a, b) for a, b in zip(l, base_l)), (streams, graphs)
        assert all(torch.equal(a, b) for a, b in zip(p, base_p)), (streams, graphs)
    monkeypatch.undo()
    # the same engine again after restart_engine(): identical clip, identical results (graphs replayed)
    l, p, _ = _run_tta(eng, g, imgs, first, new, forced=False)
    assert all(torch.equal(a, b) for a, b in zip(l, base_l))


def test_tta_engine_second_geometry_and_bounded_bank(golden_dir):
    g, sd, frames, first, new = S.load(golden_dir, "aott_flip_ms")
    imgs = S.aug_images(g, frames, "cuda")
    eng = _tta(g, sd, long_term_mem_max=2)
    l1, p1, _ = _run_tta(eng, g, imgs, first, new, forced=False)
    for e in eng.aug_engines:
        for sub in e.aot_engines:
            assert sub.long_term_mem_max == 2 and sub.bank_cap == 2 * sub.enc_hw and sub.bank_len == 2 * sub.enc_hw
    # another geometry (the clip cropped), then the first clip again: same results as a fresh engine
    crop = [[i[..., :81, :113] if i.shape[-2] == g["H"] else i[..., :113, :145] for i in per] for per in imgs]
    g2 = dict(g, H=81, W=113)
    _run_tta(eng, g2, crop, first[..., :81, :113], {}, forced=False)
    l2, p2, _ = _run_tta(eng, g, imgs, first, new, forced=False)
    assert all(torch.equal(a, b) for a, b in zip(l1, l2)) and all(torch.equal(a, b) for a, b in zip(p1, p2))


def test_one_augmentation_matches_the_single_engine_fused_path(golden_dir):
    from aot_benchmark_b200 import EngineConfig, TTAInferEngine, build_engine
    g, sd, frames, first, new = S.load(golden_dir, "aott_flip_ms")
    H, W = g["H"], g["W"]
    imgs = [per[0] for per in S.aug_images(g, frames, "cuda")]
    m = S.model(g["model"], sd, "cuda")
    tta = TTAInferEngine(m, long_term_mem_gap=g["gap"], flip=False, multi_scale=[1.0])
    cfg = EngineConfig("t", g["model"])
    one = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=m, gpu_id=0, long_term_mem_gap=g["gap"]).eval()
    with torch.no_grad():
        tta.add_reference_frame([imgs[0]], first.cuda(), obj_nums=g["first_objs"])
        one.add_reference_frame(imgs[0], first.cuda(), obj_nums=[g["first_objs"]], frame_step=0)
        for t in range(1, len(imgs)):
            lab = tta.propagate([imgs[t]], (H, W), keep_prob=True)
            one.match_propogate_one_frame(imgs[t])
            one.decode_current_logits(None)
            ref = one.aot_engines[0].predict_current_mask((H, W)).float()     # fused upsample + argmax
            top2 = tta.pred_prob.topk(2, dim=1).values
            band = (top2[:, 0] - top2[:, 1]) < 1e-5
            assert int(((lab[0].cpu() != ref.cpu()) & ~band.cpu()).sum()) == 0, t
            one.update_memory(F.interpolate(ref.view(1, 1, H, W), size=one.input_size_2d, mode="nearest"))
            assert torch.equal(tta._feedback_buf(0, (H, W)), F.interpolate(lab, size=(H, W), mode="nearest"))
