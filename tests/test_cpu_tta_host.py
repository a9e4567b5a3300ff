"""CPU: host side of the test-time augmentation engine (aot_benchmark_b200/tta.py) -- the per-augmentation engines, the
order of the merge / feedback / memory-update calls, the flip and resize of every label, new objects under flip -- against
the real reference's TTA loop (tests/golden/tta_*.pt), with every C-ABI entry point replaced by a torch-CPU emulation.  The
two TTA entry points are emulated here as the evaluator's own tensor expressions (evaluator.py:332-422); the kernels are
checked against them on the GPU (tests/test_gpu_tta.py)."""
import pytest
import torch
import torch.nn.functional as F

import tta_support as S
from oracle import aot_oracle as O
from oracle import tta_oracle as TO


def _up(logits, size, align):
    return F.interpolate(logits.reshape(1, *logits.shape[-3:]), size=size, mode="bilinear", align_corners=bool(align))


def emu_tta_merge(logits, flips, label, align_corners, new_label=None, prob=None, stream=None):
    """evaluator.py:332-369."""
    H, W = label.shape[-2:]
    probs = [torch.softmax(torch.flip(_up(l, (H, W), align_corners), dims=[3]) if f else _up(l, (H, W), align_corners), dim=1)
             for l, f in zip(logits, flips)]
    p = torch.mean(torch.cat(probs, dim=0), dim=0, keepdim=True)
    lab = torch.argmax(p, dim=1, keepdim=True).float()
    if new_label is not None:
        new = new_label.reshape(1, 1, H, W)
        keep = (new == 0).float()
        lab = lab * keep + new * (1 - keep)
    label.copy_(lab.reshape(label.shape))
    if prob is not None:
        prob.copy_(p.reshape(prob.shape))
    return label


def emu_tta_feedback(logits, out, output_size, align_corners, flip, new_label=None, stream=None):
    """evaluator.py:315-319 (no logits), :346-353 + :400-422, and :363-399 (new label)."""
    H, W = int(output_size[0]), int(output_size[1])
    if logits is None:
        lab = torch.zeros(1, 1, H, W)
    else:
        up = _up(logits, (H, W), align_corners)
        lab = torch.argmax(torch.softmax(torch.flip(up, dims=[3]) if flip else up, dim=1), dim=1, keepdim=True).float()
    if new_label is not None:
        new = new_label.reshape(1, 1, H, W)
        keep = (new == 0).float()
        lab = lab * keep + new * (1 - keep)
    if flip:
        lab = torch.flip(lab, dims=[3])
    out.copy_(F.interpolate(lab, size=tuple(out.shape[-2:]), mode="nearest").reshape(out.shape))
    return out


def _install(monkeypatch):
    import emu_ops
    from aot_benchmark_b200 import ops
    emu_ops.install_engine(monkeypatch)
    monkeypatch.setattr(ops, "tta_merge", emu_tta_merge)
    monkeypatch.setattr(ops, "tta_feedback", emu_tta_feedback)


def _frames(g):
    return 3 if g["model"].startswith("swinb") else g["frames"]       # Swin-B on CPU: keep the test short


@pytest.mark.parametrize("name", S.CASES)
def test_tta_engine_orchestration_vs_reference_golden(monkeypatch, golden_dir, name):
    from aot_benchmark_b200 import TTAInferEngine
    _install(monkeypatch)
    g, sd, frames, first, new = S.load(golden_dir, name)
    T, H, W, flips = _frames(g), g["H"], g["W"], g["flips"]
    imgs = S.aug_images(g, frames[:T])
    ac = O.OracleConfig(g["model"]).MODEL_ALIGN_CORNERS
    eng = TTAInferEngine(S.model(g["model"], sd), long_term_mem_gap=g["gap"], flip=True, multi_scale=g["scales"])
    assert [tuple(i.shape[2:]) for i in imgs[0]] == [tuple(s) for s in g["aug_sizes"]]
    bad_ens = bad_aug = 0
    with torch.no_grad():
        eng.restart_engine()
        eng.add_reference_frame(imgs[0], first, obj_nums=g["first_objs"], frame_step=0)
        for t in range(1, T):
            nl = new.get(t)
            forced = [g["aug"][t - 1, e] for e in range(len(flips))]
            label = eng.propagate(imgs[t], (H, W), new_label=nl, keep_prob=True, forced_labels=forced)
            bad_ens += S.outside_band(label, g["ens"][t - 1], eng.pred_prob, new=nl)
            if t in g["prob"]:
                ref = g["prob"][t]
                assert (eng.pred_prob[0, :ref.shape[0]] - ref).abs().max().item() < S.PROB_TOL
                assert float(eng.pred_prob[0, ref.shape[0]:].abs().sum()) < 1e-6      # masked ids: probability 0
            for e, f in enumerate(flips):
                own, p = S.own_label(eng.aug_logits[e], (H, W), f, ac, new=nl)
                bad_aug += S.outside_band(own, g["aug"][t - 1, e], p, new=nl)
                # the engine stores the forced label, mirrored for a flipped augmentation, nearest-resized to its input
                fb = g["aug"][t - 1, e].reshape(1, 1, H, W)
                fb = F.interpolate(torch.flip(fb, dims=[3]) if f else fb, size=eng.aug_engines[e].input_size_2d, mode="nearest")
                assert torch.equal(eng._feedback_buf(e, eng.aug_engines[e].input_size_2d), fb)
    assert bad_ens == 0 and bad_aug == 0, (bad_ens, bad_aug)
    assert [len(e.aot_engines) for e in eng.aug_engines] == g["sub_engines"]


@pytest.mark.parametrize("name", S.CASES)
def test_run_video_tta_over_oracle_engines_vs_reference_golden(golden_dir, name):
    g, sd, frames, first, new = S.load(golden_dir, name)
    T = _frames(g)
    imgs = S.aug_images(g, frames[:T])
    engines = [O.OracleInferEngine(sd, O.OracleConfig(g["model"]), long_term_mem_gap=g["gap"]) for _ in g["flips"]]
    forced = [[g["aug"][t, e].reshape(1, 1, g["H"], g["W"]) for e in range(len(g["flips"]))] for t in range(T - 1)]
    with torch.no_grad():
        ens, _, probs = TO.run_video_tta(engines, imgs, g["flips"], first, g["first_objs"], (g["H"], g["W"]), new_objects=new,
                                         forced_labels=forced, prob_frames=[t for t in g["prob"] if t < T])
    for t, p in probs.items():
        ref = g["prob"][t]
        assert (p[0, :ref.shape[0]] - ref).abs().max().item() < S.PROB_TOL
    # the same CPU arithmetic as the reference's: the generator pinned these at 0 mismatches
    for t, lab in enumerate(ens, start=1):
        assert torch.equal(lab.reshape(g["H"], g["W"]), g["ens"][t - 1]), t


def test_tta_engine_refusals(monkeypatch):
    from aot_benchmark_b200 import TTAInferEngine
    from oracle import weights as OW
    _install(monkeypatch)
    m = S.model("aott", OW.build_state_dict("aott", seed=0))
    with pytest.raises(ValueError, match="1 to 8 augmentations"):
        TTAInferEngine(m, flip=True, multi_scale=[0.75, 1.0, 1.25, 1.5, 1.75])            # 10 augmentations
    assert len(TTAInferEngine(m, flip=True, multi_scale=[0.75, 1.0, 1.25, 1.5]).aug_engines) == 8
    m.cfg.MODEL_USE_PREV_PROB = True
    with pytest.raises(NotImplementedError, match="evaluator.py:438"):
        TTAInferEngine(m, flip=True, multi_scale=[1.0])
    m.cfg.MODEL_USE_PREV_PROB = False
    eng = TTAInferEngine(m)                                   # cfg.TEST_FLIP / TEST_MULTISCALE defaults: one augmentation
    assert eng.flips == [False]
    with pytest.raises(NotImplementedError):
        eng.enable_kv_sharding(0, 2)
