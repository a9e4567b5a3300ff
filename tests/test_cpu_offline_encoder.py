"""CPU: the offline-encoder protocol (AOTEngine.offline_encoder and the image-free add_reference_frame /
match_propogate_one_frame that read the stored features) under the C-ABI emulations of tests/emu_ops.py: the same logits
as the per-frame path and the reference goldens, its protocol edges, and static graph bodies across offline frames,
encoder chunks and videos."""
import os

import pytest
import torch

from oracle import aot_oracle as O
from oracle import weights as OW
from offline_support import clip_masks, run_video_events_offline, run_video_offline


def _engine(model_name, sd, gap, skip=None):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", model_name)
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    model.load_state_dict(sd, strict=True)
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                       short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP if skip is None else skip)
    eng.eval()
    return eng


def _golden_clip(golden_dir, name, T_max=6):
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    T = min(g["frames"], T_max)
    sd = OW.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    return g, sd, frames[:T], mask


@pytest.mark.parametrize("stored_masks", [True, False])
@pytest.mark.parametrize("name", ["aott_raw_257", "deaott_small", "r50_aotl_small"])
def test_offline_path_matches_per_frame_path_and_golden(monkeypatch, golden_dir, name, stored_masks):
    import emu_ops
    from aot_benchmark_b200 import engine
    emu_ops.install_engine(monkeypatch)
    monkeypatch.setattr(engine, "OFFLINE_ENC_CHUNK", 4)            # a full chunk and a partial one
    g, sd, frames, mask = _golden_clip(golden_dir, name)
    forced = [l.float() for l in g["ref_labels"]]
    out = tuple(g["out_size"])
    eng = _engine(g["model"], sd, g["gap"], g.get("skip"))
    with torch.no_grad():
        lo_f, lab_f = O.run_video(eng, frames, mask, g["objs"], out, forced_masks=forced)
        lo_o, lab_o = run_video_offline(eng, frames, mask, g["objs"], out, forced_masks=forced, stored_masks=stored_masks)
    n = g["objs"] + 1
    assert len(lo_o) == len(lo_f) == len(frames) - 1
    for a, b, ref in zip(lo_o, lo_f, g["ref_logits_lo"]):
        assert (a[:, :n] - b[:, :n]).abs().max().item() < 1e-5           # the batched emulated conv may round differently
        assert (a[:, :n] - ref[:, :n]).abs().max().item() < 2e-4
    for a, b in zip(lab_o, lab_f):
        assert torch.equal(a, b)
    e0 = eng.aot_engines[0]
    assert e0.enable_offline_enc and e0.total_offline_frame_num == len(frames)


def test_offline_path_with_14_objects_appearing_mid_video(monkeypatch, golden_dir):
    import emu_ops
    from aot_benchmark_b200 import engine
    emu_ops.install_engine(monkeypatch)
    monkeypatch.setattr(engine, "OFFLINE_ENC_CHUNK", 3)
    g = torch.load(os.path.join(golden_dir, "events_aott_multi14_events.pt"))
    sd = OW.build_state_dict(g["model"], seed=g["seed"])
    frames, full = O.synthetic_video(g["frames"], g["H"], g["W"], 14, seed=g["video_seed"])
    first = torch.where(full <= g["first_objs"], full, torch.zeros_like(full))
    eng = _engine(g["model"], sd, g["gap"])
    with torch.no_grad():
        lo = run_video_events_offline(eng, frames, first, g["first_objs"], tuple(g["out_size"]),
                                      {g["event_frame"]: g["new_label"].float()}, [l.float() for l in g["ref_labels"]])
    assert len(eng.aot_engines) == 2
    for a, b, n in zip(lo, g["ref_logits"], g["live_channels"]):
        assert (a[:, :n] - b).abs().max().item() < 2e-4


def test_protocol_edges(monkeypatch):
    import emu_ops
    from aot_benchmark_b200 import engine
    emu_ops.install_engine(monkeypatch)
    monkeypatch.setattr(engine, "OFFLINE_ENC_CHUNK", 2)
    sd = OW.build_state_dict("aott", seed=3)
    frames, mask = O.synthetic_video(3, 97, 129, 2, seed=8)
    eng = _engine("aott", sd, 2)
    clip = torch.cat(frames)
    with torch.no_grad():
        base, _ = run_video_offline(eng, frames, mask, 2, (97, 129))
        # an image handed while offline encoding is on is ignored
        eng.restart_engine()
        eng.offline_encoder(clip, clip_masks(mask, 3))
        junk = torch.full_like(frames[0], 7.0)
        eng.add_reference_frame(junk, obj_nums=[2], frame_step=0)
        got = []
        for t in range(1, 3):
            eng.match_propogate_one_frame(junk)
            eng.decode_current_logits((97, 129))
            got.append(eng.aot_engines[0].pred_id_logits.clone())
            eng.update_memory(torch.zeros(1, 1, 97, 129))
        assert torch.equal(got[0], base[0])
        # a step past the stored clip
        with pytest.raises(IndexError, match="outside the clip"):
            eng.match_propogate_one_frame()
        assert eng.aot_engines[0].frame_step == 2                   # the failed call did not advance the step
        with pytest.raises(IndexError, match="outside the clip"):
            eng.add_reference_frame(obj_nums=[2], frame_step=3)
        # restart_engine drops the stored clip
        e0 = eng.aot_engines[0]
        eng.restart_engine()
        assert not e0.enable_offline_enc and e0.offline_enc_embs is None and e0.offline_masks is None
        assert e0.total_offline_frame_num == 0 and not eng.enable_offline_enc
        # bad inputs
        single = engine.AOTEngine(eng.AOT, long_term_mem_gap=2)
        with pytest.raises(ValueError, match=r"\[T,3,H,W\]"):
            single.offline_encoder(clip[:, :2])
        with pytest.raises(ValueError, match=r"\[T,3,H,W\]"):
            single.offline_encoder(clip[0])
        with pytest.raises(ValueError, match=r"all_masks must be \[T,1,H,W\]"):
            single.offline_encoder(clip, torch.zeros(2, 1, 97, 129))
        with pytest.raises(ValueError, match=r"all_masks must be \[T,1,H,W\]"):
            single.offline_encoder(clip, torch.zeros(3, 97, 129))
        assert not single.enable_offline_enc


def test_cpu_tensors_are_refused():
    """Without the emulations the engine refuses a CPU clip, as it refuses a CPU frame."""
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", "aott")
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=-1)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        eng.offline_encoder(torch.zeros(2, 3, 65, 65))


@pytest.mark.parametrize("T", [1, 3, 4])
def test_clip_lengths_around_the_chunk(monkeypatch, T):
    """T = 1, T = chunk and T = chunk + 1 (chunk 3): every stored frame equals the per-frame encoder's maps of that frame,
    and the sizes are set from the clip."""
    import emu_ops
    from aot_benchmark_b200 import engine
    emu_ops.install_engine(monkeypatch)
    monkeypatch.setattr(engine, "OFFLINE_ENC_CHUNK", 3)
    sd = OW.build_state_dict("aott", seed=3)
    frames, mask = O.synthetic_video(T, 81, 113, 1, seed=9)
    eng = engine.AOTEngine(_engine("aott", sd, 2).AOT, long_term_mem_gap=2)
    with torch.no_grad():
        eng.offline_encoder(torch.cat(frames))
        assert eng.offline_frames == eng.total_offline_frame_num == len(eng.offline_enc_embs) == T
        assert eng.input_size_2d == (81, 113) and eng.enc_size_2d == tuple(eng.offline_enc_embs[0][-1].shape[2:])
        for t in range(T):
            ref = eng._encode(frames[t], 0)
            got = eng.offline_enc_embs[t]
            assert len(got) == len(ref) == 4
            for a, b, an, bn in zip(got, ref, got.nhwc, ref.nhwc):
                assert a.shape == b.shape and an.shape == bn.shape
                assert (a - b).abs().max().item() < 1e-5 * max(b.abs().max().item(), 1.0)   # CPU conv rounding at B > 1
        eng.add_reference_frame(mask=mask, obj_nums=[1], frame_step=0)
        for t in range(1, T):
            eng.match_propogate_one_frame()
            eng.decode_current_logits((81, 113))
            eng.update_short_term_memory(torch.zeros(1, 1, 81, 113))


@pytest.mark.parametrize("model_name,objs", [("aott", 3), ("aott", 14), ("deaott", 3), ("r50_aotl", 2)])
def test_graph_bodies_are_static_across_offline_frames_chunks_and_videos(monkeypatch, model_name, objs):
    """The LSTT, decoder, memory-update and batched encoder bodies issue identical launches over identical memory across
    offline frames, full chunks and the overlapping tail chunk, and two videos (the tracer of test_cpu_graph_static)."""
    from test_cpu_graph_static import TracingGraphCache, _install
    from aot_benchmark_b200 import engine
    _install(monkeypatch)
    monkeypatch.setattr(engine, "OFFLINE_ENC_CHUNK", 2)
    sd = OW.build_state_dict(model_name, seed=4)
    eng = _engine(model_name, sd, 2)
    outs = []
    for video in range(2):
        frames, mask = O.synthetic_video(5, 97, 129, objs, seed=31)
        with torch.no_grad():
            lo, _ = run_video_offline(eng, frames, mask, objs, (97, 129))
        outs.append(lo)
    assert TracingGraphCache.replays > 8
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)


def test_encoder_keeps_one_batched_set_whatever_the_clip_lengths(monkeypatch):
    """Clips of many lengths (shorter than a chunk, a chunk, and longer with every remainder) leave the encoder with the
    buffers and graph of at most two batch sizes: 1 (the per-frame path) and OFFLINE_ENC_CHUNK.  The tail of a long clip runs
    at the chunk size over the clip's last frames, and the one pass of a short clip is freed when the call returns."""
    import emu_ops
    from aot_benchmark_b200 import engine
    emu_ops.install_engine(monkeypatch)
    monkeypatch.setattr(engine, "OFFLINE_ENC_CHUNK", 4)
    sd = OW.build_state_dict("aott", seed=3)
    frames, mask = O.synthetic_video(11, 65, 97, 1, seed=9)
    eng = engine.AOTEngine(_engine("aott", sd, 2).AOT, long_term_mem_gap=2)
    seen = set()
    with torch.no_grad():
        eng.add_reference_frame(frames[0], mask, obj_nums=[1], frame_step=0)       # the per-frame path's B = 1 set
        for T in (3, 4, 5, 6, 7, 9, 11, 2, 1, 10):
            eng.restart_engine()
            calls = []
            enc_call = engine._Encoder.__call__
            monkeypatch.setattr(engine._Encoder, "__call__", lambda self, img, st: calls.append(img.shape[0]) or
                                enc_call(self, img, st))
            eng.offline_encoder(torch.cat(frames[:T]))
            monkeypatch.setattr(engine._Encoder, "__call__", enc_call)
            seen.update(calls)
            assert calls == ([T] if T < 4 else [4] * -(-T // 4)), (T, calls)
            assert set(eng._enc.batch_sizes()) <= {1, 4}, (T, eng._enc.batch_sizes())
            for t in range(T):                                      # the overlapping tail stored every frame once, right
                ref = eng._encode(frames[t], 0)
                for a, b in zip(eng.offline_enc_embs[t].nhwc, ref.nhwc):
                    assert (a - b).abs().max().item() < 1e-5 * max(b.abs().max().item(), 1.0), (T, t)
    assert seen >= {1, 2, 3, 4}


@pytest.mark.parametrize("name,chunk", [("swinb_aotl_small", 2), ("aotl_mbv3_small", 2), ("rs50_aotl_small", 2)])
def test_offline_path_swin_mobilenetv3_resnest(monkeypatch, golden_dir, name, chunk):
    """Swin-B, MobileNetV3 and ResNeSt-50 on the offline path with the batched entry points emulated (tests/emu_batched.py):
    the same logits as the per-frame path and the reference golden's tolerance, over full chunks and an overlapping tail."""
    import emu_batched
    import emu_ops
    from aot_benchmark_b200 import engine
    if name.startswith("swinb"):
        emu_ops.install_engine(monkeypatch)
        g, sd, frames, mask = _golden_clip(golden_dir, name, T_max=3)
        eng = _engine(g["model"], sd, g["gap"], g.get("skip"))
    else:
        from oracle import mobilenetv3_oracle as MO
        import test_cpu_mbv3_rs50_host as MH
        MH._install(monkeypatch)
        g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
        sd = MO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
        frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
        frames = frames[:3]
        eng = MH._engine(g["model"], sd, g["gap"])
    emu_batched.install(monkeypatch)
    monkeypatch.setattr(engine, "OFFLINE_ENC_CHUNK", chunk)
    forced = [l.float() for l in g["ref_labels"]]
    out = tuple(g["out_size"])
    with torch.no_grad():
        lo_f, _ = O.run_video(eng, frames, mask, g["objs"], out, forced_masks=forced)
        lo_o, _ = run_video_offline(eng, frames, mask, g["objs"], out, forced_masks=forced)
    n = g["objs"] + 1
    assert len(lo_o) == len(lo_f) == len(frames) - 1
    for a, b, ref in zip(lo_o, lo_f, g["ref_logits_lo"]):
        assert (a[:, :n] - b[:, :n]).abs().max().item() < 1e-5
        assert (a[:, :n] - ref[:, :n]).abs().max().item() < 2e-4
    assert set(eng.aot_engines[0]._enc.batch_sizes()) <= {1, chunk}
