"""GPU: the batched encoder kernels (image b of a B-image launch equals the one-image launch on image b, bit for bit), the
batched encoder of every family against the single-frame encoder, and the engines on the offline path (offline_encoder,
then add_reference_frame / match_propogate_one_frame without images) against the reference goldens and the per-frame path."""
import os

import pytest
import torch

from offline_support import clip_masks, run_video_events_offline, run_video_offline

pytestmark = pytest.mark.gpu

BATCHES = [1, 2, 3, 5]


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rand(*shape, seed=0, scale=1.0):
    return (torch.randn(*shape, generator=_gen(seed)) * scale).cuda()


# ------------------------------------------------------------------ kernels
@pytest.mark.parametrize("B", BATCHES)
def test_image_to_nhwc4_batched(B):
    from aot_benchmark_b200 import ops
    img = _rand(B, 3, 37, 53, seed=B)
    out = torch.empty(B, 37, 53, 4, device="cuda")
    ops.image_to_nhwc4(img, out)
    for b in range(B):
        one = torch.empty(1, 37, 53, 4, device="cuda")
        ops.image_to_nhwc4(img[b:b + 1], one)
        assert torch.equal(out[b:b + 1], one)
    again = torch.empty_like(out)
    ops.image_to_nhwc4(img, again)
    assert torch.equal(out, again)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("H,W,shift", [(14, 21, 0), (14, 21, 3), (17, 23, 3), (10, 9, 0), (25, 38, 3)])
def test_window_attention_batched(B, H, W, shift):
    """H or W not a multiple of 7 (per-image padding), shifted windows (per-image roll and mask)."""
    from aot_benchmark_b200 import ops
    heads, C = 4, 128
    qkv = _rand(B * H * W, 3 * C, seed=H * W + B)
    bias = _rand(3 * C, seed=1, scale=0.5)
    relb = _rand(heads, 49, 49, seed=2, scale=0.5)
    out = torch.empty(B * H * W, C, device="cuda")
    ops.window_attention(qkv, bias, relb, out, H, W, heads, shift, B=B)
    n = H * W
    for b in range(B):
        one = torch.empty(n, C, device="cuda")
        ops.window_attention(qkv[b * n:(b + 1) * n], bias, relb, one, H, W, heads, shift)
        assert torch.equal(out[b * n:(b + 1) * n], one), b
    again = torch.empty_like(out)
    ops.window_attention(qkv, bias, relb, again, H, W, heads, shift, B=B)
    assert torch.equal(out, again)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("H,W", [(9, 13), (8, 12), (1, 7)])
def test_patch_merge_batched(B, H, W):
    from aot_benchmark_b200 import ops
    C = 64
    x = _rand(B * H * W, C, seed=B + H)
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    out = torch.empty(B * H2 * W2, 4 * C, device="cuda")
    ops.patch_merge(x, out, H, W, B=B)
    n, m = H * W, H2 * W2
    for b in range(B):
        one = torch.empty(m, 4 * C, device="cuda")
        ops.patch_merge(x[b * n:(b + 1) * n], one, H, W)
        assert torch.equal(out[b * m:(b + 1) * m], one)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("C,H,W,pool", [(64, 33, 47, 0), (64, 33, 47, 2), (128, 61, 75, 2), (256, 17, 9, 0)])
def test_splat_attention_and_combine_batched(B, C, H, W, pool):
    """Per-image pixel means (many CTAs per image: each image keeps its own partials and counter) and per-image avd pool."""
    from aot_benchmark_b200 import ops
    inter = 32
    x = _rand(B, H, W, 2 * C, seed=C + B, scale=2.0)
    w1, b1 = _rand(C, inter, seed=3, scale=0.2), _rand(inter, seed=4, scale=0.2)
    w2, b2 = _rand(inter, 2 * C, seed=5, scale=0.2), _rand(2 * C, seed=6, scale=0.2)
    ws = ops.splat_workspace(C, "cuda", B)
    att = torch.empty(B, 2 * C, device="cuda")
    ops.splat_attention(x, w1, b1, w2, b2, att, ws)
    Ho, Wo = (ops.pool2d_size(H, 3, pool, 1), ops.pool2d_size(W, 3, pool, 1)) if pool else (H, W)
    out = torch.empty(B, Ho, Wo, C, device="cuda")
    ops.splat_combine(x, att, out, pool_stride=pool)
    ws1 = ops.splat_workspace(C, "cuda")
    for b in range(B):
        a1 = torch.empty(2 * C, device="cuda")
        ops.splat_attention(x[b:b + 1], w1, b1, w2, b2, a1, ws1)
        assert torch.equal(att[b], a1), b
        o1 = torch.empty(1, Ho, Wo, C, device="cuda")
        ops.splat_combine(x[b:b + 1], a1, o1, pool_stride=pool)
        assert torch.equal(out[b:b + 1], o1), b
    att2 = torch.empty_like(att)
    ops.splat_attention(x, w1, b1, w2, b2, att2, ws)          # the counters were left at zero
    assert torch.equal(att, att2)
    if B > 1:
        with pytest.raises(ops.AotbError, match="workspace"):
            ops.splat_attention(x, w1, b1, w2, b2, att2, ws1)      # a one-image workspace is too small for B images


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("C,H,W,sliced", [(96, 29, 41, True), (480, 15, 21, False), (960, 7, 9, True)])
def test_se_gate_and_gate_scale_batched(B, C, H, W, sliced):
    """SE on channel-slice inputs (the row stride is wider than C), gate * x with h_swish."""
    from aot_benchmark_b200 import ops
    inter = C // 4
    full = _rand(B, H, W, C + 32 if sliced else C, seed=C + B, scale=2.0)
    x = full[..., :C]
    w1, b1 = _rand(C, inter, seed=7, scale=0.1), _rand(inter, seed=8, scale=0.1)
    w2, b2 = _rand(inter, C, seed=9, scale=0.1), _rand(C, seed=10, scale=0.1)
    ws = ops.splat_workspace(C, "cuda", B)
    gate = torch.empty(B, C, device="cuda")
    ops.se_gate(x, w1, b1, w2, b2, gate, ws)
    out = torch.empty(B, H, W, C, device="cuda")
    ops.gate_scale(x, gate, out, act=ops.ACT_HSWISH)
    ws1 = ops.splat_workspace(C, "cuda")
    for b in range(B):
        g1 = torch.empty(C, device="cuda")
        ops.se_gate(x[b:b + 1], w1, b1, w2, b2, g1, ws1)
        assert torch.equal(gate[b], g1), b
        o1 = torch.empty(1, H, W, C, device="cuda")
        ops.gate_scale(x[b:b + 1], g1, o1, act=ops.ACT_HSWISH)
        assert torch.equal(out[b:b + 1], o1), b
    gate2 = torch.empty_like(gate)
    ops.se_gate(x, w1, b1, w2, b2, gate2, ws)
    assert torch.equal(gate, gate2)


# ------------------------------------------------------------------ batched encoder
_MO_CASES = {"aotl_mbv3": "AOTL with mobilenetv3", "rs50_aotl": "R50-AOTL with resnest50"}


def _model(name, seed=0):
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    from oracle import mobilenetv3_oracle as MO
    from oracle import resnest_oracle as RO
    from oracle import weights as OW
    if name in _MO_CASES:
        sd = MO.build_state_dict(_MO_CASES[name], seed=seed)
        cfg = MO.engine_config(_MO_CASES[name], "t")
    else:
        sd = (RO if name in RO.MODELS else OW).build_state_dict(name, seed=seed)
        cfg = EngineConfig("t", name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    return model.cuda().eval()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("name", ["aott", "aotl_mbv3", "r50_aotl", "r101_aotl", "rs50_aotl", "rs101_aotl", "swinb_aotl"])
def test_batched_encoder_vs_single_frame(name, precision):
    """Every family, B = 3 (and Swin at a size that needs its pad to a multiple of 4): each frame and level within the
    split-K bounds of the single-frame encoder; the replayed graph equals the eager pass bit for bit."""
    from aot_benchmark_b200 import engine, ops, plan
    model = _model(name)
    H, W = (98, 131) if name.startswith("swinb") else (97, 129)
    imgs = _rand(3, 3, H, W, seed=11)
    tol = 1e-5 if precision == "fp32" else 2e-2
    st = torch.cuda.current_stream().cuda_stream
    with torch.no_grad(), ops.precision(precision):
        enc = engine._Encoder(plan.get_plan(model), H, W)
        singles = []
        for b in range(3):
            singles.append([t.clone() for t in enc(imgs[b:b + 1], st).nhwc])
        runs = []
        for rep in range(3):                                          # eager, capture, replay
            runs.append([t.clone() for t in enc(imgs, st).nhwc])
        again = [t.clone() for t in enc(imgs[1:2], st).nhwc]         # B = 1 after B = 3: its own buffers and graph
    torch.cuda.synchronize()
    for lvl, (x, y) in enumerate(zip(again, singles[1])):
        assert torch.equal(x, y), lvl
    for r in runs[1:]:
        for x, y in zip(r, runs[0]):
            assert torch.equal(x, y)
    for b in range(3):
        for lvl, (x, ref) in enumerate(zip(runs[0], singles[b])):
            d = (x[b:b + 1] - ref).abs().max().item()
            assert d <= tol * max(ref.abs().max().item(), 1.0), (b, lvl, d)


# ------------------------------------------------------------------ engines on the offline path
def _engine(model_name, sd, gap, **kw):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", model_name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                       short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP, **kw)
    eng.eval()
    return eng


@pytest.mark.parametrize("name", ["r50_aotl_small", "r50_deaotl_small", "swinb_aotl_small"])
def test_offline_engine_vs_reference_golden(name, golden_dir):
    from oracle import aot_oracle as O
    from oracle import weights as OW
    from test_gpu_engine import _tie_band_ok
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    sd = OW.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    eng = _engine(g["model"], sd, g["gap"])
    with torch.no_grad():
        lo, labels = run_video_offline(eng, [f.cuda() for f in frames], mask.cuda(), g["objs"], tuple(g["out_size"]),
                                       forced_masks=[l.float() for l in g["ref_labels"]])
    n = g["objs"] + 1
    dmax = max((a.cpu()[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(lo, g["ref_logits_lo"]))
    print(f"{name} offline: max |dlogit| vs reference = {dmax:.3e}")
    assert dmax < 1e-3, dmax
    assert _tie_band_ok(lo, g["ref_logits_lo"], labels, g["ref_labels"], tuple(g["out_size"]), n) == 0


def test_offline_fourteen_objects_vs_reference_golden(golden_dir):
    from oracle import aot_oracle as O
    from oracle import weights as OW
    g = torch.load(os.path.join(golden_dir, "events_aott_multi14_events.pt"))
    sd = OW.build_state_dict(g["model"], seed=g["seed"])
    frames, full = O.synthetic_video(g["frames"], g["H"], g["W"], 14, seed=g["video_seed"])
    first = torch.where(full <= g["first_objs"], full, torch.zeros_like(full))
    eng = _engine(g["model"], sd, g["gap"])
    with torch.no_grad():
        lo = run_video_events_offline(eng, [f.cuda() for f in frames], first.cuda(), g["first_objs"], tuple(g["out_size"]),
                                      {g["event_frame"]: g["new_label"].float()},
                                      [l.float() for l in g["ref_labels"]])
    assert len(eng.aot_engines) == 2
    dmax = max((a.cpu()[:, :n] - b).abs().max().item() for a, b, n in zip(lo, g["ref_logits"], g["live_channels"]))
    assert dmax < 1e-3, dmax


def _both_paths(eng, frames, mask, objs, size):
    from oracle import aot_oracle as O
    with torch.no_grad():
        lo_f, lab_f = O.run_video(eng, frames, mask, objs, size)
        lo_o, lab_o = run_video_offline(eng, frames, mask, objs, size, forced_masks=lab_f)
    return lo_f, lab_f, lo_o, lab_o


@pytest.mark.parametrize("model_name,objs,kw,tol", [
    ("r50_aotl", 5, {}, 1e-3), ("r50_deaotl", 5, {}, 1e-3), ("swinb_aotl", 3, {}, 1e-3), ("aott", 14, {}, 1e-3),
    ("r50_aotl", 5, {"precision": "fp16"}, 2e-2),
    ("r50_aotl", 5, {"long_term_mem_max": 3}, 1e-3),
    ("r50_aotl", 5, {"long_term_mem_max": 3, "long_term_mem_policy": "usage"}, 1e-3)])
def test_offline_path_vs_per_frame_path_on_a_20_frame_clip(model_name, objs, kw, tol):
    """20 frames, memory every 2nd frame: the offline path (chunks of OFFLINE_ENC_CHUNK frames, stored masks) against the
    per-frame path of the same engine, teacher-forced on the per-frame labels; labels equal outside the tie band.  Also in
    fp16 and with the bounded bank in FIFO and usage eviction."""
    from oracle import aot_oracle as O
    from oracle import weights as OW
    from test_gpu_engine import _tie_band_ok
    H, W = (192, 288) if model_name.startswith("swinb") else (193, 289)
    sd = OW.build_state_dict(model_name, seed=6)
    frames, mask = O.synthetic_video(20, H, W, objs, seed=60)
    eng = _engine(model_name, sd, 2, **kw)
    lo_f, lab_f, lo_o, lab_o = _both_paths(eng, [f.cuda() for f in frames], mask.cuda(), objs, (H, W))
    n = objs + 1
    dmax = max((a[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(lo_o, lo_f))
    print(f"{model_name} {kw}: offline vs per-frame max |dlogit| = {dmax:.3e}")
    assert dmax < tol, dmax
    assert _tie_band_ok(lo_o, [t.cpu() for t in lo_f], lab_o, lab_f, (H, W), n) == 0
    if kw.get("long_term_mem_policy") == "usage":
        assert eng.long_term_memory_usage[0] is not None


def test_offline_graphs_vs_eager(monkeypatch):
    """The offline path with graphs (two videos: the second replays every body) equals the same path run eagerly."""
    from aot_benchmark_b200 import engine
    from oracle import aot_oracle as O
    from oracle import weights as OW
    sd = OW.build_state_dict("r50_aotl", seed=2)
    frames, mask = O.synthetic_video(11, 129, 193, 3, seed=5)
    frames, mask = [f.cuda() for f in frames], mask.cuda()
    eng = _engine("r50_aotl", sd, 2)
    with torch.no_grad():
        run_video_offline(eng, frames, mask, 3, (129, 193))
        graphed, _ = run_video_offline(eng, frames, mask, 3, (129, 193))
        monkeypatch.setattr(engine, "USE_GRAPHS", False)
        eager, _ = run_video_offline(_engine("r50_aotl", sd, 2), frames, mask, 3, (129, 193))
    for a, b in zip(graphed, eager):
        assert torch.equal(a, b)
