"""GPU: the fp16 inference mode.

- The single-pass tensor-core conv (aotb_conv2d_nhwc_tc with wl = NULL) at every forced N tile x split-K size, at M / K tails,
  general Cin, stride 2, batch 2, an aliased residual and every activation: within the fp32-accumulation bound of a float64
  reference over the fp16-rounded operands, visibly off the unrounded one, and bitwise equivariant under weight scaling.
- R50-AOTL, R50-DeAOTL and SwinB-AOTL engines with precision="fp16", teacher-forced on the small goldens: against the
  reference goldens and against the CPU emulation of the same fp16 engine (tests/fp16_support.py); graph replay equals eager
  launches, runs are reproducible, and an fp32 engine interleaved with an fp16 one is unaffected.
- The bounded bank, more than 10 objects and TTAInferEngine in fp16 mode."""
import math
import os

import pytest
import torch

import fp16_support as F16
from test_gpu_tc_envelope import TILING_CASES, _pack_w, _ref_conv, _weight_scale_case

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


# ------------------------------------------------------------------ single-pass conv kernel
def _rounded_w4(wh, ws, Cout, Cin, K):
    """fp16(w 2^e) 2^-e as [Cout, Cin, K, K] float64: the weight the single-pass kernel multiplies by."""
    r = wh[:, :K * K * Cin].double().cpu() * ws.double().cpu().view(-1, 1)
    return r.view(Cout, K, K, Cin).permute(0, 3, 1, 2)


@pytest.mark.parametrize("case", TILING_CASES + [(1, 13, 11, 256, 256, 3, 1, 1, "res", 1, False)],
                         ids=[f"c{i}" for i in range(len(TILING_CASES) + 1)])
def test_single_pass_conv_tiling_sweep(case):
    """Every N tile (64, 128, 256) x split-K size forced: within 1e-5 of max |ref| (+1e-5) of float64 over fp16(x) and
    fp16(w 2^e) 2^-e, reproducible, writes only its columns; against unrounded float64 it is off by more than 1e-4 of
    max |ref| (the lo terms are really gone: measured 1.9e-4 .. 3.8e-4 of max |ref| on an H100)."""
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import lib
    B, H, W, Cin, Cout, K, stride, pad, rmode, act, wide = case
    g = torch.Generator().manual_seed(H * 131 + Cin)
    x = torch.randn(B, H, W, Cin, generator=g) * 2
    w = torch.randn(Cout, Cin, K, K, generator=g) / math.sqrt(Cin * K * K)
    b = torch.randn(Cout, generator=g)
    Ho, Wo = (H + 2 * pad - K) // stride + 1, (W + 2 * pad - K) // stride + 1
    r = torch.randn(B, Ho, Wo, Cout, generator=g) if rmode else None
    wh, _, ws = ops.split_fp16_scaled(_pack_w(w).to(DEV))
    ref16 = _ref_conv(x.half().double(), _rounded_w4(wh, ws, Cout, Cin, K), b, stride, pad, r, act)
    ref = _ref_conv(x, w, b, stride, pad, r, act)
    scale = ref.abs().max().item()
    ex = 8 if wide else 0
    xg = torch.zeros(B, H, W, Cin + ex, device=DEV)
    xg[..., :Cin] = x.to(DEV)
    xv = xg[..., :Cin]
    obuf = torch.full((B, Ho, Wo, Cout + 2 * ex), float("nan"), device=DEV)
    out = obuf[..., ex:ex + Cout]
    rbuf = torch.full((B, Ho, Wo, Cout + ex), float("nan"), device=DEV) if rmode == "res" else None
    if rbuf is not None:
        rbuf[..., :Cout] = r.to(DEV)
    nchunks = (K * K * Cin + 63) // 64
    tried, off = 0, []
    try:
        for bn_code, BN in ((1, 64), (2, 128), (3, 256)):
            if Cout % BN:
                continue
            for S in (1, 2, 4, 8):
                if S > nchunks:
                    continue
                assert lib().aotb_set_conv_tiling((bn_code << 4) | (S << 8)) == 0
                runs = []
                for _ in range(2):
                    obuf.fill_(float("nan"))
                    if rmode == "alias":
                        out.copy_(r.to(DEV))
                    res = out if rmode == "alias" else (None if rbuf is None else rbuf[..., :Cout])
                    ops.conv2d_tc(xv, wh, None, b.to(DEV), out, res=res, KH=K, KW=K, stride=stride, pad=pad, act=act,
                                  wscale=ws)
                    torch.cuda.synchronize()
                    runs.append(obuf.clone())
                o = runs[0][..., ex:ex + Cout].double().cpu()
                err = (o - ref16).abs().max().item()
                assert err < 1e-5 * max(scale, 1.0) + 1e-5, f"BN {BN} S {S}: err {err:.3e} (scale {scale:.2f})"
                off.append((o - ref).abs().max().item() / max(scale, 1.0))
                assert torch.equal(runs[0][..., ex:ex + Cout], runs[1][..., ex:ex + Cout]), f"BN {BN} S {S}: not reproducible"
                for o in runs:
                    assert torch.isnan(o[..., :ex]).all() and torch.isnan(o[..., ex + Cout:]).all(), \
                        f"BN {BN} S {S}: wrote outside its columns"
                tried += 1
    finally:
        lib().aotb_set_conv_tiling(0)
    assert tried >= 1
    print(f"single-pass vs unrounded float64: {min(off):.2e} .. {max(off):.2e} of max |ref|")
    assert min(off) > 1e-4, off


@pytest.mark.parametrize("kind", ["conv3x3", "linear"])
def test_single_pass_weight_scale_equivariance(kind):
    """Weights scaled by 2^k, k = -14 .. 4: the single-pass output is bitwise 2^k times the output at k = 0."""
    from aot_benchmark_b200 import ops
    x, w, pad = _weight_scale_case(kind)
    xg = x.to(DEV)
    K = w.shape[2]
    outs = {}
    for k in range(-14, 5):
        wh, _, ws = ops.split_fp16_scaled(_pack_w(w * 2.0 ** k).to(DEV))
        Ho, Wo = x.shape[1] + 2 * pad - K + 1, x.shape[2] + 2 * pad - K + 1
        out = torch.full((1, Ho, Wo, w.shape[0]), float("nan"), device=DEV)
        ops.conv2d_tc(xg, wh, None, None, out, KH=K, KW=K, pad=pad, wscale=ws)
        outs[k] = out
    torch.cuda.synchronize()
    for k, o in outs.items():
        assert torch.equal(o, outs[0] * 2.0 ** k), f"not equivariant at 2^{k}"


def test_registered_weights_follow_the_precision_context():
    """ops.conv2d / ops.linear with registered weights launch the split kernel by default and the single-pass kernel
    inside ops.precision("fp16"), bit for bit like conv2d_tc with wl = NULL."""
    from aot_benchmark_b200 import ops
    g = torch.Generator().manual_seed(9)
    x = torch.randn(300, 256, generator=g).to(DEV)
    wk = (torch.randn(256, 128, generator=g) / 16).to(DEV)
    wh, wl, ws = ops.split_fp16_scaled(wk)
    ops.register_tc_weights(wk, wh, wl, ws)
    try:
        o32, o16, d16 = (torch.empty(300, 128, device=DEV) for _ in range(3))
        ops.linear(x, wk, None, o32)
        with ops.precision("fp16"):
            ops.linear(x, wk, None, o16)
        ops.conv2d_tc(x.view(1, 300, 1, 256), wh, None, None, d16.view(1, 300, 1, 128), wscale=ws)
        torch.cuda.synchronize()
    finally:
        ops._TC_WEIGHTS.pop(wk.data_ptr(), None)
    assert torch.equal(o16, d16) and not torch.equal(o32, o16)


# ------------------------------------------------------------------ engines
def _golden(golden_dir, name):
    from oracle import aot_oracle as O
    from oracle import weights as OW
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    sd = OW.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    return g, sd, frames, mask


def _run(eng, g, frames, mask, device):
    from oracle import aot_oracle as O
    with torch.no_grad():
        lo, labels = O.run_video(eng, [f.to(device) for f in frames], mask.to(device), g["objs"], tuple(g["out_size"]),
                                 forced_masks=[l.float().to(device) for l in g["ref_labels"]])
    return [t.cpu() for t in lo], labels


def _emulated(g, sd, frames, mask, **kw):
    with pytest.MonkeyPatch.context() as mp:
        F16.install_engine(mp, bounded="long_term_mem_max" in kw)
        return _run(F16.build_engine(g["model"], sd, g["gap"], "fp16", **kw), g, frames, mask, "cpu")[0]


def _dmax(a_list, b_list, n):
    return max((a[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(a_list, b_list))


# (vs golden, vs emulation): measured on an H100 80GB HBM3 (700 W) plus margin, see the test's docstring
TOL = {"r50_aotl_small": (2e-2, 2e-2), "r50_deaotl_small": (2e-2, 2e-2), "swinb_aotl_small": (1.5e-2, 1e-2)}


@pytest.mark.parametrize("name", ["r50_aotl_small", "r50_deaotl_small", "swinb_aotl_small"])
def test_fp16_engine_vs_golden_and_emulation(golden_dir, name):
    """fp16 engine, teacher-forced on the golden clip: max |dlogit| against the fp32 reference golden and against the CPU
    emulation of the same fp16 engine, within TOL[name] = (golden, emulation).  Measured on an H100 (vs golden, vs
    emulation): R50-AOTL 4.3e-3, 4.4e-3; R50-DeAOTL 5.1e-3, 3.8e-3; SwinB-AOTL 3.3e-3, 2.1e-3; the tolerances are about 4x.
    The emulation is not closer than the fp32 golden: fp16(x) is a step function, so fp32 summation-order differences
    upstream flip single roundings, and P is rounded against the running, not the final, row max.  Graph replay equals eager
    launches bitwise over two videos, and two runs are bitwise equal."""
    from aot_benchmark_b200 import engine as engine_mod
    g, sd, frames, mask = _golden(golden_dir, name)
    n = g["objs"] + 1
    eng = F16.build_engine(g["model"], sd, g["gap"], "fp16", device="cuda")
    lo = [_run(eng, g, frames, mask, "cuda")[0] for _ in range(2)]          # second video: replayed graphs
    assert all(torch.equal(a, b) for a, b in zip(*lo)), "fp16 engine not reproducible across videos"
    old = engine_mod.USE_GRAPHS
    engine_mod.USE_GRAPHS = False
    try:
        eager = _run(F16.build_engine(g["model"], sd, g["gap"], "fp16", device="cuda"), g, frames, mask, "cuda")[0]
    finally:
        engine_mod.USE_GRAPHS = old
    assert all(torch.equal(a, b) for a, b in zip(lo[0], eager)), "graph replay differs from eager launches"
    d_gold = _dmax(lo[0], g["ref_logits_lo"], n)
    d_emu = _dmax(lo[0], _emulated(g, sd, frames, mask), n)
    print(f"{name}: fp16 max|dlogit| vs fp32 golden {d_gold:.3e}, vs CPU fp16 emulation {d_emu:.3e}")
    assert d_gold < TOL[name][0] and d_emu < TOL[name][1], (d_gold, d_emu)


def test_fp32_engine_interleaved_with_fp16_engine_is_unchanged(golden_dir):
    """Frame by frame alternation of an fp32 and an fp16 R50-AOTL engine in one process: each gives bitwise the logits it
    gives alone."""
    from test_cpu_fp16_host import interleaved
    g, sd, frames, mask = _golden(golden_dir, "r50_aotl_small")
    clip = ([f.cuda() for f in frames], mask.cuda())
    alone = [interleaved([F16.build_engine(g["model"], sd, g["gap"], p, device="cuda")], *clip, objs=g["objs"])[0]
             for p in ("fp32", "fp16")]
    both = interleaved([F16.build_engine(g["model"], sd, g["gap"], p, device="cuda") for p in ("fp32", "fp16")], *clip,
                       objs=g["objs"])
    for i in range(2):
        assert all(torch.equal(a, b) for a, b in zip(both[i], alone[i]))
    assert not any(torch.equal(a, b) for a, b in zip(*both))


@pytest.mark.parametrize("model_name", ["r50_aotl", "r50_deaotl"])
def test_fp16_bounded_bank_vs_emulation(golden_dir, model_name):
    """long_term_mem_max = 2 on the golden clip (gap 2: the ring wraps): the fp16 engine against its CPU emulation within
    2e-2 (measured on an H100: 4.4e-3 R50-AOTL, 4.1e-3 R50-DeAOTL)."""
    g, sd, frames, mask = _golden(golden_dir, f"{model_name}_small")
    lo = _run(F16.build_engine(g["model"], sd, g["gap"], "fp16", device="cuda", long_term_mem_max=2), g, frames, mask,
              "cuda")[0]
    d = _dmax(lo, _emulated(g, sd, frames, mask, long_term_mem_max=2), g["objs"] + 1)
    print(f"{model_name} bounded: fp16 max|dlogit| vs emulation {d:.3e}")
    assert d < 2e-2, d


@pytest.mark.parametrize("model_name", ["aott", "deaott"])
def test_fp16_fourteen_objects_vs_emulation(model_name):
    """14 objects: two fp16 sub-engines on concurrent streams, against the CPU emulation fed the same labels (merged
    logits), within 8e-3 (measured on an H100: 1.5e-3 AOTT, 1.8e-3 DeAOTT)."""
    from oracle import aot_oracle as O
    from oracle import weights as OW
    sd = OW.build_state_dict(model_name, seed=2)
    frames, mask = O.synthetic_video(4, 129, 161, 14, seed=5)
    with torch.no_grad():
        lo, labels = O.run_video(F16.build_engine(model_name, sd, 2, "fp16", device="cuda"), [f.cuda() for f in frames],
                                 mask.cuda(), 14, (129, 161))
        with pytest.MonkeyPatch.context() as mp:
            F16.install_engine(mp)
            elo, _ = O.run_video(F16.build_engine(model_name, sd, 2, "fp16"), frames, mask, 14, (129, 161),
                                 forced_masks=[l.float().cpu() for l in labels])
    d = _dmax([a.cpu() for a in lo], elo, 15)
    print(f"{model_name} 14 objects: fp16 max|dlogit| vs emulation {d:.3e}")
    assert d < 8e-3, d


def test_fp16_tta_augmentations_equal_standalone_fp16_engines():
    """TTAInferEngine(precision="fp16") with flip: both augmentation engines (concurrent streams) are fp16 and each
    augmentation's logits equal, bitwise, a standalone fp16 engine fed the same (flipped) frames and labels."""
    from aot_benchmark_b200 import TTAInferEngine
    from oracle import aot_oracle as O
    from oracle import weights as OW
    sd = OW.build_state_dict("aott", seed=3)
    H, W, objs = 97, 129, 3
    frames, mask = O.synthetic_video(4, H, W, objs, seed=8)
    frames = [f.cuda() for f in frames]
    forced = [torch.randint(0, objs + 1, (1, 1, H, W), generator=torch.Generator().manual_seed(t)).float().cuda()
              for t in range(len(frames))]
    tta = TTAInferEngine(_model("aott", sd), long_term_mem_gap=2, flip=True, multi_scale=[1.0], precision="fp16")
    assert all(e.precision == "fp16" for e in tta.aug_engines)
    aug = []
    with torch.no_grad():
        tta.add_reference_frame([frames[0], frames[0].flip(-1)], mask.cuda(), obj_nums=[objs])
        for t in range(1, len(frames)):
            tta.propagate([frames[t], frames[t].flip(-1)], (H, W), forced_labels=[forced[t], forced[t]])
            aug.append([m.clone() for m in tta.aug_logits])
        for e, flip in enumerate((False, True)):
            f = (lambda x: x.flip(-1)) if flip else (lambda x: x)
            eng = F16.build_engine("aott", sd, 2, "fp16", device="cuda")
            eng.restart_engine()
            eng.add_reference_frame(f(frames[0]), f(mask.cuda()), obj_nums=[objs], frame_step=0)
            for t in range(1, len(frames)):
                eng.match_propogate_one_frame(f(frames[t]))
                lo = eng.decode_current_logits(None)
                assert torch.equal(lo, aug[t - 1][e]), f"augmentation {e}, frame {t}"
                eng.update_memory(f(forced[t]))


def _model(model_name, sd):
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    cfg = EngineConfig("t", model_name)
    m = build_vos_model(cfg.MODEL_VOS, cfg)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()
