"""CPU: the host side of the fp16 inference mode (precision="fp16"), through the emulated C ABI.

- Every tensor-core conv / linear launch of an fp16 engine passes wl = NULL (the single-pass kernel) and every tensor-core
  attention launch has the exact bit clear; an fp32 engine's launches are unchanged.
- Two engines of different precision interleaved in one process each launch in their own mode.
- Captured bodies stay static across frames, bank growth and videos in fp16 mode.
- The keyword, cfg.TEST_PRECISION and their precedence; the knobs and the sharded bank that fp16 mode refuses."""
import pytest
import torch

import fp16_support as F16
from oracle import aot_oracle as O
from oracle import weights as OW


class _FakeLib:
    """Stands in for libaotb200.so under the real ops.conv2d / ops.linear: records the wl pointer of every tensor-core
    launch (the emulation computes the values)."""

    def __init__(self):
        self.wl = []

    def aotb_conv2d_nhwc_tc(self, *args):
        self.wl.append(args[2])
        return 0

    def aotb_conv2d_nhwc_f32(self, *args):
        return 0

    def aotb_linear_f32(self, *args):
        return 0


def _install_traced(monkeypatch):
    """fp16_support emulations, with the real ops.conv2d / ops.linear run first against a fake library and every
    tensor-core attention call's `exact` recorded.  -> (fake library, list of exact bits)."""
    from aot_benchmark_b200 import ops
    real_conv2d, real_linear = ops.conv2d, ops.linear
    F16.install_engine(monkeypatch)
    fake, exact = _FakeLib(), []
    monkeypatch.setattr(ops, "lib", lambda: fake)
    monkeypatch.setattr(ops, "_chk", lambda *ts: None)
    monkeypatch.setattr(ops, "_tc_workspace", lambda dev: torch.zeros(1, dtype=torch.uint8))

    def conv2d(*a, **k):
        real_conv2d(*a, **k)
        return F16.conv2d(*a, **k)

    def linear(*a, **k):
        real_linear(*a, **k)
        return F16.linear(*a, **k)

    def attn(fn):
        def wrapper(*a, **k):
            exact.append(k.get("exact", True))
            return fn(*a, **k)
        return wrapper
    monkeypatch.setattr(ops, "conv2d", conv2d)
    monkeypatch.setattr(ops, "linear", linear)
    monkeypatch.setattr(ops, "lt_attention_tc", attn(F16.lt_attention_tc))
    monkeypatch.setattr(ops, "gp_attention_tc", attn(F16.gp_attention_tc))
    return fake, exact


def _run(eng, objs=3, H=97, W=129, frames=4, seed=31):
    fr, mask = O.synthetic_video(frames, H, W, objs, seed=seed)
    with torch.no_grad():
        return O.run_video(eng, fr, mask, objs, (H, W))


@pytest.mark.parametrize("model_name,objs", [("aott", 3), ("deaott", 3), ("r50_aotl", 2), ("aott", 14)])
def test_fp16_engine_launches_single_pass_kernels(monkeypatch, model_name, objs):
    fake, exact = _install_traced(monkeypatch)
    sd = OW.build_state_dict(model_name, seed=4)
    calls = {}
    for prec in ("fp32", "fp16"):
        fake.wl.clear()
        exact.clear()
        _run(F16.build_engine(model_name, sd, 2, prec), objs=objs)
        calls[prec] = (list(fake.wl), list(exact))
    wl32, ex32 = calls["fp32"]
    wl16, ex16 = calls["fp16"]
    assert len(wl16) == len(wl32) > 20 and len(ex16) == len(ex32) > 4
    assert all(p is not None for p in wl32) and all(ex32)
    assert all(p is None for p in wl16), "an fp16 engine launched the split conv"
    assert not any(ex16), "an fp16 engine launched exact attention"


def test_interleaved_engines_keep_their_precision(monkeypatch):
    """An fp32 engine driven frame by frame alternately with an fp16 engine gives bitwise what it gives alone, and
    differs from the fp16 engine."""
    F16.install_engine(monkeypatch)
    sd = OW.build_state_dict("aott", seed=4)
    clip = O.synthetic_video(4, 97, 129, 3, seed=31)
    alone = [interleaved([F16.build_engine("aott", sd, 2, p)], *clip)[0] for p in ("fp32", "fp16")]
    both = interleaved([F16.build_engine("aott", sd, 2, p) for p in ("fp32", "fp16")], *clip)
    for i in range(2):
        assert len(both[i]) == len(alone[i]) == 3
        assert all(torch.equal(a, b) for a, b in zip(both[i], alone[i]))
    assert not any(torch.equal(a, b) for a, b in zip(*both))


def interleaved(engs, frames, mask, objs=3):
    """Drive the engines frame by frame, alternating between them -> per engine, the low-resolution logits of every
    propagated frame."""
    H, W = mask.shape[-2:]
    outs = [[] for _ in engs]
    with torch.no_grad():
        for e in engs:
            e.restart_engine()
            e.add_reference_frame(frames[0], mask, obj_nums=[objs], frame_step=0)
        for t in range(1, len(frames)):
            for i, e in enumerate(engs):
                e.match_propogate_one_frame(frames[t])
                lo = e.decode_current_logits((H, W))
                outs[i].append(e.pred_id_logits.clone())
                e.update_memory(lo.argmax(1, keepdim=True).float())
    return outs


@pytest.mark.parametrize("model_name", ["aott", "deaott"])
def test_fp16_captured_bodies_are_static(monkeypatch, model_name):
    """test_cpu_graph_static's tracer over an fp16 engine: two videos, bank re-allocation mid-clip."""
    import test_cpu_graph_static as GS
    from aot_benchmark_b200 import engine
    GS._install(monkeypatch)
    for name in F16.EMULATED:
        monkeypatch.setattr(engine.ops, name, GS._traced(name, getattr(F16, name)))
    monkeypatch.setattr(engine, "BANK_INIT_FRAMES", 2)
    sd = OW.build_state_dict(model_name, seed=4)
    eng = F16.build_engine(model_name, sd, 2, "fp16")
    outs = [_run(eng, frames=8)[0] for _ in range(2)]
    assert GS.TracingGraphCache.replays > 10
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def _cfg_model(model_name="aott", **attrs):
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    cfg = EngineConfig("t", model_name)
    for k, v in attrs.items():
        setattr(cfg, k, v)
    return build_vos_model(cfg.MODEL_VOS, cfg).eval()


def test_precision_keyword_cfg_and_precedence(monkeypatch):
    from aot_benchmark_b200 import TTAInferEngine
    from aot_benchmark_b200.engine import AOTEngine, AOTInferEngine, DeAOTInferEngine
    F16.install_engine(monkeypatch)
    m = _cfg_model()
    assert AOTEngine(m).precision == "fp32" and AOTInferEngine(m).precision == "fp32"
    assert AOTInferEngine(m, precision="fp16").precision == "fp16"
    m16 = _cfg_model(TEST_PRECISION="fp16")
    assert AOTEngine(m16).precision == "fp16"
    assert AOTInferEngine(m16, precision="fp32").precision == "fp32"           # the keyword wins
    t = TTAInferEngine(m16, flip=True, multi_scale=[1.0])
    assert [e.precision for e in t.aug_engines] == ["fp16", "fp16"]
    t = TTAInferEngine(m, flip=True, multi_scale=[1.0], precision="fp16")
    assert [e.precision for e in t.aug_engines] == ["fp16", "fp16"]
    assert DeAOTInferEngine(_cfg_model("deaott"), precision="fp16").precision == "fp16"
    # sub-engines inherit it, pooled ones keep it
    eng = AOTInferEngine(_cfg_model(), precision="fp16")
    _run(eng, objs=14, frames=2)
    assert [e.precision for e in eng.aot_engines] == ["fp16", "fp16"]
    for bad in ("bf16", "FP16", 16, "amp"):
        with pytest.raises(ValueError, match="precision"):
            AOTInferEngine(m, precision=bad)
        with pytest.raises(ValueError, match="precision"):
            AOTEngine(_cfg_model(TEST_PRECISION=bad))


def test_autocast_does_not_select_fp16(monkeypatch):
    from aot_benchmark_b200.engine import AOTInferEngine
    F16.install_engine(monkeypatch)
    with torch.autocast("cpu", dtype=torch.bfloat16):
        assert AOTInferEngine(_cfg_model()).precision == "fp32"


@pytest.mark.parametrize("knob,value,vos", [("LT_IMPL", "simt", "aott"), ("DEAOT_LT", "gemm", "deaott"),
                                            ("DEAOT_LT", "simt", "deaott"), ("CONV_IMPL", "simt", "aott")])
def test_fp16_refuses_fp32_only_paths(monkeypatch, knob, value, vos):
    from aot_benchmark_b200 import engine, ops
    from aot_benchmark_b200.engine import AOTInferEngine, DeAOTInferEngine
    F16.install_engine(monkeypatch)
    monkeypatch.setattr(ops if knob == "CONV_IMPL" else engine, knob, value)
    cls = DeAOTInferEngine if vos == "deaott" else AOTInferEngine
    env = {"LT_IMPL": "AOTB_LT_IMPL", "DEAOT_LT": "AOTB_DEAOT_LT", "CONV_IMPL": "AOTB_CONV_IMPL"}[knob]
    with pytest.raises(NotImplementedError, match=f"{env}={value}"):
        cls(_cfg_model(vos), precision="fp16")
    cls(_cfg_model(vos), precision="fp32")                      # the fp32 mode still takes the knob


def test_fp16_refuses_kv_sharding(monkeypatch):
    from aot_benchmark_b200.engine import AOTEngine, AOTInferEngine
    F16.install_engine(monkeypatch)
    for cls in (AOTEngine, AOTInferEngine):
        with pytest.raises(NotImplementedError, match="fp16"):
            cls(_cfg_model(), precision="fp16").enable_kv_sharding(0, 2)


def test_fp16_emulation_differs_from_fp32_at_fp16_level(monkeypatch):
    """Sanity of the emulation the GPU tests compare with: the fp16 engine's logits move away from the fp32 engine's by
    far more than fp32 rounding and far less than the logits' scale."""
    F16.install_engine(monkeypatch)
    sd = OW.build_state_dict("aott", seed=4)
    lo32, _ = _run(F16.build_engine("aott", sd, 2, "fp32"))
    lo16, _ = _run(F16.build_engine("aott", sd, 2, "fp16"))
    d = max((a[:, :4] - b[:, :4]).abs().max().item() for a, b in zip(lo32, lo16))     # 3 objects + background
    s = max(a[:, :4].abs().max().item() for a in lo32)
    assert 1e-5 * s < d < 0.05 * s, (d, s)
