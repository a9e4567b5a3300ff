"""CPU: the MobileNetV3-Large and ResNeSt-50 encoder paths (AOTL with mobilenetv3, R50-AOTL with resnest50) without a GPU --
state_dict contract against the real reference, the oracle against the reference's goldens (with negative controls that show the
fixtures see the MobileNetV3 details), the host orchestration (plan, engine._Encoder, the engines) with every C-ABI entry point
replaced by a torch-CPU emulation of its contract, the captured encoder bodies checked static, and the MODEL_ENCODER_DIM check.
The emulations of the SE entry points live here; the kernels themselves are checked on the GPU (tests/test_gpu_mbv3_rs50.py)."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

import test_cpu_graph_static as GS
import test_cpu_resnest_host as RH
from oracle import aot_oracle as O
from oracle import mobilenetv3_oracle as MO
from oracle import resnest_oracle as RO
from oracle import weights as OW

MBV3, RS50 = "AOTL with mobilenetv3", "R50-AOTL with resnest50"
CLIPS = {"aotl_mbv3_small": MBV3, "rs50_aotl_small": RS50}


# ------------------------------------------------------------------ contract emulations of aotb_se_gate_f32 / aotb_gate_scale_f32
def _act(x, act):
    if act == 5:
        return MO.h_swish(x)
    return _emu_act(x, act)


def se_gate(x, w1, b1, w2, b2, gate, workspace, stream=None):
    x2 = x.reshape(-1, x.shape[-1])
    gap = (x2.double().sum(0) / x2.shape[0]).float()
    gate.copy_(MO.h_sigmoid(torch.relu(gap @ w1 + b1) @ w2 + b2))
    return gate


def gate_scale(x, gate, out, act=0, stream=None):
    out.copy_(_act(gate * x, act))
    return out


_emu_act = None


def _install(monkeypatch, traced=False):
    global _emu_act
    import emu_ops
    from aot_benchmark_b200 import engine, ops
    RH._install(monkeypatch)
    if _emu_act is None:
        _emu_act = emu_ops._act
    monkeypatch.setattr(emu_ops, "_act", _act)                 # emu_ops knows activations 0-4
    for f in (se_gate, gate_scale):
        monkeypatch.setattr(ops, f.__name__, f)
    if traced:
        for name in list(emu_ops.EMULATED) + ["splat_workspace", "splat_attention", "splat_combine", "avgpool", "se_gate",
                                              "gate_scale"]:
            monkeypatch.setattr(ops, name, GS._traced(name, getattr(ops, name)))
        monkeypatch.setattr(engine, "GraphCache", GS.TracingGraphCache)
        GS.TracingGraphCache.replays = 0


def _model(case, sd=None):
    from aot_benchmark_b200 import build_vos_model
    cfg = MO.engine_config(case, "t")
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    if sd is not None:
        model.load_state_dict(sd, strict=True)
    return cfg, model


def _engine(case, sd, gap):
    from aot_benchmark_b200 import build_engine
    cfg, model = _model(case, sd)
    return build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                        short_term_mem_skip=1).eval()


# ------------------------------------------------------------------ tests
@pytest.mark.parametrize("case", [MBV3, RS50])
def test_state_dict_contract_against_reference(case):
    from oracle.gen_contract import state_dict_digest
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_contract_mbv3_rs50.json")
    want = json.load(open(path))["models"][case]
    cfg, model = _model(case)
    sd = model.state_dict()
    assert len(sd) == {MBV3: 393, RS50: 460}[case]
    assert sum(k.startswith("encoder.") for k in sd) == {MBV3: 262, RS50: 329}[case]
    assert (len(sd), state_dict_digest(sd)) == (want["state_dict_keys"], want["state_dict_sha256"])
    for k, v in cfg.__dict__.items():
        if k not in ("EXP_NAME", "MODEL_NAME"):
            assert json.loads(json.dumps(v, default=repr)) == want["config"][k], k
    if case == MBV3:
        assert sd["encoder.features.15.conv.5.fc.0.weight"].shape == (240, 960)
        assert sd["encoder.features.4.conv.3.weight"].shape == (72, 1, 5, 5)
        assert sd["encoder.conv.0.weight"].shape == (960, 160, 1, 1)
    else:
        assert sd["encoder.conv1.6.weight"].shape == (64, 32, 3, 3)
        assert sd["encoder.layer1.0.conv1.weight"].shape == (64, 64, 1, 1)


@pytest.mark.parametrize("encoder,dims", [("mobilenetv3", [24, 32, 96, 1280]), ("resnest50", [24, 40, 112, 960]),
                                          ("mobilenetv2", [24, 40, 112, 960])])
def test_wrong_encoder_dim_raises(encoder, dims):
    """A MODEL_ENCODER_DIM that does not list the encoder's channel counts is one clear error at model build time."""
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    cfg = EngineConfig("t", "aotl")
    cfg.MODEL_ENCODER, cfg.MODEL_ENCODER_DIM = encoder, dims
    with pytest.raises(ValueError, match="MODEL_ENCODER_DIM"):
        build_vos_model(cfg.MODEL_VOS, cfg)


def test_product_block_table_matches_the_oracle():
    """model.mobilenetv3_plan (computed like the reference's constructor loop) == the oracle's restated block table."""
    from aot_benchmark_b200.model import mobilenetv3_plan
    plan, last = mobilenetv3_plan(16)
    assert plan == MO.MBV3_BLOCKS and last == 960


def test_resnest_forward_is_resnest101_forward_for_resnest101():
    """The generalised ResNeSt forward the ResNeSt-50 fixtures use computes RS101 bit for bit as resnest_oracle does."""
    sd = RO.build_state_dict("rs101_aotl", seed=1)
    img = torch.randn(1, 3, 67, 91, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        a = MO.resnest_forward(sd, img, MO.RESNEST_LAYERS["resnest101"])
        b = RO.resnest101_forward(sd, img)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def _oracle_clip(g, **variant):
    sd = MO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    assert OW.checksum(sd) == g["weights_checksum"], "seeded weights are not reproducible on this machine"
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    eng = MO.OracleEngine(sd, MO.OracleConfig(g["model"]), long_term_mem_gap=g["gap"], variant=variant)
    forced = [l.float() for l in g["ref_labels"]]
    with torch.no_grad():
        lo, labels = O.run_video(eng, frames, mask, g["objs"], tuple(g["out_size"]), forced_masks=forced)
    n = g["objs"] + 1
    return max((a[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(lo, g["ref_logits_lo"])), labels


@pytest.mark.parametrize("name", list(CLIPS))
def test_oracle_vs_reference_golden(name, golden_dir):
    """Teacher-forced oracle engine against the real reference's clip (pins recorded at generation time: 3.5e-6 for
    MobileNetV3, 2.9e-6 for ResNeSt-50, no label mismatch)."""
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    assert g["model"] == CLIPS[name]
    assert g["oracle_pin_max_dlogit"] < 1e-5 and g["oracle_pin_label_mismatch"] == 0
    dmax, labels = _oracle_clip(g)
    assert dmax < 1e-4, dmax
    mism = sum((a.to(torch.uint8) != b).sum().item() for a, b in zip(labels, g["ref_labels"]))
    assert mism <= 1e-4 * sum(b.numel() for b in g["ref_labels"])


@pytest.mark.parametrize("variant", [dict(se_after_act=True), dict(sigmoid_gate=True), dict(relu_for_hswish=True),
                                     dict(undilated=True)])
def test_mobilenetv3_golden_detects_mistakes(golden_dir, variant):
    """Negative controls: the SE after the activation, the logistic sigmoid for h_sigmoid, ReLU for h_swish in blocks 7-15 and
    dilation 1 in blocks 14-15 each miss the reference by far more than the tolerance the GPU engine is held to."""
    g = torch.load(os.path.join(golden_dir, "video_aotl_mbv3_small.pt"))
    dmax, _ = _oracle_clip(g, **variant)
    assert dmax > 10 * 1e-3, dmax


def test_mobilenetv3_weights_spread_the_se_gates():
    """The calibrated recipe puts the SE gates across (0, 1), not at h_sigmoid(0) = 0.5, and keeps the features O(1)."""
    sd = MO.build_state_dict(MBV3)
    frames, _ = O.synthetic_video(1, 161, 241, 10, seed=1234)
    gates = []
    base = MO.h_sigmoid

    def probe(v):
        if v.dim() == 2:
            gates.append(base(v))
        return base(v)

    MO.h_sigmoid = probe
    try:
        with torch.no_grad():
            xs = MO.mobilenetv3_forward(sd, frames[0])
    finally:
        MO.h_sigmoid = base
    assert len(gates) == 8
    for gt in gates:
        assert gt.std().item() > 0.25 and (gt < 0.1).any() and (gt > 0.9).any()
    for x in xs:
        assert 0.3 < x.std().item() < 3.0


@pytest.mark.parametrize("case,hw", [(MBV3, (97, 131)), (MBV3, (70, 45)), (RS50, (97, 131))])
def test_encoder_orchestration_matches_oracle(monkeypatch, case, hw):
    """plan + engine._Encoder through the contract emulations == the oracle encoder + projector at odd sizes."""
    from aot_benchmark_b200 import engine, plan
    _install(monkeypatch)
    sd = MO.build_state_dict(case, seed=2)
    _, model = _model(case, sd)
    P = plan.Plan(model)
    H, W = hw
    img = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(3))
    enc = engine._Encoder(P, H, W)
    with torch.no_grad():
        got = enc(img, 0)
        want = MO.encode_image(sd, MO.OracleConfig(case), img)
    assert len(got) == 4
    for a, b in zip(got, want):
        assert tuple(a.shape) == tuple(b.shape)
        assert (a - b).abs().max().item() < 2e-4 * max(1.0, b.abs().max().item())


@pytest.mark.parametrize("name", list(CLIPS))
def test_engine_orchestration_vs_reference_golden(monkeypatch, golden_dir, name):
    _install(monkeypatch)
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    sd = MO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    eng = _engine(g["model"], sd, g["gap"])
    with torch.no_grad():
        lo, _ = O.run_video(eng, frames, mask, g["objs"], tuple(g["out_size"]),
                            forced_masks=[l.float() for l in g["ref_labels"]])
    n = g["objs"] + 1
    dmax = max((a[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(lo, g["ref_logits_lo"]))
    assert dmax < 2e-4, f"max |dlogit| vs reference = {dmax}"


@pytest.mark.parametrize("case", [MBV3, RS50])
def test_captured_encoder_body_is_static_across_frames_and_videos(monkeypatch, case):
    """Every launch of the encoder body (SE workspace and gates included) reads and writes the same buffers on every call:
    the captured graph replays fixed addresses."""
    _install(monkeypatch, traced=True)
    eng = _engine(case, MO.build_state_dict(case, seed=4), 2)
    outs = []
    for _ in range(2):
        frames, mask = O.synthetic_video(5, 97, 129, 3, seed=31)
        with torch.no_grad():
            lo, _ = O.run_video(eng, frames, mask, 3, (97, 129))
        outs.append(lo)
    assert GS.TracingGraphCache.replays > 8
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)


def test_full_geometry_fixture_pin(golden_dir):
    """The 481x849 MobileNetV3 golden of the real reference: the oracle pin recorded at generation time and the stored layout
    the GPU test reads."""
    from oracle.fixtures import load_full_labels
    g = torch.load(os.path.join(golden_dir, "full_aotl_mbv3_480p.pt"))
    assert g["model"] == MBV3
    assert g["oracle_pin_max_dlogit"] < 1e-4 and g["oracle_pin_label_mismatch"] <= 1e-5 * g["frames"] * 480 * 854
    assert OW.checksum(MO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])) == g["weights_checksum"]
    labels = load_full_labels(g)
    assert len(labels) == g["frames"] - 1 and tuple(labels[0].shape[-2:]) == tuple(g["out_size"])
    s = g["logit_stride"]
    for t in g["logit_frames"]:
        assert tuple(g["ref_logits_lo"][t].shape) == (1, 11, -(-121 // s), -(-213 // s))
