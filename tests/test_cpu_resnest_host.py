"""CPU: the ResNet-101 / ResNeSt-101 encoder paths (R101-AOTL, RS101-AOTL) without a GPU -- state_dict contract against the
real reference, the oracle against the reference's goldens (with negative controls that show the fixtures see the split-attention
details), and the host orchestration (plan._resnest, engine._Encoder._resnest, the engines) with every C-ABI entry point replaced
by a torch-CPU emulation of its contract.  The emulations of the three split-attention entry points live here and follow the
kernels' index arithmetic (csrc/splat.cu); the kernels themselves are checked on the GPU (tests/test_gpu_resnest.py)."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import aot_oracle as O
from oracle import resnest_oracle as RO
from oracle import weights as OW

MODELS = ["r101_aotl", "rs101_aotl"]
CLIPS = ["r101_aotl_small", "rs101_aotl_small"]


# ------------------------------------------------------------------ contract emulations of csrc/splat.cu
def splat_workspace(C, device):
    return torch.zeros(1, dtype=torch.float64, device=device)


def splat_attention(x, w1, b1, w2, b2, att, workspace, radix=2, stream=None):
    """aotb_splat_attention_f32: gap = mean over pixels of the sum of the radix splits, fc1' + ReLU, fc2, softmax over r."""
    x2 = x.reshape(-1, x.shape[-1])
    C = w1.shape[0]
    gap = sum(x2[:, r * C:(r + 1) * C].double().sum(0) for r in range(radix)) / x2.shape[0]
    h = torch.relu(gap.float() @ w1 + b1)
    logit = (h @ w2 + b2).view(radix, C)
    att.copy_(torch.softmax(logit, dim=0).reshape(-1))
    return att


def _pool_window(o, n, k, s, pad, include_pad):
    lo = o * s - pad
    hi = min(lo + k, n + pad)
    padded = hi - lo
    lo, hi = max(lo, 0), min(hi, n)
    return lo, hi, (padded if include_pad else hi - lo)


def _pool(x, k, s, pad, ceil_mode, include_pad):
    """x [H, W, C] -> [Ho, Wo, C] with the kernels' window / divisor rule (PyTorch's)."""
    from aot_benchmark_b200.ops import pool2d_size
    H, W, C = x.shape
    Ho, Wo = pool2d_size(H, k, s, pad, ceil_mode), pool2d_size(W, k, s, pad, ceil_mode)
    out = torch.empty(Ho, Wo, C, dtype=x.dtype)
    for oy in range(Ho):
        y0, y1, dy = _pool_window(oy, H, k, s, pad, include_pad)
        for ox in range(Wo):
            x0, x1, dx = _pool_window(ox, W, k, s, pad, include_pad)
            out[oy, ox] = x[y0:y1, x0:x1].sum((0, 1)) / (dy * dx)
    return out


def splat_combine(x, att, out, radix=2, pool_stride=0, stream=None):
    C = out.shape[3]
    y = sum(att[r * C:(r + 1) * C] * x[0, :, :, r * C:(r + 1) * C] for r in range(radix))
    out[0].copy_(_pool(y, 3, pool_stride, 1, False, True) if pool_stride else y)
    return out


def avgpool(x, out, k, s, pad=0, ceil_mode=False, count_include_pad=True, stream=None):
    for b in range(x.shape[0]):
        out[b].copy_(_pool(x[b], k, s, pad, ceil_mode, count_include_pad))
    return out


def _install(monkeypatch):
    import emu_ops
    from aot_benchmark_b200 import ops
    emu_ops.install_engine(monkeypatch)
    for f in (splat_workspace, splat_attention, splat_combine, avgpool):
        monkeypatch.setattr(ops, f.__name__, f)


# ------------------------------------------------------------------ tests
def test_pool_emulation_matches_torch():
    """The window / divisor rule the kernels and the emulation share is PyTorch's, ceil-mode overhang included."""
    x = torch.randn(7, 10, 4, generator=torch.Generator().manual_seed(1))
    xt = x.permute(2, 0, 1).unsqueeze(0)
    for k, s, pad, ceil, inc in [(2, 2, 0, True, False), (3, 2, 1, False, True), (3, 2, 1, True, False), (1, 1, 0, True, False),
                                 (3, 3, 1, True, True), (2, 2, 1, True, True)]:
        want = F.avg_pool2d(xt, k, s, pad, ceil_mode=ceil, count_include_pad=inc)[0].permute(1, 2, 0)
        got = _pool(x, k, s, pad, ceil, inc)
        assert got.shape == want.shape and torch.allclose(got, want, atol=1e-6), (k, s, pad, ceil, inc)


@pytest.mark.parametrize("model_name", MODELS)
def test_state_dict_contract_against_reference(model_name):
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    from oracle.gen_contract import state_dict_digest
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_contract_r101.json")
    want = json.load(open(path))["models"][model_name]
    cfg = EngineConfig("x", model_name)
    sd = build_vos_model(cfg.MODEL_VOS, cfg).state_dict()
    assert len(sd) == {"r101_aotl": 601, "rs101_aotl": 851}[model_name]
    assert (len(sd), state_dict_digest(sd)) == (want["state_dict_keys"], want["state_dict_sha256"])
    for k, v in cfg.__dict__.items():
        if k not in ("EXP_NAME", "MODEL_NAME"):
            assert json.loads(json.dumps(v, default=repr)) == want["config"][k], k
    if model_name == "rs101_aotl":
        assert sd["encoder.layer1.0.conv2.conv.weight"].shape == (128, 32, 3, 3)          # radix 2 grouped conv, gw 64
        assert sd["encoder.layer3.22.conv2.fc2.weight"].shape == (512, 128, 1, 1)
        assert sd["encoder.layer2.0.downsample.1.weight"].shape == (512, 256, 1, 1)


def _oracle_clip(g, **resnest_kw):
    sd = RO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    assert OW.checksum(sd) == g["weights_checksum"], "seeded weights are not reproducible on this machine"
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    eng = RO.OracleEngine(sd, RO.OracleConfig(g["model"]), long_term_mem_gap=g["gap"], resnest_kw=resnest_kw)
    forced = [l.float() for l in g["ref_labels"]]
    with torch.no_grad():
        lo, labels = O.run_video(eng, frames, mask, g["objs"], tuple(g["out_size"]), forced_masks=forced)
    n = g["objs"] + 1
    return max((a[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(lo, g["ref_logits_lo"])), labels


@pytest.mark.parametrize("name", CLIPS)
def test_oracle_vs_reference_golden(name, golden_dir):
    """Teacher-forced oracle engine against the real reference's clip (pins recorded at generation time: 2.9e-6 for R101, 3.4e-6
    for RS101, no label mismatch)."""
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    assert g["oracle_pin_max_dlogit"] < 1e-5 and g["oracle_pin_label_mismatch"] == 0
    dmax, labels = _oracle_clip(g)
    assert dmax < 1e-4, dmax
    mism = sum((a.to(torch.uint8) != b).sum().item() for a, b in zip(labels, g["ref_labels"]))
    assert mism <= 1e-4 * sum(b.numel() for b in g["ref_labels"])


@pytest.mark.parametrize("variant", [dict(swap_radix=True), dict(avd_include_pad=False)])
def test_resnest_golden_detects_split_attention_mistakes(golden_dir, variant):
    """Negative controls: exchanging the two radix attention maps, or leaving the padding out of the avd pool's divisor, misses
    the reference by far more than the tolerance the GPU engine is held to."""
    g = torch.load(os.path.join(golden_dir, "video_rs101_aotl_small.pt"))
    dmax, _ = _oracle_clip(g, **variant)
    assert dmax > 10 * 1e-3, dmax


@pytest.mark.parametrize("model_name,hw", [("rs101_aotl", (97, 131)), ("rs101_aotl", (70, 45)), ("r101_aotl", (97, 131))])
def test_encoder_orchestration_matches_oracle(monkeypatch, model_name, hw):
    """plan + engine._Encoder (deep stem, grouped conv on channel slices, split attention, fused avd pool, avg_down) through
    the contract emulations == the oracle encoder + projector at odd sizes."""
    from aot_benchmark_b200 import EngineConfig, build_vos_model, engine, plan
    _install(monkeypatch)
    cfg = EngineConfig("t", model_name)
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    sd = RO.build_state_dict(model_name, seed=2)
    model.load_state_dict(sd)
    P = plan.Plan(model)
    H, W = hw
    img = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(3))
    enc = engine._Encoder(P, H, W)
    with torch.no_grad():
        got = enc(img, 0)
        want = RO.encode_image(sd, RO.OracleConfig(model_name), img)
    assert len(got) == 4
    for a, b in zip(got, want):
        assert tuple(a.shape) == tuple(b.shape)
        assert (a - b).abs().max().item() < 2e-4 * max(1.0, b.abs().max().item())


@pytest.mark.parametrize("name", CLIPS)
def test_engine_orchestration_vs_reference_golden(monkeypatch, golden_dir, name):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    _install(monkeypatch)
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    sd = RO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    cfg = EngineConfig("t", g["model"])
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    model.load_state_dict(sd, strict=True)
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=g["gap"],
                       short_term_mem_skip=1).eval()
    with torch.no_grad():
        lo, _ = O.run_video(eng, frames, mask, g["objs"], tuple(g["out_size"]),
                            forced_masks=[l.float() for l in g["ref_labels"]])
    n = g["objs"] + 1
    dmax = max((a[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(lo, g["ref_logits_lo"]))
    assert dmax < 2e-4, f"max |dlogit| vs reference = {dmax}"
    e0 = eng.aot_engines[0]
    assert e0.bank_len == e0.enc_hw * (1 + (g["frames"] - 1) // g["gap"])


def test_full_geometry_fixture_pin(golden_dir):
    """The 481x849 RS101-AOTL golden of the real reference: the oracle pin recorded at generation time (whole clip,
    teacher-forced; 4.5e-6, one tie pixel) and the stored layout the GPU test reads."""
    from oracle.fixtures import load_full_labels
    g = torch.load(os.path.join(golden_dir, "full_rs101_aotl_480p.pt"))
    assert g["oracle_pin_max_dlogit"] < 1e-4 and g["oracle_pin_label_mismatch"] <= 1e-5 * g["frames"] * 480 * 854
    assert OW.checksum(RO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])) == g["weights_checksum"]
    labels = load_full_labels(g)
    assert len(labels) == g["frames"] - 1 and tuple(labels[0].shape[-2:]) == tuple(g["out_size"])
    s = g["logit_stride"]
    for t in g["logit_frames"]:
        assert tuple(g["ref_logits_lo"][t].shape) == (1, 11, -(-121 // s), -(-213 // s))
