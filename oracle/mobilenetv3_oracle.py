"""CPU oracle of the MobileNetV3-Large and ResNeSt-50 encoders (AOTL with mobilenetv3, R50-AOTL with resnest50) and their
seeded test weights.

TEST INFRASTRUCTURE ONLY, like ``aot_oracle.py`` and ``resnest_oracle.py``, which it extends without changing: functional
torch-CPU restatements of networks/encoders/mobilenetv3.py (MobileNetV3Large as encoders/__init__.py:17-18 builds it) and of
networks/encoders/resnest/ for any layer counts and stem width (resnest50 and resnest101 as encoders/__init__.py:24-31 build
them), a config mirror, an ``OracleEngine`` that encodes frames with them, and the calibrated weight recipe of
``weights.py`` for the two encoders.  ``oracle/gen_golden_mbv3.py`` pins it to the real reference.

Neither encoder has a model config of its own in the reference: a user selects one by setting ``cfg.MODEL_ENCODER`` and
``cfg.MODEL_ENCODER_DIM`` on a model config.  The case names of ``CASES`` are this module's own labels for those settings.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

from oracle import aot_oracle as O
from oracle import resnest_oracle as RO

Tensor = torch.Tensor

# case: (model config, MODEL_ENCODER, MODEL_ENCODER_DIM)
CASES = {
    "AOTL with mobilenetv3": ("aotl", "mobilenetv3", [24, 40, 112, 960]),
    "R50-AOTL with resnest50": ("r50_aotl", "resnest50", [256, 512, 1024, 1024]),
}
RESNEST_LAYERS = {"resnest50": (3, 4, 6), "resnest101": (3, 4, 23)}


class OracleConfig(RO.OracleConfig):
    _TABLE = {
        **RO.OracleConfig._TABLE,
        **{case: ("aot", enc, dims, 3, True, 5) for case, (_, enc, dims) in CASES.items()},   # aotl / r50_aotl otherwise
    }


def engine_config(case: str, exp_name: str = "golden"):
    """The product's EngineConfig of the case: its model config with MODEL_ENCODER / MODEL_ENCODER_DIM set."""
    from aot_benchmark_b200 import EngineConfig
    model, enc, dims = CASES[case]
    cfg = EngineConfig(exp_name, model)
    cfg.MODEL_ENCODER = enc
    cfg.MODEL_ENCODER_DIM = list(dims)
    return cfg


# ------------------------------------------------------------------ MobileNetV3-Large
# InvertedResidual blocks features.1 ... features.15 of MobileNetV3Large(output_stride=16) (mobilenetv3.py:152-192 with
# width_mult 1 and _make_divisible(., 8)): (in, hidden, out, kernel, stride, dilation, SE, h_swish).  With output stride 16 the
# stride-2 block 13 runs at stride 1 and blocks 14-15 at dilation 2 (:180-186).
MBV3_BLOCKS = [
    (16, 16, 16, 3, 1, 1, False, False),
    (16, 64, 24, 3, 2, 1, False, False), (24, 72, 24, 3, 1, 1, False, False),
    (24, 72, 40, 5, 2, 1, True, False), (40, 120, 40, 5, 1, 1, True, False), (40, 120, 40, 5, 1, 1, True, False),
    (40, 240, 80, 3, 2, 1, False, True), (80, 200, 80, 3, 1, 1, False, True), (80, 184, 80, 3, 1, 1, False, True),
    (80, 184, 80, 3, 1, 1, False, True),
    (80, 480, 112, 3, 1, 1, True, True), (112, 672, 112, 3, 1, 1, True, True),
    (112, 672, 160, 5, 1, 1, True, True), (160, 960, 160, 5, 1, 2, True, True), (160, 960, 160, 5, 1, 2, True, True),
]


def h_sigmoid(v: Tensor) -> Tensor:
    return F.relu6(v + 3) / 6                                   # mobilenetv3.py:33-39


def h_swish(v: Tensor) -> Tensor:
    return v * h_sigmoid(v)                                     # mobilenetv3.py:42-48


def mobilenetv3_forward(W: Dict[str, Tensor], img: Tensor, p: str = "encoder.", se_after_act: bool = False,
                        sigmoid_gate: bool = False, relu_for_hswish: bool = False,
                        undilated: bool = False) -> List[Tensor]:
    """MobileNetV3Large.forward (mobilenetv3.py:142-215) with output_stride 16 and FrozenBN: stem, 15 InvertedResidual blocks
    (:78-139), taps after blocks 3, 6, 12 and 15, the last one through conv_1x1_bn(160, 960) + h_swish.

    The keyword arguments select deliberately wrong variants that the tests use as negative controls: the SE after the
    activation, the logistic sigmoid in place of h_sigmoid in the SE gate, ReLU in place of h_swish in blocks 7-15, and
    dilation 1 in blocks 14-15."""
    hs = h_swish

    def bn(x, name):
        return O.frozen_bn(x, W, name)

    def se(x, q):
        y = F.adaptive_avg_pool2d(x, 1).flatten(1)                      # SELayer :61-65
        y = F.relu(F.linear(y, W[q + "fc.0.weight"], W[q + "fc.0.bias"]))
        y = F.linear(y, W[q + "fc.2.weight"], W[q + "fc.2.bias"])
        y = torch.sigmoid(y) if sigmoid_gate else h_sigmoid(y)
        return x * y.view(y.shape[0], y.shape[1], 1, 1)

    x = hs(bn(F.conv2d(img, W[p + "features.0.0.weight"], None, 2, 1), p + "features.0.1"))
    feats = []
    for idx, (inp, hid, oup, k, s, dil, use_se, use_hs) in enumerate(MBV3_BLOCKS, start=1):
        q = f"{p}features.{idx}.conv."
        act = (F.relu if relu_for_hswish else h_swish) if use_hs else F.relu
        if undilated and dil > 1:
            dil = 1
        pad = (k - 1) // 2 * dil
        if inp == hid:                                                  # :94-111
            assert not use_se
            y = act(bn(F.conv2d(x, W[q + "0.weight"], None, s, pad, dil, hid), q + "1"))
            y = bn(F.conv2d(y, W[q + "4.weight"]), q + "5")
        else:                                                           # :113-133
            y = act(bn(F.conv2d(x, W[q + "0.weight"]), q + "1"))
            y = bn(F.conv2d(y, W[q + "3.weight"], None, s, pad, dil, hid), q + "4")
            if use_se and not se_after_act:
                y = se(y, q + "5.")
            y = act(y)
            if use_se and se_after_act:
                y = se(y, q + "5.")
            y = bn(F.conv2d(y, W[q + "7.weight"]), q + "8")
        x = x + y if (s == 1 and inp == oup) else y
        if idx in (3, 6, 12):
            feats.append(x)
    feats.append(hs(bn(F.conv2d(x, W[p + "conv.0.weight"]), p + "conv.1")))
    return feats


# ------------------------------------------------------------------ ResNeSt of any depth
def resnest_forward(W: Dict[str, Tensor], img: Tensor, layers: Sequence[int], p: str = "encoder.") -> List[Tensor]:
    """resnest_oracle.resnest101_forward with `layers` bottlenecks in layer1..3 (resnest50: [3, 4, 6]); the stem width follows
    from the weights.  For resnest101 it computes what resnest101_forward computes, operation for operation."""
    x = F.relu(O.frozen_bn(F.conv2d(img, W[p + "conv1.0.weight"], None, 2, 1), W, p + "conv1.1"))
    x = F.relu(O.frozen_bn(F.conv2d(x, W[p + "conv1.3.weight"], None, 1, 1), W, p + "conv1.4"))
    x = F.relu(O.frozen_bn(F.conv2d(x, W[p + "conv1.6.weight"], None, 1, 1), W, p + "bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    xs = []
    for li, (nblk, stride) in enumerate(zip(layers, (1, 2, 2)), start=1):
        for bi in range(nblk):
            q = f"{p}layer{li}.{bi}."
            s = stride if bi == 0 else 1
            out = F.relu(O.frozen_bn(F.conv2d(x, W[q + "conv1.weight"]), W, q + "bn1"))
            out = RO.splat_conv(W, q + "conv2.", out)
            if s > 1:
                out = F.avg_pool2d(out, 3, s, 1, count_include_pad=True)
            out = O.frozen_bn(F.conv2d(out, W[q + "conv3.weight"]), W, q + "bn3")
            if (q + "downsample.1.weight") in W:
                r = F.avg_pool2d(x, s, s, ceil_mode=True, count_include_pad=False) if s > 1 else x
                res = O.frozen_bn(F.conv2d(r, W[q + "downsample.1.weight"]), W, q + "downsample.2")
            else:
                res = x
            x = F.relu(out + res)
        xs.append(x)
    xs.append(x)
    return xs


def encode_image(W: Dict[str, Tensor], cfg, img: Tensor, **variant) -> List[Tensor]:
    """aot.py:81-84 for the two encoders (any other encoder goes to resnest_oracle.encode_image).  `variant` selects the
    negative-control variants of mobilenetv3_forward."""
    if cfg.MODEL_ENCODER == "mobilenetv3":
        xs = mobilenetv3_forward(W, img, **variant)
    elif cfg.MODEL_ENCODER == "resnest50":
        xs = resnest_forward(W, img, RESNEST_LAYERS["resnest50"])
    else:
        return RO.encode_image(W, cfg, img)
    xs[-1] = F.conv2d(xs[-1], W["encoder_projector.weight"], W["encoder_projector.bias"])
    return xs


class OracleEngine(RO.OracleEngine):
    """aot_oracle.OracleEngine whose frames are encoded by `encode_image` above (with `variant`)."""

    def __init__(self, weights, cfg, *args, variant=None, **kwargs):
        super().__init__(weights, cfg, *args, **kwargs)
        self._variant = dict(variant or {})

    def _encoding(self, fn, *args, **kwargs):
        base = O.encode_image
        O.encode_image = lambda W, cfg, img: encode_image(W, cfg, img, **self._variant)
        try:
            return fn(*args, **kwargs)
        finally:
            O.encode_image = base


# ------------------------------------------------------------------ seeded weights (the recipe of weights.build_state_dict)
# projector-output std of the calibrated encoder on the synthetic clips (measured once through this oracle and frozen)
_PROJ_STD = {"mobilenetv3": 1.2, "resnest50": 0.95}
# MobileNetV3: SE fc2 gain per block (measured once and frozen) that spreads the SE logits to std ~2.5, so the gates cover
# (0, 1) instead of sitting at h_sigmoid(0) = 0.5
_SE_GAIN = {4: 1.4, 5: 1.5, 6: 2.6, 11: 1.1, 12: 2.4, 13: 1.7, 14: 3.9, 15: 3.8}
# MobileNetV3: the pw-linear convs feed the residual stream with no activation after them; fan-in init alone lets the stream
# grow to std ~60 by block 12, damping them keeps activations O(1) through the 15 blocks
_PW_LINEAR_DAMP = 0.7


def build_state_dict(case: str, seed: int = 0, flavour: str = "calibrated", q_scale: float = 4.0,
                     id_scale: float = 100.0) -> Dict[str, Tensor]:
    """weights.build_state_dict for the two cases: the product model's seeded init, then the same calibration steps in the
    same order (randomised FrozenBN statistics, projector rescaled to ~unit-std tokens, ID bank x100, linear_Q x4).
    MobileNetV3 additionally gets fan-in scaled convs (the reference's fan-out init makes every depthwise conv shrink its input
    by ~sqrt(C)) and SE weights whose gates spread over (0, 1).  Element-wise RNG and constants only: bit-identical on every
    machine (weights.checksum)."""
    from aot_benchmark_b200 import build_vos_model
    cfg = engine_config(case)
    torch.manual_seed(seed)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    if flavour == "raw":
        return sd
    g = torch.Generator().manual_seed(seed + 7919)
    for k in list(sd.keys()):
        if k.endswith("running_var"):
            n = sd[k].numel()
            sd[k] = 0.7 + 0.6 * torch.rand(n, generator=g)
            base = k[: -len("running_var")]
            sd[base + "running_mean"] = 0.1 * torch.randn(n, generator=g)
            sd[base + "weight"] = 0.9 + 0.2 * torch.rand(n, generator=g)
            sd[base + "bias"] = 0.05 * torch.randn(n, generator=g)
    if cfg.MODEL_ENCODER == "mobilenetv3":
        _calibrate_mobilenetv3(sd, g)
    s = 1.0 / _PROJ_STD[cfg.MODEL_ENCODER]
    sd["encoder_projector.weight"] = sd["encoder_projector.weight"] * s
    sd["encoder_projector.bias"] = sd["encoder_projector.bias"] * s
    sd["patch_wise_id_bank.weight"] = sd["patch_wise_id_bank.weight"] * id_scale
    for i in range(cfg.MODEL_LSTT_NUM):
        p = f"LSTT.layers.{i}."
        sd[p + "linear_Q.weight"] = sd[p + "linear_Q.weight"] * q_scale
        sd[p + "linear_Q.bias"] = sd[p + "linear_Q.bias"] * q_scale
    return sd


def _calibrate_mobilenetv3(sd: Dict[str, Tensor], g: torch.Generator) -> None:
    import math
    for k in sorted(sd.keys()):
        if not k.startswith("encoder.") or not k.endswith(".weight") or sd[k].dim() != 4:
            continue
        co, ci, kh, kw = sd[k].shape
        sd[k] = sd[k] * math.sqrt(co / ci)                       # fan-out init -> fan-in init: std sqrt(2 / (ci kh kw))
        if k.endswith(("conv.4.weight", "conv.7.weight")):       # pw-linear (no activation after it): damp the residual stream
            sd[k] = sd[k] * _PW_LINEAR_DAMP
    for k in sorted(sd.keys()):
        if k.startswith("encoder.") and k.endswith(".fc.0.weight"):
            q = k[: -len("0.weight")]
            inter, c = sd[k].shape
            sd[q + "0.weight"] = torch.randn(inter, c, generator=g) * math.sqrt(2.0 / c)
            sd[q + "0.bias"] = 0.1 * torch.randn(inter, generator=g)
            blk = int(k.split(".")[2])                           # encoder.features.<blk>.conv.5.fc.0.weight
            sd[q + "2.weight"] = torch.randn(c, inter, generator=g) * (_SE_GAIN[blk] / math.sqrt(inter))
            sd[q + "2.bias"] = 0.5 * torch.randn(c, generator=g)
