"""CPU oracle of the ResNet-101 and ResNeSt-101 encoders (R101-AOTL, RS101-AOTL) and their seeded test weights.

TEST INFRASTRUCTURE ONLY, like ``aot_oracle.py``, which it extends without changing: a functional torch-CPU restatement of
networks/encoders/resnet.py (ResNet101) and networks/encoders/resnest/ (resnest101 as encoders/__init__.py:28-31 builds it),
a config mirror with the two model configs, an ``OracleEngine`` that encodes frames with them, and the calibrated weight
recipe of ``weights.py`` for the two encoders.  ``oracle/gen_golden_resnest.py`` pins it to the real reference.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

from oracle import aot_oracle as O
from oracle import weights as OW

Tensor = torch.Tensor


class OracleConfig(O.OracleConfig):
    _TABLE = {
        **O.OracleConfig._TABLE,
        "r101_aotl": ("aot", "resnet101", [256, 512, 1024, 1024], 3, True, 5),    # configs/models/r101_aotl.py:7-16
        "rs101_aotl": ("aot", "resnest101", [256, 512, 1024, 1024], 3, True, 5),  # configs/models/rs101_aotl.py:7-16
    }


MODELS = ("r101_aotl", "rs101_aotl")


def resnet_forward(W: Dict[str, Tensor], img: Tensor, layers: Sequence[int], p: str = "encoder.") -> List[Tensor]:
    """resnet.py:140-157 (+ Bottleneck :34-54) with `layers` bottlenecks in layer1..3 (ResNet101: [3,4,23], :190-201);
    strides [1,2,2], layer4 dropped."""
    x = F.conv2d(img, W[p + "conv1.weight"], None, 2, 3)
    x = F.relu(O.frozen_bn(x, W, p + "bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    xs = []
    for li, (nblk, stride) in enumerate(zip(layers, (1, 2, 2)), start=1):
        for bi in range(nblk):
            q = f"{p}layer{li}.{bi}."
            s = stride if bi == 0 else 1
            out = F.relu(O.frozen_bn(F.conv2d(x, W[q + "conv1.weight"]), W, q + "bn1"))
            out = F.relu(O.frozen_bn(F.conv2d(out, W[q + "conv2.weight"], None, s, 1), W, q + "bn2"))
            out = O.frozen_bn(F.conv2d(out, W[q + "conv3.weight"]), W, q + "bn3")
            if (q + "downsample.0.weight") in W:
                res = O.frozen_bn(F.conv2d(x, W[q + "downsample.0.weight"], None, s), W, q + "downsample.1")
            else:
                res = x
            x = F.relu(out + res)
        xs.append(x)
    xs.append(x)  # 16x twice (resnet.py:153-155)
    return xs


def splat_conv(W: Dict[str, Tensor], q: str, x: Tensor, swap_radix: bool = False) -> Tensor:
    """SplAtConv2d.forward resnest/splat.py:80-115 with radix 2, cardinality 1, stride 1 (avd pools afterwards), FrozenBN.
    `swap_radix` exchanges the two attention maps (a deliberately wrong variant the tests use as a negative control)."""
    x = F.relu(O.frozen_bn(F.conv2d(x, W[q + "conv.weight"], None, 1, 1, 1, 2), W, q + "bn0"))
    gw = x.shape[1] // 2
    x0, x1 = x[:, :gw], x[:, gw:]
    gap = F.adaptive_avg_pool2d(x0 + x1, 1)
    gap = F.relu(O.frozen_bn(F.conv2d(gap, W[q + "fc1.weight"], W[q + "fc1.bias"]), W, q + "bn1"))
    att = F.conv2d(gap, W[q + "fc2.weight"], W[q + "fc2.bias"])
    att = torch.softmax(att.view(x.shape[0], 1, 2, gw).transpose(1, 2), dim=1).reshape(x.shape[0], -1, 1, 1)   # rSoftMax :118-132
    a0, a1 = att[:, :gw], att[:, gw:]
    if swap_radix:
        a0, a1 = a1, a0
    return a0 * x0 + a1 * x1


def resnest101_forward(W: Dict[str, Tensor], img: Tensor, p: str = "encoder.", swap_radix: bool = False,
                       avd_include_pad: bool = True) -> List[Tensor]:
    """resnest/resnet.py:418-435 for resnest101(dilation=2) (resnest.py:51-68, encoders/__init__.py:28-31): deep stem,
    layers [3,4,23] of Bottleneck :37-166 with SplAtConv2d, avd pool after conv2 in the first block of layer2 / layer3,
    avg_down downsample [AvgPool2d(s, s, ceil_mode, count_include_pad=False), conv1x1, BN] (:327-357), layer4 dropped.
    `avd_include_pad=False` leaves the padding out of the avd pool's divisor (a negative control for the tests; with padding 0
    the avg_down pool's count_include_pad has no effect)."""
    x = F.relu(O.frozen_bn(F.conv2d(img, W[p + "conv1.0.weight"], None, 2, 1), W, p + "conv1.1"))
    x = F.relu(O.frozen_bn(F.conv2d(x, W[p + "conv1.3.weight"], None, 1, 1), W, p + "conv1.4"))
    x = F.relu(O.frozen_bn(F.conv2d(x, W[p + "conv1.6.weight"], None, 1, 1), W, p + "bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    xs = []
    for li, (nblk, stride) in enumerate(zip((3, 4, 23), (1, 2, 2)), start=1):
        for bi in range(nblk):
            q = f"{p}layer{li}.{bi}."
            s = stride if bi == 0 else 1
            out = F.relu(O.frozen_bn(F.conv2d(x, W[q + "conv1.weight"]), W, q + "bn1"))
            out = splat_conv(W, q + "conv2.", out, swap_radix)
            if s > 1:                                             # avd: AvgPool2d(3, s, padding=1), padding counted
                out = F.avg_pool2d(out, 3, s, 1, count_include_pad=avd_include_pad)
            out = O.frozen_bn(F.conv2d(out, W[q + "conv3.weight"]), W, q + "bn3")
            if (q + "downsample.1.weight") in W:
                r = F.avg_pool2d(x, s, s, ceil_mode=True, count_include_pad=False) if s > 1 else x
                res = O.frozen_bn(F.conv2d(r, W[q + "downsample.1.weight"]), W, q + "downsample.2")
            else:
                res = x
            x = F.relu(out + res)
        xs.append(x)
    xs.append(x)  # 16x twice (resnet.py:431-433)
    return xs


def encode_image(W: Dict[str, Tensor], cfg, img: Tensor, **resnest_kw) -> List[Tensor]:
    """aot.py:81-84 for the two encoders (any other encoder goes to aot_oracle.encode_image).  `resnest_kw` selects the
    negative-control variants of resnest101_forward."""
    if cfg.MODEL_ENCODER == "resnet101":
        xs = resnet_forward(W, img, (3, 4, 23))
    elif cfg.MODEL_ENCODER == "resnest101":
        xs = resnest101_forward(W, img, **resnest_kw)
    else:
        return O.encode_image(W, cfg, img)
    xs[-1] = F.conv2d(xs[-1], W["encoder_projector.weight"], W["encoder_projector.bias"])
    return xs


class OracleEngine(O.OracleEngine):
    """aot_oracle.OracleEngine whose frames are encoded by `encode_image` above (with `resnest_kw`).  The base engine calls
    its module's encode_image; the two protocol calls that encode a frame point that name here while they run."""

    def __init__(self, weights, cfg, *args, resnest_kw=None, **kwargs):
        super().__init__(weights, cfg, *args, **kwargs)
        self._resnest_kw = dict(resnest_kw or {})

    def _encoding(self, fn, *args, **kwargs):
        base = O.encode_image
        O.encode_image = lambda W, cfg, img: encode_image(W, cfg, img, **self._resnest_kw)
        try:
            return fn(*args, **kwargs)
        finally:
            O.encode_image = base

    def add_reference_frame(self, *args, **kwargs):
        return self._encoding(super().add_reference_frame, *args, **kwargs)

    def match_propogate_one_frame(self, img):
        return self._encoding(super().match_propogate_one_frame, img)


# ------------------------------------------------------------------ seeded weights (the recipe of weights.build_state_dict)
# projector-output std of the calibrated encoder (measured once through this oracle and frozen; raw init is far from the
# calibrated statistics for these deep encoders)
_PROJ_STD = {"resnet101": 0.48, "resnest101": 8.2}
# resnet101: 23 bottlenecks in layer3 with identity-like FrozenBN grow the residual stream to ~1e5 (beyond the fp16 range of the
# tensor-core operand split); damping every bn3 keeps activations O(1), as trained weights have them
_BN3_DAMP = {"resnet101": 0.2}


def build_state_dict(model_name: str, seed: int = 0, flavour: str = "calibrated", q_scale: float = 4.0,
                     id_scale: float = 100.0) -> Dict[str, Tensor]:
    """weights.build_state_dict for r101_aotl / rs101_aotl: the same seeded init and the same calibration steps in the same
    order (randomised FrozenBN statistics, projector rescaled to ~unit-std tokens, ID bank x100, linear_Q x4), plus the bn3
    damping of ResNet-101.  Element-wise RNG and constants only: bit-identical on every machine (weights.checksum)."""
    from aot_benchmark_b200 import EngineConfig
    cfg = EngineConfig("golden", model_name)
    if cfg.MODEL_ENCODER not in _PROJ_STD:
        raise ValueError(f"{model_name}: use oracle.weights.build_state_dict")
    sd = OW.build_state_dict(model_name, seed=seed, flavour="raw")
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
    damp = _BN3_DAMP.get(cfg.MODEL_ENCODER)
    if damp is not None:
        for k in list(sd.keys()):
            if k.startswith("encoder.") and (k.endswith(".bn3.weight") or k.endswith(".bn3.bias")):
                sd[k] = sd[k] * damp
    s = 1.0 / _PROJ_STD[cfg.MODEL_ENCODER]
    sd["encoder_projector.weight"] = sd["encoder_projector.weight"] * s
    sd["encoder_projector.bias"] = sd["encoder_projector.bias"] * s
    sd["patch_wise_id_bank.weight"] = sd["patch_wise_id_bank.weight"] * id_scale
    for i in range(cfg.MODEL_LSTT_NUM):
        p = f"LSTT.layers.{i}."
        sd[p + "linear_Q.weight"] = sd[p + "linear_Q.weight"] * q_scale
        sd[p + "linear_Q.bias"] = sd[p + "linear_Q.bias"] * q_scale
    return sd
