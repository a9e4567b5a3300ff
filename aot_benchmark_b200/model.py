"""Parameter trees of AOT / DeAOT with the reference's ``state_dict`` contract.

``utils/checkpoint.py:94-121`` (``load_network``) matches checkpoints to the model *by key*,
so a drop-in model must expose the reference's parameter names and shapes (SURVEY Appendix F).
The modules below are parameter containers only: no ``forward`` is defined on the layer
modules -- every per-frame FLOP is executed by the sm_90a kernels in ``csrc/`` through the
engine (``engine.py``), which reads packed copies of these parameters (``plan.py``).

Initialisation follows the same distributions as the reference (aot.py:110-115,
transformer.py:369-372, fpn.py:60-63, resnet.py:159-167, mobilenetv2.py:226-239) but not its
RNG consumption order; parity tests always copy one ``state_dict`` into both sides.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn


class ParamNode(nn.Module):
    """A parameter/buffer container with attribute-style children (never called)."""

    def forward(self, *a, **k):  # pragma: no cover - guard against accidental eager use
        raise RuntimeError("aot_benchmark_b200 parameter containers are not executable: the "
                           "hot path runs through the CUDA engine (engine.py), not nn.Module.forward")


class FrozenBN(ParamNode):
    # normalization.py:11-18 (all four are buffers)
    def __init__(self, n, eps=1e-5):
        super().__init__()
        self.register_buffer("weight", torch.ones(n))
        self.register_buffer("bias", torch.zeros(n))
        self.register_buffer("running_mean", torch.zeros(n))
        self.register_buffer("running_var", torch.ones(n) - eps)
        self.epsilon = eps


class Conv(ParamNode):
    def __init__(self, cin, cout, k, bias=True, groups=1):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin // groups, k, k))
        if bias:
            self.bias = nn.Parameter(torch.zeros(cout))
            bound = 1.0 / math.sqrt(cin // groups * k * k)
            nn.init.uniform_(self.bias, -bound, bound)
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))


class Linear(ParamNode):
    def __init__(self, cin, cout):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin))
        self.bias = nn.Parameter(torch.empty(cout))
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        bound = 1.0 / math.sqrt(cin)
        nn.init.uniform_(self.bias, -bound, bound)


class Norm(ParamNode):
    def __init__(self, n):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(n))
        self.bias = nn.Parameter(torch.zeros(n))


def _seq(mods):
    s = nn.Sequential()
    for i, m in enumerate(mods):
        s.add_module(str(i), m)
    return s


# ---------------------------------------------------------------- encoders
RESNET_LAYERS = {"resnet50": (3, 4, 6), "resnet101": (3, 4, 23)}


def _resnet(layers):
    # resnet.py:57-138: Bottleneck, stride on conv2, layer4 dropped; ResNet50 [3,4,6], ResNet101 [3,4,23] (:178-201)
    enc = ParamNode()
    enc.conv1 = Conv(3, 64, 7, bias=False)
    enc.bn1 = FrozenBN(64)
    inpl = 64
    for li, (planes, nblk, stride) in enumerate(zip((64, 128, 256), layers, (1, 2, 2)), start=1):
        blocks = []
        for bi in range(nblk):
            b = ParamNode()
            b.conv1 = Conv(inpl, planes, 1, bias=False)
            b.bn1 = FrozenBN(planes)
            b.conv2 = Conv(planes, planes, 3, bias=False)
            b.bn2 = FrozenBN(planes)
            b.conv3 = Conv(planes, planes * 4, 1, bias=False)
            b.bn3 = FrozenBN(planes * 4)
            if bi == 0 and (stride != 1 or inpl != planes * 4):
                b.downsample = _seq([Conv(inpl, planes * 4, 1, bias=False), FrozenBN(planes * 4)])
            inpl = planes * 4
            blocks.append(b)
        setattr(enc, f"layer{li}", _seq(blocks))
    for m in enc.modules():
        if isinstance(m, Conv):
            n = m.weight.shape[2] * m.weight.shape[3] * m.weight.shape[0]
            nn.init.normal_(m.weight, 0, math.sqrt(2.0 / n))  # resnet.py:160-163
    return enc


# resnest/resnest.py:32-68 with encoders/__init__.py:24-31 (dilation=2): radix 2, cardinality 1, bottleneck_width 64, deep
# stem, avg_down, avd (not first); strides 1, 2, 2 and no dilated conv; layer4 is never built.  name: (layers, stem_width)
RESNEST = {"resnest50": ((3, 4, 6), 32), "resnest101": ((3, 4, 23), 64)}


def _resnest(layers, sw):
    """Parameter tree of resnest50 / resnest101 with the reference's names (resnest/resnet.py:37-166, 191-357,
    splat.py:15-78): conv1.{0,1,3,4,6} deep stem (3 -> sw -> sw -> 2 sw) + bn1, layer<i>.<j>.{conv1, bn1, conv2.{conv, bn0,
    fc1, bn1, fc2}, conv3, bn3, downsample.{1,2}} (downsample.0 is the parameter-free AvgPool2d)."""
    enc = ParamNode()
    enc.conv1 = _seq([Conv(3, sw, 3, bias=False), FrozenBN(sw), ParamNode(), Conv(sw, sw, 3, bias=False), FrozenBN(sw),
                      ParamNode(), Conv(sw, 2 * sw, 3, bias=False)])
    enc.bn1 = FrozenBN(2 * sw)
    inpl = 2 * sw
    for li, (planes, nblk) in enumerate(zip((64, 128, 256), layers), start=1):
        gw = planes                                   # group width: planes * bottleneck_width / 64 * cardinality
        blocks = []
        for bi in range(nblk):
            b = ParamNode()
            b.conv1 = Conv(inpl, gw, 1, bias=False)
            b.bn1 = FrozenBN(gw)
            sp = ParamNode()                          # SplAtConv2d, radix 2: inter_channels = max(gw * 2 // 4, 32)
            inter = max(gw * 2 // 4, 32)
            sp.conv = Conv(gw, 2 * gw, 3, bias=False, groups=2)
            sp.bn0 = FrozenBN(2 * gw)
            sp.fc1 = Conv(gw, inter, 1)
            sp.bn1 = FrozenBN(inter)
            sp.fc2 = Conv(inter, 2 * gw, 1)
            b.conv2 = sp
            b.conv3 = Conv(gw, planes * 4, 1, bias=False)
            b.bn3 = FrozenBN(planes * 4)
            if bi == 0:                               # stride 2 (layers 2, 3) or inplanes != planes * 4 (layer 1)
                b.downsample = _seq([ParamNode(), Conv(inpl, planes * 4, 1, bias=False), FrozenBN(planes * 4)])
            inpl = planes * 4
            blocks.append(b)
        setattr(enc, f"layer{li}", _seq(blocks))
    for m in enc.modules():
        if isinstance(m, Conv):
            n = m.weight.shape[2] * m.weight.shape[3] * m.weight.shape[0]
            nn.init.normal_(m.weight, 0, math.sqrt(2.0 / n))  # resnest/resnet.py:308-311
    return enc


_MBV2_SETTING = [[1, 16, 1, 1], [6, 24, 2, 2], [6, 32, 3, 2], [6, 64, 4, 2], [6, 96, 3, 1], [6, 160, 3, 2], [6, 320, 1, 1]]


def mobilenetv2_plan(output_stride=16):
    """(inp, oup, stride, dilation, expand) per InvertedResidual, mobilenetv2.py:168-205."""
    plan, inp, cur, rate = [], 32, 2, 1
    for t, c, n, s in _MBV2_SETTING:
        if cur == output_stride:
            stride, dil = 1, rate
            rate *= s
        else:
            stride, dil = s, 1
            cur *= s
        for i in range(n):
            plan.append((inp, c, stride if i == 0 else 1, dil if i == 0 else rate, t))
            inp = c
    return plan


def _mobilenetv2():
    enc = ParamNode()

    def cbr(cin, cout, k, groups=1):
        return _seq([Conv(cin, cout, k, bias=False, groups=groups), FrozenBN(cout), ParamNode()])

    feats = [cbr(3, 32, 3)]
    for inp, oup, stride, dil, t in mobilenetv2_plan(16):
        hidden = int(round(inp * t))
        layers = []
        if t != 1:
            layers.append(cbr(inp, hidden, 1))
        layers += [cbr(hidden, hidden, 3, groups=hidden), Conv(hidden, oup, 1, bias=False), FrozenBN(oup)]
        blk = ParamNode()
        blk.conv = _seq(layers)
        feats.append(blk)
    feats.append(cbr(320, 1280, 1))
    enc.features = _seq(feats)
    for m in enc.modules():
        if isinstance(m, Conv):
            nn.init.kaiming_normal_(m.weight, mode="fan_out")  # mobilenetv2.py:229-230
    return enc


# build.py:11-22 ('swin_base'): the 4th stage is dropped at construction (swin_transformer.py:566)
SWIN_BASE = {"embed": 128, "depths": (2, 2, 18), "heads": (4, 8, 16), "window": 7, "patch": 4}


def swin_relative_position_index(ws):
    # swin_transformer.py:131-147
    ys, xs = torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij")
    y, x = ys.reshape(-1), xs.reshape(-1)
    return (y[:, None] - y[None, :] + ws - 1) * (2 * ws - 1) + (x[:, None] - x[None, :] + ws - 1)


def _swin_base():
    """Parameter tree of SwinTransformer(embed_dim=128, depths=[2,2,18,2], num_heads=[4,8,16,32]) with the
    reference's names (swin_transformer.py:571-640): patch_embed.{proj,norm}, layers.<i>.blocks.<j>.{norm1,
    attn.{relative_position_bias_table,relative_position_index,qkv,proj},norm2,mlp.{fc1,fc2}},
    layers.<i>.downsample.{reduction,norm}, norm<i>."""
    S = SWIN_BASE
    ws = S["window"]
    enc = ParamNode()
    enc.patch_embed = ParamNode()
    enc.patch_embed.proj = Conv(3, S["embed"], S["patch"])
    enc.patch_embed.norm = Norm(S["embed"])
    layers = []
    for i, (depth, heads) in enumerate(zip(S["depths"], S["heads"])):
        dim = S["embed"] * 2 ** i
        layer = ParamNode()
        blocks = []
        for _ in range(depth):
            b = ParamNode()
            b.norm1 = Norm(dim)
            b.attn = ParamNode()
            b.attn.relative_position_bias_table = nn.Parameter(torch.zeros((2 * ws - 1) ** 2, heads))
            nn.init.trunc_normal_(b.attn.relative_position_bias_table, std=0.02)    # :155
            b.attn.register_buffer("relative_position_index", swin_relative_position_index(ws))
            b.attn.qkv = Linear(dim, 3 * dim)
            b.attn.proj = Linear(dim, dim)
            b.norm2 = Norm(dim)
            b.mlp = ParamNode()
            b.mlp.fc1 = Linear(dim, 4 * dim)
            b.mlp.fc2 = Linear(4 * dim, dim)
            blocks.append(b)
        layer.blocks = nn.ModuleList(blocks)
        if i < len(S["depths"]) - 1:
            layer.downsample = ParamNode()
            red = ParamNode()
            red.weight = nn.Parameter(torch.empty(2 * dim, 4 * dim))               # Linear(4C, 2C, bias=False) :333
            nn.init.kaiming_uniform_(red.weight, a=math.sqrt(5))
            layer.downsample.reduction = red
            layer.downsample.norm = Norm(4 * dim)
        layers.append(layer)
    enc.layers = nn.ModuleList(layers)
    for i in range(len(S["depths"])):
        setattr(enc, f"norm{i}", Norm(S["embed"] * 2 ** i))
    return enc


def _make_divisible(v, divisor=8):
    # mobilenetv3.py:13-30
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < 0.9 * v else new_v


# mobilenetv3.py:152-169: k, t, c, SE, HS, s
_MBV3_CFGS = [[3, 1, 16, 0, 0, 1], [3, 4, 24, 0, 0, 2], [3, 3, 24, 0, 0, 1], [5, 3, 40, 1, 0, 2], [5, 3, 40, 1, 0, 1],
              [5, 3, 40, 1, 0, 1], [3, 6, 80, 0, 1, 2], [3, 2.5, 80, 0, 1, 1], [3, 2.3, 80, 0, 1, 1], [3, 2.3, 80, 0, 1, 1],
              [3, 6, 112, 1, 1, 1], [3, 6, 112, 1, 1, 1], [5, 6, 160, 1, 1, 2], [5, 6, 160, 1, 1, 1], [5, 6, 160, 1, 1, 1]]


def mobilenetv3_plan(output_stride=16):
    """(inp, hidden, oup, k, stride, dilation, se, hs) per InvertedResidual of MobileNetV3Large (mobilenetv3.py:172-192,
    width_mult 1), and the width of the last 1x1 conv (:195)."""
    plan, inp, cur, rate = [], _make_divisible(16), 2, 1
    for k, t, c, se, hs, s in _MBV3_CFGS:
        if cur == output_stride:
            dil = rate
            rate *= s
            s = 1
        else:
            dil = 1
            cur *= s
        oup, hid = _make_divisible(c), _make_divisible(inp * t)
        plan.append((inp, hid, oup, k, s, dil, bool(se), bool(hs)))
        inp = oup
    return plan, hid


def se_inter(c):
    return _make_divisible(c // 4)             # SELayer(channel, reduction=4), mobilenetv3.py:51-59


def _mobilenetv3():
    """Parameter tree of MobileNetV3Large (mobilenetv3.py:68-215) with the reference's names: features.0.{0,1} stem,
    features.<n>.conv.<m> per InvertedResidual (activations and a missing SE are parameter-free slots), SE as
    conv.<m>.fc.{0,2} (Linear with bias), conv.{0,1} the last 1x1 conv."""
    enc = ParamNode()

    def slot():
        return ParamNode()

    def se(c):
        m = ParamNode()
        m.fc = _seq([Linear(c, se_inter(c)), slot(), Linear(se_inter(c), c), slot()])
        return m

    feats = [_seq([Conv(3, 16, 3, bias=False), FrozenBN(16), slot()])]
    plan, last = mobilenetv3_plan(16)
    for inp, hid, oup, k, s, dil, use_se, hs in plan:
        if inp == hid:
            mods = [Conv(hid, hid, k, bias=False, groups=hid), FrozenBN(hid), slot(), se(hid) if use_se else slot()]
        else:
            mods = [Conv(inp, hid, 1, bias=False), FrozenBN(hid), slot(), Conv(hid, hid, k, bias=False, groups=hid),
                    FrozenBN(hid), se(hid) if use_se else slot(), slot()]
        blk = ParamNode()
        blk.conv = _seq(mods + [Conv(hid, oup, 1, bias=False), FrozenBN(oup)])
        feats.append(blk)
    enc.features = _seq(feats)
    enc.conv = _seq([Conv(plan[-1][2], last, 1, bias=False), FrozenBN(last), slot()])
    for m in enc.modules():                                     # mobilenetv3.py:217-230
        if isinstance(m, Conv):
            n = m.weight.shape[2] * m.weight.shape[3] * m.weight.shape[0]
            nn.init.normal_(m.weight, 0, math.sqrt(2.0 / n))
        elif isinstance(m, Linear):
            nn.init.normal_(m.weight, 0, 0.01)
            nn.init.zeros_(m.bias)
    return enc


# channel counts of the four feature maps each encoder returns (what cfg.MODEL_ENCODER_DIM must list)
ENCODER_DIMS = {"resnet50": [256, 512, 1024, 1024], "resnet101": [256, 512, 1024, 1024],
                "resnest50": [256, 512, 1024, 1024], "resnest101": [256, 512, 1024, 1024],
                "mobilenetv2": [24, 32, 96, 1280], "mobilenetv3": [24, 40, 112, 960], "swin_base": [128, 256, 512, 512]}


def build_encoder_params(name):
    if name in RESNET_LAYERS:
        return _resnet(RESNET_LAYERS[name])
    if name in RESNEST:
        return _resnest(*RESNEST[name])
    if name == "mobilenetv2":
        return _mobilenetv2()
    if name == "mobilenetv3":
        return _mobilenetv3()
    if name == "swin_base":
        return _swin_base()
    raise NotImplementedError(f"encoder '{name}' has no sm_90a path (available: {', '.join(ENCODER_DIMS)})")


# ---------------------------------------------------------------- transformer blocks
def _xavier(mod):
    for p in mod.parameters():
        if p.dim() > 1:
            nn.init.xavier_uniform_(p)


class _MHA(ParamNode):
    # attention.py:29-62
    def __init__(self, d, use_linear):
        super().__init__()
        if use_linear:
            self.linear_Q = Linear(d, d)
            self.linear_K = Linear(d, d)
            self.linear_V = Linear(d, d)
        self.projection = Linear(d, d)


class _LocalMHA(ParamNode):
    # attention.py:248-306 (use_linear=False)
    def __init__(self, d, H):
        super().__init__()
        self.relative_emb_k = Conv(d, H * 225, 1, bias=True, groups=H)
        self.relative_emb_v = nn.Parameter(torch.zeros(H, d // H, 225))
        self.projection = Linear(d, d)


class _GNAct(ParamNode):
    # basic.py:15-25
    def __init__(self, c):
        super().__init__()
        self.gn = Norm(c)
        self.conv = Conv(c, c, 5, bias=False, groups=c)


class LSTTBlock(ParamNode):
    # transformer.py:258-303 -- registration order does not matter for state_dict matching
    def __init__(self, d=256, self_H=8, att_H=8, ff=1024):
        super().__init__()
        self.norm1 = Norm(d)
        self.linear_Q = Linear(d, d)
        self.linear_V = Linear(d, d)
        self.long_term_attn = _MHA(d, use_linear=False)
        self.short_term_attn = _LocalMHA(d, att_H)
        self.norm2 = Norm(d)
        self.self_attn = _MHA(d, use_linear=True)
        self.norm3 = Norm(d)
        self.linear1 = Linear(d, ff)
        self.activation = _GNAct(ff)
        self.linear2 = Linear(ff, d)
        _xavier(self)

    def fuse_key_value_id(self, key, value, id_emb):  # transformer.py:364-367 (used by callers)
        raise RuntimeError("fuse_key_value_id runs inside the CUDA engine (aotb_linear with fused add)")


class _DW(ParamNode):
    def __init__(self, c):
        super().__init__()
        self.conv = Conv(c, c, 5, bias=False, groups=c)


class _GP(ParamNode):
    # attention.py:589-634
    def __init__(self, d_qk, d_vu, d_att, use_linear):
        super().__init__()
        e = d_vu * 2
        if use_linear:
            self.linear_QK = Linear(d_qk, d_att)
            self.linear_V1 = Linear(d_vu // 2, e // 2)
            self.linear_V2 = Linear(d_vu // 2, e // 2)
            self.linear_U1 = Linear(d_vu // 2, e // 2)
            self.linear_U2 = Linear(d_vu // 2, e // 2)
        self.dw_conv = _DW(e)
        self.projection = Linear(e, d_vu)
        _xavier(self)


class _LocalGP(ParamNode):
    # attention.py:720-787 (use_linear=False)
    def __init__(self, d_vu, d_att):
        super().__init__()
        e = d_vu * 2
        self.relative_emb_k = Conv(d_att, 225, 1, bias=True, groups=1)
        self.dw_conv = _DW(e)
        self.projection = Linear(e, d_vu)


class GPMBlock(ParamNode):
    # transformer.py:501-573 (att_nhead == 1 -> d_att = d_model // 2)
    def __init__(self, d=256, layer_idx=0):
        super().__init__()
        e = 2 * d
        d_att = d // 2
        self.norm1 = Norm(d)
        self.linear_QV = Linear(d, d_att + e)
        self.linear_U = Linear(d, e)
        if layer_idx == 0:
            self.linear_ID_V = Linear(d, e)
        else:
            self.id_norm1 = Norm(d)
            self.linear_ID_V = Linear(2 * d, e)
            self.linear_ID_U = Linear(d, e)
        self.long_term_attn = _GP(d, 2 * d, d_att, use_linear=False)
        self.short_term_attn = _LocalGP(2 * d, d_att)
        self.norm2 = Norm(d)
        self.id_norm2 = Norm(d)
        self.self_attn = _GP(2 * d, 2 * d, d_att, use_linear=True)
        _xavier(self)


class _ConvGN(ParamNode):
    def __init__(self, cin, cout, k):
        super().__init__()
        self.conv = Conv(cin, cout, k)
        self.gn = Norm(cout)


class FPNHead(ParamNode):
    # fpn.py:7-32
    def __init__(self, in_dim, out_dim, hidden, shortcut_dims):
        super().__init__()
        self.conv_in = _ConvGN(in_dim, hidden, 1)
        self.conv_16x = _ConvGN(hidden, hidden, 3)
        self.conv_8x = _ConvGN(hidden, hidden // 2, 3)
        self.conv_4x = _ConvGN(hidden // 2, hidden // 2, 3)
        self.adapter_16x = Conv(shortcut_dims[-2], hidden, 1)
        self.adapter_8x = Conv(shortcut_dims[-3], hidden, 1)
        self.adapter_4x = Conv(shortcut_dims[-4], hidden // 2, 1)
        self.conv_out = Conv(hidden // 2, out_dim, 1)
        _xavier(self)


class _GN1D(ParamNode):
    def __init__(self, c):
        super().__init__()
        self.gn = Norm(c)


# ---------------------------------------------------------------- models
class AOT(nn.Module):
    """networks/models/aot.py:9-115 (parameters only; see module docstring)."""

    def __init__(self, cfg, encoder="mobilenetv2", decoder="fpn"):
        super().__init__()
        if decoder != "fpn":
            raise NotImplementedError(decoder)
        self.cfg = cfg
        self.max_obj_num = cfg.MODEL_MAX_OBJ_NUM
        self.epsilon = cfg.MODEL_EPSILON
        d = cfg.MODEL_ENCODER_EMBEDDING_DIM
        L = cfg.MODEL_LSTT_NUM
        if not getattr(cfg, "MODEL_FREEZE_BN", True):
            raise NotImplementedError("the H100 hot path folds FrozenBatchNorm2d; MODEL_FREEZE_BN=False is train-only")
        dims = ENCODER_DIMS.get(encoder)
        if dims is not None and list(cfg.MODEL_ENCODER_DIM) != dims:
            raise ValueError(f"cfg.MODEL_ENCODER_DIM = {list(cfg.MODEL_ENCODER_DIM)} does not match encoder '{encoder}', whose "
                             f"feature maps have {dims} channels: set cfg.MODEL_ENCODER_DIM = {dims}")
        self.encoder = build_encoder_params(encoder)
        self.encoder_projector = Conv(cfg.MODEL_ENCODER_DIM[-1], d, 1)
        self._build_lstt(cfg, d, L)
        k = 17 if cfg.MODEL_ALIGN_CORNERS else 16
        self.patch_wise_id_bank = Conv(cfg.MODEL_MAX_OBJ_NUM + 1, d, k)
        nn.init.xavier_uniform_(self.encoder_projector.weight)
        with torch.no_grad():
            # aot.py:112-115 uses orthogonal_(gain=k^-2): rows of norm k^-2 in R^(11*k*k).  A
            # Gaussian with the same row norm is orthogonal up to O(1/sqrt(fan_in)) and, unlike
            # the LAPACK QR behind orthogonal_, is bit-reproducible across machines (tests rely
            # on seeded weights being identical here and on the GPU box).
            fan_in = (cfg.MODEL_MAX_OBJ_NUM + 1) * k * k
            nn.init.normal_(self.patch_wise_id_bank.weight, 0.0, float(k) ** -2 / math.sqrt(fan_in))
        self._plan = None

    def _build_lstt(self, cfg, d, L):
        lstt = ParamNode()
        lstt.mask_token = nn.Parameter(torch.randn(1, 1, d))  # transformer.py:59 (unused in forward)
        lstt.layers = nn.ModuleList([LSTTBlock(d, cfg.MODEL_SELF_HEADS, cfg.MODEL_ATT_HEADS) for _ in range(L)])
        n_norm = (L - 1 if cfg.MODEL_DECODER_INTERMEDIATE_LSTT else 0) + 1
        lstt.decoder_norms = nn.ModuleList([Norm(d) for _ in range(n_norm)])
        self.LSTT = lstt
        in_dim = d * (L + 1) if cfg.MODEL_DECODER_INTERMEDIATE_LSTT else d
        self.decoder = FPNHead(in_dim, cfg.MODEL_MAX_OBJ_NUM + 1, d, cfg.MODEL_ENCODER_DIM)

    def forward(self, *a, **k):
        raise RuntimeError("use networks.engines.build_engine(..., aot_model=model); the model has no eager forward")


class DeAOT(AOT):
    """networks/models/deaot.py:8-55."""

    def _build_lstt(self, cfg, d, L):
        lstt = ParamNode()
        lstt.layers = nn.ModuleList([GPMBlock(d, i) for i in range(L)])
        n_norm = (L - 1 if cfg.MODEL_DECODER_INTERMEDIATE_LSTT else 0) + 1
        lstt.decoder_norms = nn.ModuleList([_GN1D(2 * d) for _ in range(n_norm)])
        self.LSTT = lstt
        in_dim = d * (2 * L + 1) if cfg.MODEL_DECODER_INTERMEDIATE_LSTT else 2 * d
        self.decoder = FPNHead(in_dim, cfg.MODEL_MAX_OBJ_NUM + 1, d, cfg.MODEL_ENCODER_DIM)
        self.id_norm = Norm(d)


def build_vos_model(name, cfg, **kwargs):
    """networks/models/__init__.py:5-11."""
    if name == "aot":
        return AOT(cfg, encoder=cfg.MODEL_ENCODER, **kwargs)
    if name == "deaot":
        return DeAOT(cfg, encoder=cfg.MODEL_ENCODER, **kwargs)
    raise NotImplementedError(name)
