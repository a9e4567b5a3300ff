"""CPU oracle for the AOT / DeAOT mask-propagation hot path.

TEST INFRASTRUCTURE ONLY.  This module is the *checker*, never the product: only
``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference``
legs of ``bench.py`` may import it.  The product path (``aot_benchmark_b200``) never does.

What it is: a functional (no nn.Module) restatement, in plain torch-CPU tensor algebra,
of the per-frame algorithm of yoxu515/aot-benchmark @601c138.  Every function cites the
reference ``file:line`` it follows (paths relative to the reference root).  It consumes a
flat ``state_dict`` with the *reference's* parameter names, so the same dictionary can be
loaded into the reference model (``oracle/gen_golden.py`` does exactly that to pin this
file) and into the CUDA product model.

Parity pin: ``oracle/gen_golden.py`` imports the real reference from /root/reference (with
the MultiheadLocalAttentionV3->V2 patch of SURVEY.md 0.4), runs it on seeded inputs and
commits the outputs under ``tests/golden/``; ``tests/test_oracle_golden.py`` checks this
restatement against those vectors.  The third-party ``spatial_correlation_sampler``
boundary (ClementPinard/Pytorch-Correlation-extension, unpinned, absent) is restated from
the reference's own ``unfold`` branch (attention.py:343-348, 830-835).

``dtype`` may be float32 (reference arithmetic) or float64 (a higher-precision truth used
to size tolerances).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor

WINDOW = 15  # 2*max_dis+1, max_dis=7 (attention.py:253,262; transformer.py:269,514)
MAX_DIS = 7


# --------------------------------------------------------------------------------------
# configuration (restates configs/models/*.py; only the keys the hot path reads)
# --------------------------------------------------------------------------------------
class OracleConfig:
    """Mirror of the reference's merged model config (configs/default.py:7-9)."""

    _TABLE = {
        # name: (vos, encoder, encoder_dim, lstt_num, align_corners, test_gap)
        "aott": ("aot", "mobilenetv2", [24, 32, 96, 1280], 1, True, 9999),      # configs/models/aott.py, default.py:5-27
        "aots": ("aot", "mobilenetv2", [24, 32, 96, 1280], 2, True, 9999),      # configs/models/aots.py
        "aotb": ("aot", "mobilenetv2", [24, 32, 96, 1280], 3, True, 9999),      # configs/models/aotb.py
        "aotl": ("aot", "mobilenetv2", [24, 32, 96, 1280], 3, True, 5),         # configs/models/aotl.py:9-12
        "r50_aotl": ("aot", "resnet50", [256, 512, 1024, 1024], 3, True, 5),    # configs/models/r50_aotl.py:7-16
        "deaott": ("deaot", "mobilenetv2", [24, 32, 96, 1280], 1, True, 9999),  # configs/models/deaott.py
        "deaots": ("deaot", "mobilenetv2", [24, 32, 96, 1280], 2, True, 9999),  # configs/models/deaots.py
        "deaotb": ("deaot", "mobilenetv2", [24, 32, 96, 1280], 3, True, 9999),  # configs/models/deaotb.py
        "deaotl": ("deaot", "mobilenetv2", [24, 32, 96, 1280], 3, True, 5),     # configs/models/deaotl.py
        "r50_deaotl": ("deaot", "resnet50", [256, 512, 1024, 1024], 3, True, 5),  # configs/models/r50_deaotl.py
        "swinb_aotl": ("aot", "swin_base", [128, 256, 512, 512], 3, False, 5),   # configs/models/swinb_aotl.py:9-18
        "swinb_deaotl": ("deaot", "swin_base", [128, 256, 512, 512], 3, False, 5),  # configs/models/swinb_deaotl.py
    }

    def __init__(self, model: str = "r50_aotl"):
        vos, enc, enc_dim, lstt, ac, gap = self._TABLE[model]
        self.MODEL_NAME = model
        self.MODEL_VOS = vos
        self.MODEL_ENGINE = vos + "engine"
        self.MODEL_ENCODER = enc
        self.MODEL_ENCODER_DIM = enc_dim
        self.MODEL_ENCODER_EMBEDDING_DIM = 256
        self.MODEL_LSTT_NUM = lstt
        self.MODEL_ALIGN_CORNERS = ac
        self.MODEL_MAX_OBJ_NUM = 10
        self.MODEL_SELF_HEADS = 1 if vos == "deaot" else 8     # default_deaot.py:14-15 / default.py:16-17
        self.MODEL_ATT_HEADS = 1 if vos == "deaot" else 8
        self.MODEL_DECODER_INTERMEDIATE_LSTT = vos != "deaot"  # default_deaot.py:12
        self.TEST_LONG_TERM_MEM_GAP = gap
        self.TEST_SHORT_TERM_MEM_SKIP = 1


# --------------------------------------------------------------------------------------
# small building blocks
# --------------------------------------------------------------------------------------
def _lin(x: Tensor, W: Dict[str, Tensor], name: str) -> Tensor:
    return F.linear(x, W[name + ".weight"], W[name + ".bias"])


def _ln(x: Tensor, W: Dict[str, Tensor], name: str) -> Tensor:
    # nn.LayerNorm default eps 1e-5 (transformer.py:14-18)
    return F.layer_norm(x, (x.shape[-1],), W[name + ".weight"], W[name + ".bias"], 1e-5)


def silu(x: Tensor) -> Tensor:
    # attention.py:585-586
    return x * torch.sigmoid(x)


def seq_to_2d(x: Tensor, size_2d: Tuple[int, int]) -> Tensor:
    # basic.py:88-92  [hw, n, c] -> [n, c, h, w]
    h, w = size_2d
    _, n, c = x.shape
    return x.view(h, w, n, c).permute(2, 3, 0, 1).contiguous()


def frozen_bn(x: Tensor, W: Dict[str, Tensor], name: str, eps: float = 1e-5) -> Tensor:
    # normalization.py:19-43 (eval branch == F.batch_norm(training=False))
    scale = W[name + ".weight"] * torch.rsqrt(W[name + ".running_var"] + eps)
    shift = W[name + ".bias"] - W[name + ".running_mean"] * scale
    return x * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)


def dwconv5(x_seq: Tensor, weight: Tensor, size_2d: Tuple[int, int]) -> Tensor:
    # basic.py:38-57 (DWConv2d; Dropout2d is identity in eval): depthwise 5x5, pad 2, no bias
    h, w = size_2d
    _, bs, c = x_seq.shape
    x = x_seq.view(h, w, bs, c).permute(2, 3, 0, 1)
    x = F.conv2d(x, weight, None, 1, 2, 1, c)
    return x.reshape(bs, c, h * w).permute(2, 0, 1)


# --------------------------------------------------------------------------------------
# encoders
# --------------------------------------------------------------------------------------
def resnet50_forward(W: Dict[str, Tensor], img: Tensor, p: str = "encoder.") -> List[Tensor]:
    """resnet.py:140-157 (+ Bottleneck :34-54); layers [3,4,6], strides [1,2,2], layer4 dropped."""
    x = F.conv2d(img, W[p + "conv1.weight"], None, 2, 3)
    x = F.relu(frozen_bn(x, W, p + "bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    xs = []
    for li, (nblk, stride) in enumerate(((3, 1), (4, 2), (6, 2)), start=1):
        for bi in range(nblk):
            q = f"{p}layer{li}.{bi}."
            s = stride if bi == 0 else 1
            out = F.relu(frozen_bn(F.conv2d(x, W[q + "conv1.weight"]), W, q + "bn1"))
            out = F.relu(frozen_bn(F.conv2d(out, W[q + "conv2.weight"], None, s, 1), W, q + "bn2"))
            out = frozen_bn(F.conv2d(out, W[q + "conv3.weight"]), W, q + "bn3")
            if (q + "downsample.0.weight") in W:
                res = frozen_bn(F.conv2d(x, W[q + "downsample.0.weight"], None, s), W, q + "downsample.1")
            else:
                res = x
            x = F.relu(out + res)
        xs.append(x)
    xs.append(x)  # 16x twice (resnet.py:153-155)
    return xs


# (t, c, n, s) of mobilenetv2.py:149-158
_MBV2_SETTING = [[1, 16, 1, 1], [6, 24, 2, 2], [6, 32, 3, 2], [6, 64, 4, 2], [6, 96, 3, 1], [6, 160, 3, 2], [6, 320, 1, 1]]


def mobilenetv2_plan(output_stride: int = 16):
    """Restates the constructor loop mobilenetv2.py:168-205: list of (inp, oup, stride, dilation, t)."""
    plan = []
    inp = 32
    cur = 2
    rate = 1
    for t, c, n, s in _MBV2_SETTING:
        if cur == output_stride:
            stride, dil = 1, rate
            rate *= s
        else:
            stride, dil = s, 1
            cur *= s
        for i in range(n):
            if i == 0:
                plan.append((inp, c, stride, dil, t))
            else:
                plan.append((inp, c, 1, rate, t))
            inp = c
    return plan


def mobilenetv2_forward(W: Dict[str, Tensor], img: Tensor, p: str = "encoder.") -> List[Tensor]:
    """mobilenetv2.py:219-224; stages = features[0:4], [4:7], [7:14], [14:] (:207-212)."""

    def cbr(x, name, stride=1, groups=1, k=3, dil=1):
        pad = (k - 1) // 2 * dil  # mobilenetv2.py:41-42
        x = F.conv2d(x, W[name + ".0.weight"], None, stride, pad, dil, groups)
        return F.relu6(frozen_bn(x, W, name + ".1"))

    feats = []
    x = cbr(img, p + "features.0", stride=2)
    plan = mobilenetv2_plan(16)
    for idx, (inp, oup, stride, dil, t) in enumerate(plan, start=1):
        q = f"{p}features.{idx}.conv."
        hidden = int(round(inp * t))
        y = x
        j = 0
        if t != 1:
            y = cbr(y, q + "0", k=1)
            j = 1
        y = cbr(y, q + str(j), stride=stride, groups=hidden, dil=dil)
        y = F.conv2d(y, W[q + f"{j + 1}.weight"])
        y = frozen_bn(y, W, q + str(j + 2))
        x = x + y if (stride == 1 and inp == oup) else y
        if idx in (3, 6, 13):
            feats.append(x)
    x = cbr(x, p + "features.18", k=1)
    feats.append(x)
    return feats


# Swin-B as build.py:11-22 instantiates it: embed 128, depths [2,2,18,(2)], heads [4,8,16,(32)], window 7,
# ape=False, patch_norm=True, out_indices (0,1,2); the 4th stage is never built (swin_transformer.py:566).
SWIN_BASE = {"embed": 128, "depths": (2, 2, 18), "heads": (4, 8, 16), "window": 7, "patch": 4}


def swin_rel_index(ws: int) -> Tensor:
    """swin_transformer.py:131-147: index into the (2ws-1)^2 bias table for every (query, key) pair."""
    ys, xs = torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij")
    y, x = ys.reshape(-1), xs.reshape(-1)
    return (y[:, None] - y[None, :] + ws - 1) * (2 * ws - 1) + (x[:, None] - x[None, :] + ws - 1)


def swin_shift_mask(Hp: int, Wp: int, ws: int, shift: int, dtype) -> Tensor:
    """swin_transformer.py:416-438: region ids of the cyclically shifted padded map -> additive mask
    [nW, ws*ws, ws*ws] with -100 between tokens of different regions."""
    def band(n):
        r = torch.zeros(n, dtype=torch.long)
        r[n - ws:n - shift] = 1
        r[n - shift:] = 2
        return r
    reg = band(Hp)[:, None] * 3 + band(Wp)[None, :]
    reg = reg.view(Hp // ws, ws, Wp // ws, ws).permute(0, 2, 1, 3).reshape(-1, ws * ws)
    diff = reg[:, None, :] != reg[:, :, None]
    return torch.where(diff, torch.tensor(-100.0, dtype=dtype), torch.tensor(0.0, dtype=dtype))


def swin_block(W: Dict[str, Tensor], p: str, x: Tensor, H: int, Wd: int, heads: int, ws: int, shift: int) -> Tensor:
    """SwinTransformerBlock.forward swin_transformer.py:257-323 + WindowAttention.forward :158-196.
    x [H*Wd, C] (batch 1).  Zero padding is applied AFTER norm1 (:273-278), so padded tokens carry the
    qkv bias and take part in the softmax of their window."""
    C = x.shape[1]
    d = C // heads
    y = _ln(x, W, p + "norm1").view(H, Wd, C)
    pb, pr = (ws - H % ws) % ws, (ws - Wd % ws) % ws
    y = F.pad(y, (0, 0, 0, pr, 0, pb))
    Hp, Wp = H + pb, Wd + pr
    if shift > 0:
        y = torch.roll(y, shifts=(-shift, -shift), dims=(0, 1))
    nwy, nwx = Hp // ws, Wp // ws
    win = y.view(nwy, ws, nwx, ws, C).permute(0, 2, 1, 3, 4).reshape(nwy * nwx, ws * ws, C)
    qkv = _lin(win, W, p + "attn.qkv").view(nwy * nwx, ws * ws, 3, heads, d).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0] * (d ** -0.5), qkv[1], qkv[2]
    att = q @ k.transpose(-2, -1)                                              # [nW, heads, 49, 49]
    table = W[p + "attn.relative_position_bias_table"]                          # [(2ws-1)^2, heads]
    bias = table[swin_rel_index(ws).reshape(-1).to(table.device)].view(ws * ws, ws * ws, heads).permute(2, 0, 1)
    att = att + bias.unsqueeze(0)
    if shift > 0:
        att = att + swin_shift_mask(Hp, Wp, ws, shift, att.dtype).to(att.device).unsqueeze(1)
    att = torch.softmax(att, dim=-1)
    o = (att @ v).transpose(1, 2).reshape(nwy * nwx, ws * ws, C)
    o = _lin(o, W, p + "attn.proj")
    o = o.view(nwy, nwx, ws, ws, C).permute(0, 2, 1, 3, 4).reshape(Hp, Wp, C)
    if shift > 0:
        o = torch.roll(o, shifts=(shift, shift), dims=(0, 1))
    x = x + o[:H, :Wd].reshape(H * Wd, C)                                      # drop_path is identity in eval
    m = _lin(F.gelu(_lin(_ln(x, W, p + "norm2"), W, p + "mlp.fc1")), W, p + "mlp.fc2")   # Mlp :41-63, exact GELU
    return x + m


def swin_patch_merge(W: Dict[str, Tensor], p: str, x: Tensor, H: int, Wd: int) -> Tensor:
    """PatchMerging.forward swin_transformer.py:339-365: 2x2 neighbours concatenated in the order
    (0,0), (1,0), (0,1), (1,1), LayerNorm(4C), bias-free Linear 4C -> 2C."""
    C = x.shape[1]
    y = F.pad(x.view(H, Wd, C), (0, 0, 0, Wd % 2, 0, H % 2))
    y = torch.cat([y[0::2, 0::2], y[1::2, 0::2], y[0::2, 1::2], y[1::2, 1::2]], dim=-1)
    y = _ln(y.reshape(-1, 4 * C), W, p + "norm")
    return F.linear(y, W[p + "reduction.weight"])


def swin_forward(W: Dict[str, Tensor], img: Tensor, p: str = "encoder.") -> List[Tensor]:
    """SwinTransformer.forward swin_transformer.py:684-716 (+ PatchEmbed :473-489, BasicLayer :404-452) for
    'swin_base' (build.py:11-22).  Returns [4x(128), 8x(256), 16x(512), 16x(512)] NCHW (last one repeated, :714)."""
    S = SWIN_BASE
    ps, ws = S["patch"], S["window"]
    _, _, Hi, Wi = img.shape
    img = F.pad(img, (0, (ps - Wi % ps) % ps, 0, (ps - Hi % ps) % ps))
    x = F.conv2d(img, W[p + "patch_embed.proj.weight"], W[p + "patch_embed.proj.bias"], ps)
    H, Wd = x.shape[2], x.shape[3]
    x = x.flatten(2).transpose(1, 2)[0]                                        # [H*Wd, C]
    x = _ln(x, W, p + "patch_embed.norm")
    outs = []
    for i, (depth, heads) in enumerate(zip(S["depths"], S["heads"])):
        for j in range(depth):
            x = swin_block(W, f"{p}layers.{i}.blocks.{j}.", x, H, Wd, heads, ws, 0 if j % 2 == 0 else ws // 2)
        C = x.shape[1]
        outs.append(_ln(x, W, f"{p}norm{i}").view(1, H, Wd, C).permute(0, 3, 1, 2).contiguous())
        if i < len(S["depths"]) - 1:
            x = swin_patch_merge(W, f"{p}layers.{i}.downsample.", x, H, Wd)
            H, Wd = (H + 1) // 2, (Wd + 1) // 2
    outs.append(outs[-1])
    return outs


def encode_image(W: Dict[str, Tensor], cfg, img: Tensor) -> List[Tensor]:
    # aot.py:81-84
    if cfg.MODEL_ENCODER == "resnet50":
        xs = resnet50_forward(W, img)
    elif cfg.MODEL_ENCODER == "mobilenetv2":
        xs = mobilenetv2_forward(W, img)
    elif cfg.MODEL_ENCODER == "swin_base":
        xs = swin_forward(W, img)
    else:
        raise NotImplementedError(cfg.MODEL_ENCODER)
    xs[-1] = F.conv2d(xs[-1], W["encoder_projector.weight"], W["encoder_projector.bias"])
    return xs


# --------------------------------------------------------------------------------------
# positional / identity embeddings
# --------------------------------------------------------------------------------------
def pos_emb_sine(h: int, w: int, num_pos_feats: int = 128, dtype=torch.float32) -> Tensor:
    """position.py:49-74 with normalize=True, scale=2*pi, temperature=1e4 -> [1, 2*npf, h, w]."""
    y = torch.arange(h, dtype=torch.float32).view(1, h, 1).expand(1, h, w)
    x = torch.arange(w, dtype=torch.float32).view(1, 1, w).expand(1, h, w)
    eps = 1e-6
    y = y / (y[:, -1:, :] + eps) * (2 * math.pi)
    x = x / (x[:, :, -1:] + eps) * (2 * math.pi)
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32)
    dim_t = 10000 ** (2 * (dim_t // 2) / num_pos_feats)
    px = x[:, :, :, None] / dim_t
    py = y[:, :, :, None] / dim_t
    px = torch.stack((px[..., 0::2].sin(), px[..., 1::2].cos()), dim=4).flatten(3)
    py = torch.stack((py[..., 0::2].sin(), py[..., 1::2].cos()), dim=4).flatten(3)
    return torch.cat((py, px), dim=3).permute(0, 3, 1, 2).to(dtype)


def one_hot_mask(mask: Tensor, cls_num: int) -> Tensor:
    # utils/image.py:69-74
    if mask.dim() == 3:
        mask = mask.unsqueeze(1)
    idx = torch.arange(0, cls_num + 1, device=mask.device).view(1, -1, 1, 1).to(mask.dtype)
    return (mask == idx).to(mask.dtype)


def get_id_emb(W: Dict[str, Tensor], cfg, one_hot: Tensor) -> Tensor:
    """aot.py:50-63,76-79 (conv k17 s16 p8 if align_corners else k16 s16 p0); DeAOT adds LayerNorm
    over channels (deaot.py:51-55).  Returns [n, c, h16, w16]."""
    if cfg.MODEL_ALIGN_CORNERS:
        e = F.conv2d(one_hot, W["patch_wise_id_bank.weight"], W["patch_wise_id_bank.bias"], 16, 8)
    else:
        e = F.conv2d(one_hot, W["patch_wise_id_bank.weight"], W["patch_wise_id_bank.bias"], 16, 0)
    if cfg.MODEL_VOS == "deaot":
        e = _ln(e.permute(2, 3, 0, 1), W, "id_norm").permute(2, 3, 0, 1)
    return e


# --------------------------------------------------------------------------------------
# attention kernels (K1, K1', K2, K2', K3)
# --------------------------------------------------------------------------------------
def multihead_attention(Q: Tensor, K: Tensor, V: Tensor, H: int, d_att: Optional[int] = None) -> Tensor:
    """attention.py:82-117 core: Q/=T; per head softmax(QK^T)V; returns [Tq, bs, H*dv] *before*
    the projection.  Q [Tq,bs,H*d_att], K [Tk,bs,H*d_att], V [Tk,bs,H*dv]."""
    Tq, bs, _ = Q.shape
    d_att = Q.shape[2] // H if d_att is None else d_att
    dv = V.shape[2] // H
    Q = Q / (d_att ** 0.5)
    q = Q.view(Tq, bs, H, d_att).permute(1, 2, 0, 3)
    k = K.view(-1, bs, H, d_att).permute(1, 2, 3, 0)
    v = V.view(-1, bs, H, dv).permute(1, 2, 0, 3)
    attn = torch.softmax(q @ k, dim=-1)
    out = (attn @ v).permute(2, 0, 1, 3).reshape(Tq, bs, H * dv)
    return out


def local_window_scores(q2d: Tensor, k2d: Tensor, relk_w: Tensor, relk_b: Tensor, H: int) -> Tensor:
    """Window scores of SURVEY Appendix C == attention.py:318-357 (unfold branch :343-348).
    q2d,k2d [n, H*d, h, w].  Returns s [n, H, 225, h, w] (already masked with -1e8 / offsets
    in F.unfold order wi=(dy+7)*15+(dx+7))."""
    n, c, h, w = q2d.shape
    d = c // H
    T = d ** 0.5
    rel = F.conv2d(q2d, relk_w, relk_b, groups=H).view(n, H, WINDOW * WINDOW, h, w)  # on UNSCALED q (:327)
    qs = (q2d / T).view(n, H, d, h, w)
    kp = F.pad(k2d, (MAX_DIS, MAX_DIS, MAX_DIS, MAX_DIS)).view(n, H, d, h + 2 * MAX_DIS, w + 2 * MAX_DIS)
    ones = F.pad(torch.ones(1, 1, h, w, dtype=q2d.dtype, device=q2d.device), (MAX_DIS, MAX_DIS, MAX_DIS, MAX_DIS))
    s = torch.empty(n, H, WINDOW * WINDOW, h, w, dtype=q2d.dtype, device=q2d.device)
    big = 1e8 if q2d.dtype in (torch.float32, torch.float64) else 1e4
    for iy in range(WINDOW):
        for ix in range(WINDOW):
            wi = iy * WINDOW + ix
            ks = kp[:, :, :, iy:iy + h, ix:ix + w]
            inside = ones[:, :, iy:iy + h, ix:ix + w]
            s[:, :, wi] = (qs * ks).sum(dim=2) + rel[:, :, wi] - (1 - inside) * big
    return s


def local_window_aggregate(p: Tensor, v2d: Tensor, H: int, relv: Optional[Tensor]) -> Tensor:
    """o[g,:,y,x] = sum_wi p * (v[g,:,y+dy,x+dx] + relv[g,:,wi]) (attention.py:363-371; the
    dense local2global matmul :366-368 is the same sum).  p [n,H,225,h,w]; v2d [n,H*dv,h,w].
    Returns [hw, n, H*dv]."""
    n, cv, h, w = v2d.shape
    dv = cv // H
    vp = F.pad(v2d, (MAX_DIS, MAX_DIS, MAX_DIS, MAX_DIS)).view(n, H, dv, h + 2 * MAX_DIS, w + 2 * MAX_DIS)
    o = torch.zeros(n, H, dv, h, w, dtype=v2d.dtype, device=v2d.device)
    for iy in range(WINDOW):
        for ix in range(WINDOW):
            wi = iy * WINDOW + ix
            o += p[:, :, wi].unsqueeze(2) * vp[:, :, :, iy:iy + h, ix:ix + w]
    if relv is not None:
        # agg_bias = einsum('bhwn,hcw->bhnc') (attention.py:363-364)
        o += torch.einsum("bhwyx,hcw->bhcyx", p, relv)
    return o.permute(3, 4, 0, 1, 2).reshape(h * w, n, cv)


def local_attention_loop(q2d, k2d, v2d, relk_w, relk_b, relv, H) -> Tensor:
    """K2 / K2' before projection, tap-by-tap form of SURVEY Appendix C (independent cross-check of
    the unfold form below; slow on many-core hosts)."""
    s = local_window_scores(q2d, k2d, relk_w, relk_b, H)
    p = torch.softmax(s, dim=2)
    return local_window_aggregate(p, v2d, H, relv)


def local_attention(q2d, k2d, v2d, relk_w, relk_b, relv, H, chunk: int = 256) -> Tensor:
    """K2 / K2' before projection, in the reference's own `unfold` formulation
    (attention.py:318-371 / :805-853): zero-padded F.unfold windows of k and v, scores + relative_emb_k(q)
    (on UNSCALED q, :327) - 1e8 outside the frame (:355-357), softmax over the 225 taps, then
    sum_w p * v_window (+ einsum with relative_emb_v, :363-364).  The dense local2global matmul of
    :366-368 is the same sum.  v is processed in channel chunks to bound memory."""
    n, c, h, w = q2d.shape
    d = c // H
    T = d ** 0.5
    cv = v2d.shape[1]
    dv = cv // H
    P = WINDOW * WINDOW
    rel = F.conv2d(q2d, relk_w, relk_b, groups=H).view(n, H, P, h * w)
    ku = F.unfold(k2d, WINDOW, padding=MAX_DIS).view(n, H, d, P, h * w)
    s = torch.einsum("nhdp,nhdwp->nhwp", (q2d / T).view(n, H, d, h * w), ku) + rel
    inside = F.unfold(torch.ones(1, 1, h, w, dtype=q2d.dtype, device=q2d.device), WINDOW, padding=MAX_DIS).view(1, 1, P, h * w)
    s = s - (1 - inside) * 1e8
    p = torch.softmax(s, dim=2)
    o = torch.empty(n, H, dv, h * w, dtype=v2d.dtype, device=v2d.device)
    v5 = v2d.view(n, H, dv, h, w)
    for c0 in range(0, dv, chunk):
        c1 = min(dv, c0 + chunk)
        vu = F.unfold(v5[:, :, c0:c1].reshape(n, H * (c1 - c0), h, w), WINDOW, padding=MAX_DIS)
        o[:, :, c0:c1] = torch.einsum("nhwp,nhdwp->nhdp", p, vu.view(n, H, c1 - c0, P, h * w))
    if relv is not None:
        o = o + torch.einsum("nhwp,hcw->nhcp", p, relv)
    return o.permute(3, 0, 1, 2).reshape(h * w, n, cv)


# --------------------------------------------------------------------------------------
# AOT block  (transformer.py:312-367)
# --------------------------------------------------------------------------------------
def lstt_block(W, p: str, tgt: Tensor, long_mem, short_mem, curr_id_emb, pos: Tensor,
               size_2d, H: int = 8, taps: Optional[dict] = None):
    # 1) self-attention (transformer.py:321-326; attention.py:64-121 use_linear=True)
    s = _ln(tgt, W, p + "norm1")
    qk = s + pos
    Q = _lin(qk, W, p + "self_attn.linear_Q")
    K = _lin(qk, W, p + "self_attn.linear_K")
    V = _lin(s, W, p + "self_attn.linear_V")
    sa = _lin(multihead_attention(Q, K, V, H), W, p + "self_attn.projection")
    tgt = tgt + sa
    # 2) long + short term (transformer.py:329-352)
    s = _ln(tgt, W, p + "norm2")
    curr_Q = _lin(s, W, p + "linear_Q")
    curr_K = curr_Q
    curr_V = s
    local_Q = seq_to_2d(curr_Q, size_2d)
    if curr_id_emb is not None:
        global_K = curr_K
        global_V = _lin(curr_V + curr_id_emb, W, p + "linear_V")  # fuse_key_value_id :364-367
        local_K = seq_to_2d(global_K, size_2d)
        local_V = seq_to_2d(global_V, size_2d)
    else:
        global_K, global_V = long_mem
        local_K, local_V = short_mem
    lt_core = multihead_attention(curr_Q, global_K, global_V, H)
    lt = _lin(lt_core, W, p + "long_term_attn.projection")
    st_core = local_attention(local_Q, local_K, local_V,
                              W[p + "short_term_attn.relative_emb_k.weight"],
                              W[p + "short_term_attn.relative_emb_k.bias"],
                              W[p + "short_term_attn.relative_emb_v"], H)
    st = _lin(st_core, W, p + "short_term_attn.projection")
    if taps is not None:
        taps[p + "lt_in"] = (curr_Q, global_K, global_V)
        taps[p + "lt_core"] = lt_core
        taps[p + "st_in"] = (local_Q, local_K, local_V)
        taps[p + "st_core"] = st_core
    tgt = tgt + lt + st
    # 3) FFN (transformer.py:354-359; basic.py:27-35)
    s = _ln(tgt, W, p + "norm3")
    u = _lin(s, W, p + "linear1")
    h, w = size_2d
    _, bs, c = u.shape
    u2 = u.view(h, w, bs, c).permute(2, 3, 0, 1)
    u2 = F.group_norm(u2, 32, W[p + "activation.gn.weight"], W[p + "activation.gn.bias"], 1e-5)
    u2 = F.gelu(u2)
    u2 = F.conv2d(u2, W[p + "activation.conv.weight"], None, 1, 2, 1, c)
    u = u2.reshape(bs, c, h * w).permute(2, 0, 1)
    tgt = tgt + _lin(u, W, p + "linear2")
    return tgt, [[curr_K, curr_V], [global_K, global_V], [local_K, local_V]]


def lstt_forward(W, cfg, tgt, long_mems, short_mems, curr_id_emb, pos, size_2d, taps=None):
    """LongShortTermTransformer.forward transformer.py:95-140 (return_intermediate=True,
    intermediate_norm=True, final_norm=True)."""
    L = cfg.MODEL_LSTT_NUM
    out = tgt
    inter, mems = [], []
    for i in range(L):
        out, m = lstt_block(W, f"LSTT.layers.{i}.", out,
                            long_mems[i] if long_mems is not None else None,
                            short_mems[i] if short_mems is not None else None,
                            curr_id_emb, pos, size_2d, cfg.MODEL_ATT_HEADS, taps)
        inter.append(out)
        mems.append(m)
    # decoder_norms: L-1 intermediate + final  (:85-93,124-135)
    embs = [_ln(inter[i], W, f"LSTT.decoder_norms.{i}") for i in range(L - 1)]
    embs.append(_ln(inter[-1], W, f"LSTT.decoder_norms.{L - 1}"))
    return embs, mems


# --------------------------------------------------------------------------------------
# DeAOT block  (transformer.py:582-665; attention.py:636-712, 789-861)
# --------------------------------------------------------------------------------------
def gated_propagation(W, p: str, Q, K, V, U, size_2d, use_linear: bool):
    """GatedPropagation.forward attention.py:636-712, 1 head.  Returns [N, bs, d_vu]."""
    if use_linear:
        Q = K = _lin(Q, W, p + "linear_QK")
        half = V.shape[-1] // 2
        V = silu(torch.cat([_lin(V[..., :half], W, p + "linear_V1"), _lin(V[..., half:], W, p + "linear_V2")], -1))
        U = silu(torch.cat([_lin(U[..., :half], W, p + "linear_U1"), _lin(U[..., half:], W, p + "linear_U2")], -1))
    core = multihead_attention(Q, K, V, 1, d_att=Q.shape[-1])
    out = core * U
    out = dwconv5(out, W[p + "dw_conv.conv.weight"], size_2d)
    return _lin(out, W, p + "projection"), core


def local_gated_propagation(W, p: str, q2d, k2d, v2d, u_seq, size_2d):
    """LocalGatedPropagation.forward attention.py:789-861 with use_linear=False, 1 head."""
    core = local_attention(q2d, k2d, v2d, W[p + "relative_emb_k.weight"], W[p + "relative_emb_k.bias"], None, 1)
    out = core * u_seq
    out = dwconv5(out, W[p + "dw_conv.conv.weight"], size_2d)
    return _lin(out, W, p + "projection"), core


def gpm_fuse_id(W, p: str, value, id_emb):
    # transformer.py:659-665
    if value is not None:
        return silu(_lin(torch.cat([value, id_emb], dim=2), W, p + "linear_ID_V"))
    return silu(_lin(id_emb, W, p + "linear_ID_V"))


def gpm_block(W, p: str, layer_idx: int, tgt, tgt_id, long_mem, short_mem, curr_id_emb, size_2d,
              d_model: int = 256, taps: Optional[dict] = None):
    d_att = d_model // 2
    s = _ln(tgt, W, p + "norm1")
    qv = _lin(s, W, p + "linear_QV")
    curr_Q = curr_K = qv[..., :d_att]
    local_Q = seq_to_2d(curr_Q, size_2d)
    curr_V = silu(qv[..., d_att:])
    curr_U = _lin(s, W, p + "linear_U")
    if tgt_id is None:
        tgt_id = 0
        cat_U = torch.cat([silu(curr_U), torch.ones_like(curr_U)], dim=-1)
        curr_ID_V = None
    else:
        zs = _ln(tgt_id, W, p + "id_norm1")
        curr_ID_V = zs
        cat_U = silu(torch.cat([curr_U, _lin(zs, W, p + "linear_ID_U")], dim=-1))
    if curr_id_emb is not None:
        global_K, global_V = curr_K, curr_V
        local_K = seq_to_2d(global_K, size_2d)
        local_V = seq_to_2d(global_V, size_2d)
        global_ID_V = gpm_fuse_id(W, p, curr_ID_V, curr_id_emb)
        local_ID_V = seq_to_2d(global_ID_V, size_2d)
    else:
        global_K, global_V, _, global_ID_V = long_mem
        local_K, local_V, _, local_ID_V = short_mem
    cat_gV = torch.cat([global_V, global_ID_V], dim=-1)
    cat_lV = torch.cat([local_V, local_ID_V], dim=1)
    lt, lt_core = gated_propagation(W, p + "long_term_attn.", curr_Q, global_K, cat_gV, cat_U, size_2d, False)
    st, st_core = local_gated_propagation(W, p + "short_term_attn.", local_Q, local_K, cat_lV, cat_U, size_2d)
    if taps is not None:
        taps[p + "lt_in"] = (curr_Q, global_K, cat_gV, cat_U)
        taps[p + "lt_core"] = lt_core
        taps[p + "st_in"] = (local_Q, local_K, cat_lV)
        taps[p + "st_core"] = st_core
    tgt = tgt + lt[..., :d_model] + st[..., :d_model]
    tgt_id = tgt_id + lt[..., d_model:] + st[..., d_model:]
    c = torch.cat([_ln(tgt, W, p + "norm2"), _ln(tgt_id, W, p + "id_norm2")], dim=-1)
    sa, _ = gated_propagation(W, p + "self_attn.", c, c, c, c, size_2d, True)
    tgt = tgt + sa[..., :d_model]
    tgt_id = tgt_id + sa[..., d_model:]
    return tgt, tgt_id, [[curr_K, curr_V, None, curr_ID_V],
                         [global_K, global_V, None, global_ID_V],
                         [local_K, local_V, None, local_ID_V]]


def gpm_forward(W, cfg, tgt, long_mems, short_mems, curr_id_emb, size_2d, taps=None):
    """DualBranchGPM.forward transformer.py:205-255 (intermediate_norm=False, final_norm=True)."""
    L = cfg.MODEL_LSTT_NUM
    out, out_id = tgt, None
    inter, mems = [], []
    for i in range(L):
        out, out_id, m = gpm_block(W, f"LSTT.layers.{i}.", i, out, out_id,
                                   long_mems[i] if long_mems is not None else None,
                                   short_mems[i] if short_mems is not None else None,
                                   curr_id_emb, size_2d, cfg.MODEL_ENCODER_EMBEDDING_DIM, taps)
        inter.append(torch.cat([out, out_id], dim=2))
        mems.append(m)
    last = inter[-1]
    # GroupNorm1D(512, groups=2): basic.py:6-12
    last = F.group_norm(last.permute(1, 2, 0), 2, W["LSTT.decoder_norms.0.gn.weight"],
                        W["LSTT.decoder_norms.0.gn.bias"], 1e-5).permute(2, 0, 1)
    inter[-1] = last
    return inter, mems


# --------------------------------------------------------------------------------------
# FPN decoder  (fpn.py:34-58, basic.py:75-85)
# --------------------------------------------------------------------------------------
def _conv_gn(x, W, p, pad):
    x = F.conv2d(x, W[p + "conv.weight"], W[p + "conv.bias"], 1, pad)
    return F.group_norm(x, 8, W[p + "gn.weight"], W[p + "gn.bias"], 1e-5)


def fpn_decode(W, cfg, lstt_embs: Sequence[Tensor], shortcuts: Sequence[Tensor]) -> Tensor:
    """aot.py:86-92 / deaot.py:43-49 + fpn.py:34-58 -> [n, 11, h4, w4]."""
    n, c, h, w = shortcuts[-1].shape
    ac = cfg.MODEL_ALIGN_CORNERS
    inputs = [shortcuts[-1]] + [e.view(h, w, n, -1).permute(2, 3, 0, 1) for e in lstt_embs]
    x = torch.cat(inputs, dim=1) if cfg.MODEL_DECODER_INTERMEDIATE_LSTT else inputs[-1]
    p = "decoder."
    x = F.relu(_conv_gn(x, W, p + "conv_in.", 0))
    a = F.conv2d(shortcuts[-2], W[p + "adapter_16x.weight"], W[p + "adapter_16x.bias"])
    x = F.relu(_conv_gn(a + x, W, p + "conv_16x.", 1))
    x = F.interpolate(x, size=shortcuts[-3].shape[-2:], mode="bilinear", align_corners=ac)
    a = F.conv2d(shortcuts[-3], W[p + "adapter_8x.weight"], W[p + "adapter_8x.bias"])
    x = F.relu(_conv_gn(a + x, W, p + "conv_8x.", 1))
    x = F.interpolate(x, size=shortcuts[-4].shape[-2:], mode="bilinear", align_corners=ac)
    a = F.conv2d(shortcuts[-4], W[p + "adapter_4x.weight"], W[p + "adapter_4x.bias"])
    x = F.relu(_conv_gn(a + x, W, p + "conv_4x.", 1))
    return F.conv2d(x, W[p + "conv_out.weight"], W[p + "conv_out.bias"])


# --------------------------------------------------------------------------------------
# engine  (aot_engine.py:13-482, deaot_engine.py:9-56)
# --------------------------------------------------------------------------------------
class OracleEngine:
    """Single-engine (<= MODEL_MAX_OBJ_NUM objects), batch 1, eval-mode restatement of
    AOTEngine / DeAOTEngine.  Method names follow the reference."""

    def __init__(self, weights: Dict[str, Tensor], cfg, long_term_mem_gap: Optional[int] = None,
                 short_term_mem_skip: int = 1, dtype=torch.float32, keep_taps: bool = False, device="cpu"):
        # device="cuda": the same eager restatement on a GPU (bench.py's gpu_eager_baseline arm -- what the reference's
        # eager PyTorch code costs on the same GPU; still a baseline / checker, never the product path)
        self.cfg = cfg
        self.dtype = dtype
        self.device = torch.device(device)
        self.W = {k: (v.detach().to(self.device).to(dtype) if v.is_floating_point() else v.detach().to(self.device))
                  for k, v in weights.items()}
        self.deaot = cfg.MODEL_VOS == "deaot"
        self.max_obj_num = cfg.MODEL_MAX_OBJ_NUM
        self.long_term_mem_gap = cfg.TEST_LONG_TERM_MEM_GAP if long_term_mem_gap is None else long_term_mem_gap
        self.short_term_mem_skip = short_term_mem_skip
        self.keep_taps = keep_taps
        self.restart_engine()

    # aot_engine.py:445-477
    def restart_engine(self):
        self.frame_step = 0
        self.last_mem_step = -1
        self.obj_nums = None
        self.pos_emb = None
        self.enc_size_2d = None
        self.enc_hw = None
        self.input_size_2d = None
        self.long_term_memories = None
        self.short_term_memories_list = []
        self.short_term_memories = None
        self.curr_enc_embs = None
        self.curr_lstt_output = None
        self.pred_id_logits = None
        self.taps = {}

    def _lstt(self, enc_embs, long_mems, short_mems, id_emb):
        # aot.py:94-108
        n, c, h, w = enc_embs[-1].shape
        curr = enc_embs[-1].view(n, c, h * w).permute(2, 0, 1)
        taps = self.taps if self.keep_taps else None
        if taps is not None:
            taps.clear()
        if self.deaot:
            embs, mems = gpm_forward(self.W, self.cfg, curr, long_mems, short_mems, id_emb, self.enc_size_2d, taps)
        else:
            embs, mems = lstt_forward(self.W, self.cfg, curr, long_mems, short_mems, id_emb, self.pos_emb,
                                      self.enc_size_2d, taps)
        curr_m, long_m, short_m = zip(*mems)
        return embs, list(curr_m), list(long_m), list(short_m)

    def assign_identity(self, one_hot):
        # aot_engine.py:168-179
        e = get_id_emb(self.W, self.cfg, one_hot)
        return e.view(1, -1, self.enc_hw).permute(2, 0, 1)

    def add_reference_frame(self, img: Tensor, mask: Tensor, obj_nums, frame_step: int = -1):
        # aot_engine.py:188-251
        if isinstance(obj_nums, int):
            obj_nums = [obj_nums]
        self.obj_nums = obj_nums
        if frame_step == -1:
            frame_step = self.frame_step
        img = img.to(self.dtype)
        mask = mask.to(self.dtype)
        enc = encode_image(self.W, self.cfg, img)
        one_hot = one_hot_mask(mask, self.max_obj_num)
        if self.input_size_2d is None:
            self.input_size_2d = tuple(img.shape[2:])
            self.enc_size_2d = tuple(enc[-1].shape[2:])
            self.enc_hw = self.enc_size_2d[0] * self.enc_size_2d[1]
        self.curr_enc_embs = enc
        if self.pos_emb is None:
            self.pos_emb = pos_emb_sine(*self.enc_size_2d, dtype=self.dtype).to(self.device).view(1, -1, self.enc_hw).permute(2, 0, 1)
        id_emb = self.assign_identity(one_hot)
        self.curr_lstt_output = self._lstt(enc, None, None, id_emb)
        _, _, long_m, short_m = self.curr_lstt_output
        if self.long_term_memories is None:
            self.long_term_memories = long_m
        else:
            self.update_long_term_memory(long_m)
        self.last_mem_step = self.frame_step  # aot_engine.py:248 uses self.frame_step
        self.short_term_memories_list = [short_m]
        self.short_term_memories = short_m

    def update_long_term_memory(self, new_mems):
        # aot_engine.py:291-305: new frames are PREPENDED
        upd = []
        for new_m, last_m in zip(new_mems, self.long_term_memories):
            upd.append([None if (a is None or b is None) else torch.cat([a, b], dim=0)
                        for a, b in zip(new_m, last_m)])
        self.long_term_memories = upd

    def match_propogate_one_frame(self, img: Tensor):
        # aot_engine.py:340-354
        self.frame_step += 1
        enc = encode_image(self.W, self.cfg, img.to(self.dtype))
        self.curr_enc_embs = enc
        self.curr_lstt_output = self._lstt(enc, self.long_term_memories, self.short_term_memories, None)

    def decode_current_logits(self, output_size=None) -> Tensor:
        # aot_engine.py:356-380
        logits = fpn_decode(self.W, self.cfg, self.curr_lstt_output[0], self.curr_enc_embs)
        for b, obj_num in enumerate(self.obj_nums):
            logits[b, obj_num + 1:] = -1e10
        self.pred_id_logits = logits
        if output_size is not None:
            logits = F.interpolate(logits, size=tuple(int(s) for s in output_size), mode="bilinear",
                                   align_corners=self.cfg.MODEL_ALIGN_CORNERS)
        return logits

    def update_memory(self, curr_mask: Tensor, skip_long_term_update: bool = False):
        # AOTInferEngine.update_memory aot_engine.py:625-630 -> update_short_term_memory :307-338
        # (DeAOT override deaot_engine.py:20-56)
        one_hot = one_hot_mask(curr_mask.to(self.dtype), self.max_obj_num)
        id_emb = self.assign_identity(one_hot)
        curr_mems = self.curr_lstt_output[1]
        mems_2d = []
        for li in range(len(curr_mems)):
            p = f"LSTT.layers.{li}."
            if self.deaot:
                k, v, idk, idv = curr_mems[li]
                idv = gpm_fuse_id(self.W, p, idv, id_emb)
                curr_mems[li][2], curr_mems[li][3] = None, idv
                mems_2d.append([seq_to_2d(k, self.enc_size_2d), seq_to_2d(v, self.enc_size_2d), None,
                                seq_to_2d(idv, self.enc_size_2d)])
            else:
                k, v = curr_mems[li]
                v = _lin(v + id_emb, self.W, p + "linear_V")
                curr_mems[li][0], curr_mems[li][1] = k, v
                mems_2d.append([seq_to_2d(k, self.enc_size_2d), seq_to_2d(v, self.enc_size_2d)])
        self.short_term_memories_list.append(mems_2d)
        self.short_term_memories_list = self.short_term_memories_list[-self.short_term_mem_skip:]
        self.short_term_memories = self.short_term_memories_list[0]
        if self.frame_step - self.last_mem_step >= self.long_term_mem_gap:
            if not skip_long_term_update:
                self.update_long_term_memory(curr_mems)
            self.last_mem_step = self.frame_step


# --------------------------------------------------------------------------------------
# multi-engine facade  (AOTInferEngine aot_engine.py:485-635; DeAOTInferEngine deaot_engine.py:59-94 differs
# only in the sub-engine class it instantiates)
# --------------------------------------------------------------------------------------
class OracleInferEngine:
    """ceil(obj/10) OracleEngines sharing one image encoding; masks are split into per-engine id ranges
    (:515-545) and the per-engine logits are merged by soft_logit_aggregation (:565-582)."""

    def __init__(self, weights: Dict[str, Tensor], cfg, long_term_mem_gap: Optional[int] = None,
                 short_term_mem_skip: int = 1, dtype=torch.float32, device="cpu"):
        self.weights, self.cfg, self.dtype, self.device = weights, cfg, dtype, device
        self.long_term_mem_gap = cfg.TEST_LONG_TERM_MEM_GAP if long_term_mem_gap is None else long_term_mem_gap
        self.short_term_mem_skip = short_term_mem_skip
        self.max_aot_obj_num = cfg.MODEL_MAX_OBJ_NUM
        self.restart_engine()

    def restart_engine(self):                                           # :510-513
        self.aot_engines: List[OracleEngine] = []
        self.obj_nums = None

    def separate_mask(self, mask: Tensor, obj_nums: int):               # :515-545 (label-map branch)
        if len(self.aot_engines) == 1:
            return [mask], [obj_nums]
        M = self.max_aot_obj_num
        nums = [M] * len(self.aot_engines)
        if obj_nums % M > 0:
            nums[-1] = obj_nums % M
        masks = []
        for idx in range(len(self.aot_engines)):
            lo, hi = idx * M + 1, (idx + 1) * M
            fg = ((mask >= lo) & (mask <= hi)).to(mask.dtype)
            masks.append((fg * mask - lo + 1) * fg)
        return masks, nums

    def soft_logit_aggregation(self, all_logits: List[Tensor]) -> Tensor:   # :565-582
        if len(all_logits) == 1:
            return all_logits[0]
        M = self.max_aot_obj_num
        probs = [torch.softmax(l, dim=1) for l in all_logits]
        bg = torch.prod(torch.cat([p[:, 0:1] for p in probs], dim=1), dim=1, keepdim=True)
        merged = torch.cat([bg] + [p[:, 1:1 + M] for p in probs], dim=1).clamp(1e-5, 1 - 1e-5)
        return torch.logit(merged)

    def add_reference_frame(self, img: Tensor, mask: Tensor, obj_nums, frame_step: int = -1):   # :584-609
        if isinstance(obj_nums, list):
            obj_nums = obj_nums[0]
        self.obj_nums = obj_nums
        need = max(math.ceil(obj_nums / self.max_aot_obj_num), 1)
        while need > len(self.aot_engines):
            self.aot_engines.append(OracleEngine(self.weights, self.cfg, self.long_term_mem_gap,
                                                 self.short_term_mem_skip, self.dtype, device=self.device))
        masks, nums = self.separate_mask(mask, obj_nums)
        for eng, m, n in zip(self.aot_engines, masks, nums):
            # the reference encodes the image once and hands the embeddings on (:600-607); the oracle engines
            # simply re-encode (same values)
            eng.add_reference_frame(img, m, [n], frame_step)
        self.input_size_2d = self.aot_engines[0].input_size_2d
        self.enc_size_2d = self.aot_engines[0].enc_size_2d

    def match_propogate_one_frame(self, img: Tensor):                    # :611-616
        for eng in self.aot_engines:
            eng.match_propogate_one_frame(img)

    def decode_current_logits(self, output_size=None) -> Tensor:         # :618-623
        return self.soft_logit_aggregation([e.decode_current_logits(output_size) for e in self.aot_engines])

    def update_memory(self, curr_mask: Tensor, skip_long_term_update: bool = False):   # :625-630
        masks, _ = self.separate_mask(curr_mask, self.obj_nums)
        for eng, m in zip(self.aot_engines, masks):
            eng.update_memory(m, skip_long_term_update)


def run_video_events(engine, frames: Sequence[Tensor], first_mask: Tensor, obj_num: int,
                     output_size: Tuple[int, int], new_objects: Optional[Dict[int, Tensor]] = None,
                     forced_masks: Optional[Sequence[Tensor]] = None):
    """Evaluator.evaluating (evaluator.py:302-446, no TTA) including objects that first appear at a later frame
    (:338-340, :362-370, :380-402): at such a frame the predicted label is overwritten where the new annotation is
    non-zero, the frame is added as a reference frame with the enlarged object count, decoded again and written to
    memory.  `new_objects` maps frame index -> label map [1,1,H_out,W_out] holding ONLY the new ids.
    Returns (list of merged output-size logits, list of label maps fed back to the engine)."""
    new_objects = new_objects or {}
    engine.restart_engine()
    engine.add_reference_frame(frames[0], first_mask, obj_nums=[obj_num], frame_step=0)
    logits, labels = [], []
    for t in range(1, len(frames)):
        engine.match_propogate_one_frame(frames[t])
        logit = engine.decode_current_logits(output_size)
        label = torch.argmax(torch.softmax(logit, dim=1), dim=1, keepdim=True).to(logit.dtype)
        if forced_masks is not None:
            label = forced_masks[t - 1].to(label.device, label.dtype)
        new = new_objects.get(t)
        if new is not None:
            new = new.to(label.device, label.dtype)
            if forced_masks is None:
                keep = (new == 0).to(label.dtype)
                label = label * keep + new * (1 - keep)
            obj_num = max(obj_num, int(new.max().item()))
            fb = F.interpolate(label, size=tuple(engine.input_size_2d), mode="nearest")
            engine.add_reference_frame(frames[t], fb, obj_nums=[obj_num], frame_step=t)
            logit = engine.decode_current_logits(output_size)
            engine.update_memory(fb)
        else:
            fb = F.interpolate(label, size=tuple(engine.input_size_2d), mode="nearest")
            engine.update_memory(fb)
        logits.append(logit.detach().clone())
        labels.append(label.detach().clone())
    return logits, labels


# --------------------------------------------------------------------------------------
# the evaluator's per-frame span (evaluator.py:325-446), single engine, no TTA
# --------------------------------------------------------------------------------------
def run_video(engine, frames: Sequence[Tensor], first_mask: Tensor, obj_num: int,
              output_size: Tuple[int, int], forced_masks: Optional[Sequence[Tensor]] = None,
              on_frame=None):
    """Drive any engine exposing the reference protocol exactly like Evaluator.evaluating does.
    Returns (list of low-res pred_id_logits, list of output-size label maps).  If
    ``forced_masks`` is given, these labels (output size) are fed back instead of the engine's
    own argmax (teacher forcing, SURVEY Appendix E)."""
    engine.restart_engine()
    engine.add_reference_frame(frames[0], first_mask, obj_nums=[obj_num], frame_step=0)
    logits_lo, labels = [], []
    for t in range(1, len(frames)):
        engine.match_propogate_one_frame(frames[t])
        logit = engine.decode_current_logits(output_size)
        prob = torch.softmax(logit, dim=1)
        label = torch.argmax(prob, dim=1, keepdim=True).to(logit.dtype)
        lo = getattr(engine, "pred_id_logits", None)
        if lo is None and hasattr(engine, "aot_engines"):
            lo = engine.aot_engines[0].pred_id_logits
        logits_lo.append(lo.detach().clone() if lo is not None else None)
        labels.append(label.detach().clone())
        fb = label if forced_masks is None else forced_masks[t - 1].to(label.device, label.dtype)
        fb = F.interpolate(fb, size=tuple(engine.input_size_2d), mode="nearest")
        engine.update_memory(fb)
        if on_frame is not None:
            on_frame(t, logit, label)
    return logits_lo, labels


# --------------------------------------------------------------------------------------
# synthetic inputs (SURVEY 8d) -- deterministic, shared by tests / bench / golden generation
# --------------------------------------------------------------------------------------
def synthetic_video(num_frames: int, h: int, w: int, obj_num: int, seed: int = 1234,
                    label_hw: Optional[Tuple[int, int]] = None):
    """Low-pass-filtered noise frames with a per-frame drift + a first-frame mask of ``obj_num``
    non-overlapping rectangles (ids 1..obj_num).  Returns (frames list [1,3,h,w] float32,
    mask [1,1,h,w] float32)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(1, 3, h // 8 + 4, w // 8 + 4, generator=g)
    frames = []
    for t in range(num_frames):
        drift = 0.15 * torch.randn(1, 3, h // 8 + 4, w // 8 + 4, generator=g)
        cur = base + drift
        dx = (t * 3) % 16
        up = F.interpolate(cur, size=(h + 32, w + 32), mode="bilinear", align_corners=False)
        frames.append(up[:, :, 8:8 + h, dx:dx + w].contiguous() + 0.05 * torch.randn(1, 3, h, w, generator=g))
    lh, lw = (h, w) if label_hw is None else label_hw
    mask = torch.zeros(1, 1, lh, lw)
    cols = min(5, max(obj_num, 1))
    rows = (obj_num + cols - 1) // cols
    cw, rh = lw // cols, lh // max(rows, 1)
    for i in range(obj_num):
        r, c = divmod(i, cols)
        y0, x0 = r * rh + rh // 6, c * cw + cw // 6
        mask[:, :, y0:y0 + max(rh * 2 // 3, 1), x0:x0 + max(cw * 2 // 3, 1)] = i + 1
    return frames, mask
