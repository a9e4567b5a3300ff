"""Packed, device-resident copies of a model's parameters in the layouts the kernels read.

* convolutions   [Cout,Cin,KH,KW] -> [KH*KW*Cin, Cout] with FrozenBatchNorm2d folded in
  (networks/layers/normalization.py:30-43: y = (x-mean)*w/sqrt(var+eps)+b, folded in float64);
* depthwise convs [C,1,K,K]        -> [K*K, C];
* linears        [out,in]          -> [in, out]; sibling projections that share an input or an
  output are concatenated so one GEMM replaces two (self-attention Q|K, and the long-term +
  short-term output projections whose results the reference adds, transformer.py:349-352);
* ID bank        [C,11,K,K]        -> [(ky*K+kx)*11 + id, C]  (gather table == dense-conv layout).

The plan is cached on the model and rebuilt when any parameter's version counter or device
changes (``load_state_dict`` / ``.to()`` after a plan was built).
"""
from __future__ import annotations

from types import SimpleNamespace as NS

import torch

from .model import (RESNEST, RESNET_LAYERS, SWIN_BASE, mobilenetv2_plan, mobilenetv3_plan,
                    swin_relative_position_index)


def _signature(model):
    items = list(model.named_parameters()) + list(model.named_buffers())
    return tuple((n, t._version, t.data_ptr(), str(t.device)) for n, t in items)


def get_plan(model):
    sig = _signature(model)
    cached = getattr(model, "_aotb_plan", None)
    if cached is not None and cached[0] == sig:
        return cached[1]
    plan = Plan(model)
    model._aotb_plan = (sig, plan)
    return plan


class Plan:
    def __init__(self, model):
        cfg = model.cfg
        self.cfg = cfg
        dev = next(model.parameters()).device
        self._require_cuda(dev)
        self.device = dev
        # all packing arithmetic (float64 BN fold, transposes, fp16 hi/lo splits, prefix sums) runs on the HOST on a copy of
        # the state dict and only the finished tables are uploaded (_upload): building a plan launches no GPU kernels, so
        # the first launches of a process are the path's own kernels (and a reload costs memcpys, not ~1000 tiny launches)
        sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
        self.sd = sd
        self.deaot = cfg.MODEL_VOS == "deaot"
        self.L = cfg.MODEL_LSTT_NUM
        self.C = cfg.MODEL_ENCODER_EMBEDDING_DIM
        self.H = cfg.MODEL_ATT_HEADS
        self.align_corners = bool(cfg.MODEL_ALIGN_CORNERS)
        self.nid = cfg.MODEL_MAX_OBJ_NUM + 1
        self._tc_keys = []
        self._tc_list = []
        self._encoder(cfg.MODEL_ENCODER)
        w = sd["encoder_projector.weight"]
        self.proj = NS(w=self._reg(self._conv_w(w), w.shape[1]), b=self._f(sd["encoder_projector.bias"]))
        self.layers = [self._gpm_layer(i) if self.deaot else self._lstt_layer(i) for i in range(self.L)]
        self._decoder()
        self._idbank()
        self._upload()
        self.sd = None

    def _upload(self):
        """Move every packed host tensor hanging off the plan to the device (shared tensors stay shared) and register the
        split-fp16 [Cout, K] copies of the GEMM-shaped weights, normalised per output channel, and their scales under
        their device pointers."""
        from . import ops
        memo = {}

        def up(t):
            e = memo.get(id(t))
            if e is None:
                e = memo[id(t)] = (t, t.to(self.device))      # keep the host tensor alive: ids stay unique during the walk
            return e[1]

        def walk(o):
            if isinstance(o, torch.Tensor):
                return up(o)
            if isinstance(o, NS):
                for k, v in list(vars(o).items()):
                    setattr(o, k, walk(v))
                return o
            if isinstance(o, list):
                return [walk(v) for v in o]
            if isinstance(o, tuple):
                return tuple(walk(v) for v in o)
            return o

        for k, v in list(vars(self).items()):
            if k not in ("sd", "cfg", "device", "_tc_keys", "_tc_list"):
                setattr(self, k, walk(v))
        for w in self._tc_list:
            e = memo.get(id(w))
            if e is None:
                continue                                       # e.g. Q / K projections that only live on concatenated
            wh, wl, ws = ops.split_fp16_scaled(w)
            ops.register_tc_weights(e[1], wh.to(self.device), wl.to(self.device), ws.to(self.device))
            self._tc_keys.append(e[1].data_ptr())
        self._tc_list = []

    @staticmethod
    def _require_cuda(dev):
        if dev.type != "cuda":
            raise RuntimeError("aot_benchmark_b200 runs on CUDA devices only (no CPU path): move the model to "
                               "a GPU before building an engine")

    def _reg(self, w, cin=None):
        """Register split-fp16 [Cout, K] copies of a GEMM-shaped fp32 weight [K, Cout] for the tensor-core conv
        (eligible when the per-tap channel count and Cout are multiples of 64); ops.conv2d / ops.linear pick them up."""
        K, N = w.shape
        cin = K if cin is None else cin
        if cin % 4 == 0 and N % 64 == 0 and (cin % 64 == 0 or K != cin):   # general-Cin path only for real convs (stem)
            self._tc_list.append(w)                                         # split + registered at upload time
        return w

    def __del__(self):
        try:
            from . import ops
            for k in self._tc_keys:
                ops._TC_WEIGHTS.pop(k, None)
        except Exception:
            pass

    # ------------------------------------------------------------------ helpers
    def _f(self, t):
        return t.to(torch.float32).contiguous()            # host; uploaded by _upload()

    def _conv_w(self, w, scale=None):
        # [Cout,Cin,KH,KW] -> [KH*KW*Cin, Cout]
        w = w.double()
        if scale is not None:
            w = w * scale.view(-1, 1, 1, 1)
        co, ci, kh, kw = w.shape
        return self._f(w.permute(2, 3, 1, 0).reshape(kh * kw * ci, co).float())

    def _dw_w(self, w, scale=None):
        # [C,1,K,K] -> [K*K, C]
        w = w.double()
        if scale is not None:
            w = w * scale.view(-1, 1, 1, 1)
        c, _, kh, kw = w.shape
        return self._f(w.permute(2, 3, 1, 0).reshape(kh * kw, c).float())

    def _bn(self, name):
        sd = self.sd
        eps = 1e-5
        scale = sd[name + ".weight"].double() / torch.sqrt(sd[name + ".running_var"].double() + eps)
        shift = sd[name + ".bias"].double() - sd[name + ".running_mean"].double() * scale
        return scale, shift

    def _conv_bn(self, conv, bn, depthwise=False, pad_cin_to=None):
        scale, shift = self._bn(bn)
        w = self.sd[conv + ".weight"]
        if pad_cin_to is not None and w.shape[1] < pad_cin_to:
            w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, pad_cin_to - w.shape[1]))   # zero input channels
        ns = NS(b=self._f(shift.float()), k=w.shape[2], cin=w.shape[1], cout=w.shape[0])
        ns.w = self._dw_w(w, scale) if depthwise else self._reg(self._conv_w(w, scale), w.shape[1])
        return ns

    def _lin(self, name):
        return self._reg(self._f(self.sd[name + ".weight"].t())), self._f(self.sd[name + ".bias"])

    def _norm(self, name):
        return self._f(self.sd[name + ".weight"]), self._f(self.sd[name + ".bias"])

    # ------------------------------------------------------------------ encoders
    def _encoder(self, name):
        self.encoder_name = name
        p = "encoder."
        if name in RESNET_LAYERS:
            e = NS(stem=self._conv_bn(p + "conv1", p + "bn1", pad_cin_to=4), stages=[])   # image is fed as NHWC4
            for li, (nblk, stride) in enumerate(zip(RESNET_LAYERS[name], (1, 2, 2)), start=1):
                blocks = []
                for bi in range(nblk):
                    q = f"{p}layer{li}.{bi}."
                    b = NS(c1=self._conv_bn(q + "conv1", q + "bn1"), c2=self._conv_bn(q + "conv2", q + "bn2"),
                           c3=self._conv_bn(q + "conv3", q + "bn3"), stride=stride if bi == 0 else 1, down=None)
                    if (q + "downsample.0.weight") in self.sd:
                        b.down = self._conv_bn(q + "downsample.0", q + "downsample.1")
                    blocks.append(b)
                e.stages.append(blocks)
            self.enc = e
        elif name == "mobilenetv2":
            e = NS(stem=self._conv_bn(p + "features.0.0", p + "features.0.1", pad_cin_to=4), blocks=[])
            for idx, (inp, oup, stride, dil, t) in enumerate(mobilenetv2_plan(16), start=1):
                q = f"{p}features.{idx}.conv."
                b = NS(stride=stride, dil=dil, res=(stride == 1 and inp == oup), expand=None, tap=idx in (3, 6, 13))
                j = 0
                if t != 1:
                    b.expand = self._conv_bn(q + "0.0", q + "0.1")
                    j = 1
                b.dw = self._conv_bn(q + f"{j}.0", q + f"{j}.1", depthwise=True)
                b.pw = self._conv_bn(q + f"{j + 1}", q + f"{j + 2}")
                e.blocks.append(b)
            e.last = self._conv_bn(p + "features.18.0", p + "features.18.1")
            self.enc = e
        elif name == "swin_base":
            self.enc = self._swin(p)
        elif name == "mobilenetv3":
            self.enc = self._mobilenetv3(p)
        elif name in RESNEST:
            self.enc = self._resnest(p, RESNEST[name][0])
        else:
            raise NotImplementedError(f"encoder '{name}' has no sm_90a path")

    def _mobilenetv3(self, p):
        """MobileNetV3-Large (mobilenetv3.py:78-215) weights: the stem over the NHWC4 image, per block the expand conv (absent
        in block 1), the depthwise conv and the pw-linear conv with their BN folded, and the SE as fc1 [C, inter] + bias and fc2
        [inter, C] + bias; then the last 1x1 conv."""
        sd = self.sd
        e = NS(stem=self._conv_bn(p + "features.0.0", p + "features.0.1", pad_cin_to=4), blocks=[])
        plan, _ = mobilenetv3_plan(16)
        for idx, (inp, hid, oup, k, stride, dil, se, hs) in enumerate(plan, start=1):
            q = f"{p}features.{idx}.conv."
            b = NS(k=k, stride=stride, dil=dil, hs=hs, res=(stride == 1 and inp == oup), expand=None, se=None,
                   tap=idx in (3, 6, 12))
            if inp == hid:                       # dw, bn, act, SE slot, pw, bn: no block of the table has an SE here
                assert not se, "MobileNetV3 block without an expand conv and with SE is not in the reference's table"
                b.dw, b.pw = self._conv_bn(q + "0", q + "1", depthwise=True), self._conv_bn(q + "4", q + "5")
            else:                                # pw, bn, act, dw, bn, SE slot, act, pw-linear, bn
                b.expand = self._conv_bn(q + "0", q + "1")
                b.dw, b.pw = self._conv_bn(q + "3", q + "4", depthwise=True), self._conv_bn(q + "7", q + "8")
                if se:
                    f = q + "5.fc."
                    b.se = NS(w1=self._f(sd[f + "0.weight"].t()), b1=self._f(sd[f + "0.bias"]),
                              w2=self._f(sd[f + "2.weight"].t()), b2=self._f(sd[f + "2.bias"]))
            e.blocks.append(b)
        e.last = self._conv_bn(p + "conv.0", p + "conv.1")
        return e

    def _resnest(self, p, layers):
        """ResNeSt-50 / ResNeSt-101 (resnest/resnet.py:191-357, splat.py:15-115) weights: the deep stem as three 3x3 convs (the first over
        the NHWC4 image), per bottleneck conv1 / conv3 with bn1 / bn3 folded, the radix-2 grouped 3x3 conv of SplAtConv2d as
        one [9 * gw/2, gw] weight per group with its slice of bn0 folded (each group is one launch on channel slices), fc1 with
        bn1 folded as [gw, inter] + bias, fc2 as [inter, 2 gw] + bias, and the avg_down downsample conv with its BN folded."""
        sd = self.sd
        e = NS(stem=[self._conv_bn(p + "conv1.0", p + "conv1.1", pad_cin_to=4), self._conv_bn(p + "conv1.3", p + "conv1.4"),
                     self._conv_bn(p + "conv1.6", p + "bn1")], stages=[])
        for li, (nblk, stride) in enumerate(zip(layers, (1, 2, 2)), start=1):
            blocks = []
            for bi in range(nblk):
                q = f"{p}layer{li}.{bi}."
                s = q + "conv2."
                b = NS(c1=self._conv_bn(q + "conv1", q + "bn1"), c3=self._conv_bn(q + "conv3", q + "bn3"),
                       stride=stride if bi == 0 else 1, down=None)
                scale, shift = self._bn(s + "bn0")
                w = sd[s + "conv.weight"]                                   # [2 gw, gw / 2, 3, 3], groups = 2
                gw = w.shape[0] // 2
                b.gw = gw
                b.groups = [NS(w=self._reg(self._conv_w(w[g * gw:(g + 1) * gw], scale[g * gw:(g + 1) * gw]), w.shape[1]),
                               b=self._f(shift[g * gw:(g + 1) * gw].float())) for g in range(2)]
                s1, t1 = self._bn(s + "bn1")                                 # fc1 (1x1 conv with bias) -> bn1, in float64
                w1 = sd[s + "fc1.weight"].double().flatten(1) * s1.view(-1, 1)
                b.fc1_w = self._f(w1.t().float())                           # [gw, inter]
                b.fc1_b = self._f((sd[s + "fc1.bias"].double() * s1 + t1).float())
                b.fc2_w = self._f(sd[s + "fc2.weight"].flatten(1).t())      # [inter, 2 gw]
                b.fc2_b = self._f(sd[s + "fc2.bias"])
                if (q + "downsample.1.weight") in sd:
                    b.down = self._conv_bn(q + "downsample.1", q + "downsample.2")
                blocks.append(b)
            e.stages.append(blocks)
        return e

    def _swin(self, p):
        """Swin-B (build.py:11-22) weights: every Linear as [in, out] (registered for the tensor-core GEMM), the 4x4/4
        patch embedding as a conv over the NHWC4 image (fp32 CUDA-core path: K = 64), and per block the dense
        [heads, 49, 49] relative-position bias = table[index] (swin_transformer.py:176-183), gathered once here
        instead of once per block per frame."""
        sd = self.sd
        S = SWIN_BASE
        ws = S["window"]
        pw = sd[p + "patch_embed.proj.weight"]
        pw = torch.nn.functional.pad(pw, (0, 0, 0, 0, 0, 4 - pw.shape[1]))        # zero 4th input channel (NHWC4 image)
        e = NS(embed=S["embed"], window=ws, patch=NS(w=self._conv_w(pw), b=self._f(sd[p + "patch_embed.proj.bias"])),
               patch_norm=self._norm(p + "patch_embed.norm"), stages=[])
        idx = swin_relative_position_index(ws).reshape(-1)
        for i, (depth, heads) in enumerate(zip(S["depths"], S["heads"])):
            dim = S["embed"] * 2 ** i
            stg = NS(dim=dim, heads=heads, blocks=[], down=None, norm=self._norm(f"{p}norm{i}"))
            for j in range(depth):
                q = f"{p}layers.{i}.blocks.{j}."
                b = NS(shift=0 if j % 2 == 0 else ws // 2)
                b.norm1 = self._norm(q + "norm1")
                b.qkv_w, b.qkv_b = self._lin(q + "attn.qkv")
                table = sd[q + "attn.relative_position_bias_table"]                 # [(2ws-1)^2, heads]
                b.relb = self._f(table[idx].view(ws * ws, ws * ws, heads).permute(2, 0, 1))
                b.proj_w, b.proj_b = self._lin(q + "attn.proj")
                b.norm2 = self._norm(q + "norm2")
                b.fc1_w, b.fc1_b = self._lin(q + "mlp.fc1")
                b.fc2_w, b.fc2_b = self._lin(q + "mlp.fc2")
                stg.blocks.append(b)
            q = f"{p}layers.{i}.downsample."
            if (q + "reduction.weight") in sd:
                w = self._reg(self._f(sd[q + "reduction.weight"].t()))
                stg.down = NS(norm=self._norm(q + "norm"), w=w,
                              b=torch.zeros(w.shape[1], dtype=torch.float32))   # bias=False :333
            e.stages.append(stg)
        return e

    # ------------------------------------------------------------------ AOT block
    def _lstt_layer(self, i):
        p = f"LSTT.layers.{i}."
        sd = self.sd
        n = NS()
        n.norm1 = self._norm(p + "norm1")
        wq, bq = self._lin(p + "self_attn.linear_Q")
        wk, bk = self._lin(p + "self_attn.linear_K")
        n.sa_qk_w = self._reg(torch.cat([wq, wk], dim=1).contiguous())
        n.sa_qk_b = torch.cat([bq, bk]).contiguous()
        n.sa_v_w, n.sa_v_b = self._lin(p + "self_attn.linear_V")
        n.sa_proj_w, n.sa_proj_b = self._lin(p + "self_attn.projection")
        n.norm2 = self._norm(p + "norm2")
        n.linQ_w, n.linQ_b = self._lin(p + "linear_Q")
        n.linV_w, n.linV_b = self._lin(p + "linear_V")
        wl, bl = self._lin(p + "long_term_attn.projection")
        ws, bs = self._lin(p + "short_term_attn.projection")
        n.lst_proj_w = self._reg(torch.cat([wl, ws], dim=0).contiguous())   # [2C, C]: x += [lt|st] @ W
        n.lst_proj_b = (bl.double() + bs.double()).float().contiguous()
        rk = sd[p + "short_term_attn.relative_emb_k.weight"]
        n.relk_w = self._f(rk.reshape(rk.shape[0], rk.shape[1]))       # [H*225, d]
        n.relk_b = self._f(sd[p + "short_term_attn.relative_emb_k.bias"])
        n.relv = self._f(sd[p + "short_term_attn.relative_emb_v"])     # [H, d, 225]
        n.relv_t = n.relv.permute(0, 2, 1).contiguous()                # [H, 225, d] for the tiled kernel
        n.norm3 = self._norm(p + "norm3")
        n.lin1_w, n.lin1_b = self._lin(p + "linear1")
        n.gn = self._norm(p + "activation.gn")
        n.dw_w = self._dw_w(sd[p + "activation.conv.weight"])
        n.lin2_w, n.lin2_b = self._lin(p + "linear2")
        if i < self.L:
            n.dec_norm = self._norm(f"LSTT.decoder_norms.{i}")
        return n

    # ------------------------------------------------------------------ DeAOT block
    def _gpm_layer(self, i):
        p = f"LSTT.layers.{i}."
        sd = self.sd
        n = NS()
        n.norm1 = self._norm(p + "norm1")
        n.qv_w, n.qv_b = self._lin(p + "linear_QV")           # [C, d_att + 2C]
        n.u_w, n.u_b = self._lin(p + "linear_U")              # [C, 2C]
        n.idv_w, n.idv_b = self._lin(p + "linear_ID_V")       # layer 0: [C, 2C]; else [2C, 2C]
        if i > 0:
            n.id_norm1 = self._norm(p + "id_norm1")
            n.idu_w, n.idu_b = self._lin(p + "linear_ID_U")
        wl, bl = self._lin(p + "long_term_attn.projection")   # [4C, 2C]
        ws, bs = self._lin(p + "short_term_attn.projection")
        n.lst_proj_w = self._reg(torch.cat([wl, ws], dim=0).contiguous())  # [8C, 2C]
        n.lst_proj_b = (bl.double() + bs.double()).float().contiguous()
        n.lt_dw = self._dw_w(sd[p + "long_term_attn.dw_conv.conv.weight"])
        n.st_dw = self._dw_w(sd[p + "short_term_attn.dw_conv.conv.weight"])
        rk = sd[p + "short_term_attn.relative_emb_k.weight"]
        n.relk_w = self._f(rk.reshape(rk.shape[0], rk.shape[1]))   # [225, d_att]
        n.relk_b = self._f(sd[p + "short_term_attn.relative_emb_k.bias"])
        n.norm2 = self._norm(p + "norm2")
        n.id_norm2 = self._norm(p + "id_norm2")
        q = p + "self_attn."
        n.sa_qk_w, n.sa_qk_b = self._lin(q + "linear_QK")
        n.sa_v1 = self._lin(q + "linear_V1")
        n.sa_v2 = self._lin(q + "linear_V2")
        n.sa_u1 = self._lin(q + "linear_U1")
        n.sa_u2 = self._lin(q + "linear_U2")
        n.sa_dw = self._dw_w(sd[q + "dw_conv.conv.weight"])
        n.sa_proj_w, n.sa_proj_b = self._lin(q + "projection")
        return n

    # ------------------------------------------------------------------ decoder / id bank
    def _decoder(self):
        sd = self.sd
        p = "decoder."
        d = NS()

        def cg(name):
            cw = sd[p + name + ".conv.weight"]
            return NS(w=self._reg(self._conv_w(cw), cw.shape[1]), b=self._f(sd[p + name + ".conv.bias"]),
                      gn=self._norm(p + name + ".gn"), cout=cw.shape[0])

        d.conv_in, d.conv_16x, d.conv_8x, d.conv_4x = cg("conv_in"), cg("conv_16x"), cg("conv_8x"), cg("conv_4x")
        for a in ("adapter_16x", "adapter_8x", "adapter_4x", "conv_out"):
            cw = sd[p + a + ".weight"]
            setattr(d, a, NS(w=self._reg(self._conv_w(cw), cw.shape[1]), b=self._f(sd[p + a + ".bias"]),
                             cout=cw.shape[0]))
        self.dec = d
        if self.deaot:
            self.final_gn = self._norm("LSTT.decoder_norms.0.gn")
            self.id_norm = self._norm("id_norm")

    def _idbank(self):
        w = self.sd["patch_wise_id_bank.weight"]           # [C, 11, K, K]
        self.id_k = w.shape[2]
        self.id_stride = 16
        self.id_pad = 8 if self.align_corners else 0       # aot.py:50-63
        self.id_wt = self._conv_w(w)                        # [(ky*K+kx)*11 + id, C]
        # exclusive prefix sums along kx (float64) for the run-length gather: [K, K+1, 11, C]
        k = self.id_k
        t = w.double().permute(2, 3, 1, 0)                  # [ky, kx, id, C]
        pre = torch.zeros(k, k + 1, t.shape[2], t.shape[3], dtype=torch.float64, device=t.device)
        pre[:, 1:] = torch.cumsum(t, dim=1)
        self.id_wp = self._f(pre.float())
        self.id_b = self._f(self.sd["patch_wise_id_bank.bias"])
