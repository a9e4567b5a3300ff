"""GPU: the split-attention kernels (csrc/splat.cu) against float64 restatements of networks/encoders/resnest/splat.py and
nn.AvgPool2d, the radix-2 grouped conv as tensor-core launches on channel slices, the ResNet-101 / ResNeSt-101 encoders against
the oracle, and the R101-AOTL / RS101-AOTL engines against the real reference's goldens."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _splat_ref(x, w1, b1, w2, b2, radix=2):
    """splat.py:88-105 in float64: x [HW, radix*C] -> att [radix*C] (radix-major)."""
    x = x.double()
    C = w1.shape[0]
    gap = sum(x[:, r * C:(r + 1) * C] for r in range(radix)).mean(0)
    h = torch.relu(gap @ w1.double() + b1.double())
    logit = h @ w2.double() + b2.double()
    return torch.softmax(logit.view(radix, C), dim=0).reshape(-1)


def _splat_inputs(C, HW, seed=0):
    g = _gen(seed)
    inter = C // 2
    x = torch.relu(torch.randn(HW, 2 * C, generator=g)) + 0.1 * torch.rand(2 * C, generator=g)
    w1 = torch.randn(C, inter, generator=g) / C ** 0.5
    b1 = 0.1 * torch.randn(inter, generator=g)
    w2 = torch.randn(inter, 2 * C, generator=g) / inter ** 0.5
    b2 = 0.5 * torch.randn(2 * C, generator=g)
    return x, w1, b1, w2, b2


@pytest.mark.parametrize("C", [64, 128, 256])
@pytest.mark.parametrize("hw", [(1, 1), (3, 5), (31, 54), (121, 213)])
def test_splat_attention_vs_float64(C, hw):
    from aot_benchmark_b200 import ops
    HW = hw[0] * hw[1]
    x, w1, b1, w2, b2 = _splat_inputs(C, HW, seed=C + HW)
    want = _splat_ref(x, w1, b1, w2, b2)
    assert (want[:C] - want[C:]).abs().max().item() > 0.1                  # the two radix maps really differ
    xd = x.cuda().view(1, hw[0], hw[1], 2 * C)
    w1d, b1d, w2d, b2d = w1.cuda(), b1.cuda(), w2.cuda(), b2.cuda()
    ws = ops.splat_workspace(C, xd.device)
    att = torch.empty(2 * C, device="cuda")
    ops.splat_attention(xd, w1d, b1d, w2d, b2d, att, ws)
    a1 = att.clone()
    ops.splat_attention(xd, w1d, b1d, w2d, b2d, att, ws)
    torch.cuda.synchronize()
    assert torch.equal(a1, att)                                             # deterministic reduction
    assert (a1.cpu().double() - want).abs().max().item() < 2e-6
    g = torch.cuda.CUDAGraph()
    out = torch.zeros(2 * C, device="cuda")
    with torch.cuda.graph(g):
        ops.splat_attention(xd, w1d, b1d, w2d, b2d, out, ws)
    for _ in range(2):                                                      # the counter resets itself between replays
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, a1)


def test_splat_attention_channel_slice_input():
    """x as a channel slice of a wider NHWC buffer (ld > 2C)."""
    from aot_benchmark_b200 import ops
    C, H, W = 64, 9, 7
    x, w1, b1, w2, b2 = _splat_inputs(C, H * W, seed=5)
    big = torch.randn(1, H, W, 2 * C + 64).cuda()
    big[..., 32:32 + 2 * C] = x.view(1, H, W, 2 * C).cuda()
    att = torch.empty(2 * C, device="cuda")
    ops.splat_attention(big[..., 32:32 + 2 * C], w1.cuda(), b1.cuda(), w2.cuda(), b2.cuda(), att, ops.splat_workspace(C, "cuda"))
    assert (att.cpu().double() - _splat_ref(x, w1, b1, w2, b2)).abs().max().item() < 2e-6


@pytest.mark.parametrize("C", [64, 256])
@pytest.mark.parametrize("hw", [(31, 54), (30, 53), (1, 1), (8, 8)])
@pytest.mark.parametrize("pool", [0, 2])
def test_splat_combine(C, hw, pool):
    from aot_benchmark_b200 import ops
    H, W = hw
    g = _gen(H * W + C)
    x = torch.randn(1, H, W, 2 * C, generator=g)
    att = torch.softmax(torch.randn(2, C, generator=g), 0).reshape(-1)
    y = (att[:C].double() * x[..., :C].double() + att[C:].double() * x[..., C:].double()).permute(0, 3, 1, 2)
    want = (F.avg_pool2d(y, 3, pool, 1) if pool else y).permute(0, 2, 3, 1)
    out = torch.full(tuple(want.shape), float("nan"), device="cuda")
    ops.splat_combine(x.cuda(), att.cuda(), out, pool_stride=pool)
    assert (out.cpu().double() - want).abs().max().item() < 2e-6


@pytest.mark.parametrize("cfg", [(2, 2, 0, True, False), (3, 2, 1, False, True), (1, 1, 0, True, False)])
@pytest.mark.parametrize("hw", [(61, 107), (60, 106), (121, 213), (2, 3)])
def test_avgpool_vs_torch(cfg, hw):
    from aot_benchmark_b200 import ops
    k, s, pad, ceil, inc = cfg
    x = torch.randn(1, *hw, 256, generator=_gen(hw[0]))
    want = F.avg_pool2d(x.double().permute(0, 3, 1, 2), k, s, pad, ceil_mode=ceil, count_include_pad=inc).permute(0, 2, 3, 1)
    out = torch.full(tuple(want.shape), float("nan"), device="cuda")
    ops.avgpool(x.cuda(), out, k, s, pad, ceil_mode=ceil, count_include_pad=inc)
    assert (out.cpu().double() - want).abs().max().item() < 1e-6


@pytest.mark.parametrize("gw,hw", [(64, (41, 61)), (128, (21, 31)), (256, (11, 16))])
def test_grouped_conv_through_channel_slices(gw, hw):
    """The radix-2 grouped 3x3 conv of SplAtConv2d as one tensor-core launch per group on channel slices (input [g gw/2,
    (g+1) gw/2) with ld gw, output [g gw, (g+1) gw) with ld 2 gw) == F.conv2d(groups=2) in float64."""
    from aot_benchmark_b200 import ops
    H, W = hw
    g = _gen(gw)
    x = torch.relu(torch.randn(1, gw, H, W, generator=g))
    w = torch.randn(2 * gw, gw // 2, 3, 3, generator=g) * (2.0 / (9 * gw)) ** 0.5
    bias = 0.1 * torch.randn(2 * gw, generator=g)
    want = F.relu(F.conv2d(x.double(), w.double(), bias.double(), 1, 1, 1, 2)).permute(0, 2, 3, 1)
    xd = x.permute(0, 2, 3, 1).contiguous().cuda()
    out = torch.full((1, H, W, 2 * gw), float("nan"), device="cuda")
    keep = []
    for grp in range(2):
        wk = w[grp * gw:(grp + 1) * gw].permute(2, 3, 1, 0).reshape(9 * gw // 2, gw).contiguous().cuda()
        wh, wl, wsc = ops.split_fp16_scaled(wk)
        ops.register_tc_weights(wk, wh.cuda(), wl.cuda(), wsc.cuda())
        keep.append(wk)
        ops.conv2d(xd[..., grp * gw // 2:(grp + 1) * gw // 2], wk, bias[grp * gw:(grp + 1) * gw].cuda(),
                   out[..., grp * gw:(grp + 1) * gw], KH=3, KW=3, pad=1, act=ops.ACT_RELU)
    torch.cuda.synchronize()
    for wk in keep:
        ops._TC_WEIGHTS.pop(wk.data_ptr(), None)
    assert ops.CONV_IMPL == "tc"
    d = (out.cpu().double() - want).abs().max().item()
    assert d < 2e-5 * max(1.0, want.abs().max().item()), d


@pytest.mark.parametrize("model_name,H,W", [("rs101_aotl", 97, 131), ("rs101_aotl", 161, 241), ("rs101_aotl", 481, 849),
                                            ("r101_aotl", 161, 241)])
def test_encoder_vs_oracle(model_name, H, W):
    """Whole encoder + projector on the GPU vs the oracle (itself pinned to the reference's encoders), eager, captured and
    replayed, with the tolerance of test_swin_encoder_vs_oracle."""
    from aot_benchmark_b200 import EngineConfig, build_vos_model, engine, plan
    from oracle import resnest_oracle as RO
    sd = RO.build_state_dict(model_name, seed=0)
    cfg = EngineConfig("t", model_name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    img = torch.randn(1, 3, H, W, generator=_gen(3))
    with torch.no_grad():
        want = RO.encode_image(sd, RO.OracleConfig(model_name), img)
        enc = engine._Encoder(plan.get_plan(model), H, W)
        st = torch.cuda.current_stream().cuda_stream
        for rep in range(3):
            got = enc(img.cuda(), st)
            torch.cuda.synchronize()
            for a, b in zip(got, want):
                assert tuple(a.shape) == tuple(b.shape)
                assert (a.cpu() - b).abs().max().item() < 5e-4 * max(1.0, b.abs().max().item()), rep


@pytest.mark.parametrize("name", ["r101_aotl_small", "rs101_aotl_small"])
def test_engine_vs_reference_golden(name, golden_dir):
    from oracle import aot_oracle as O
    from oracle import resnest_oracle as RO
    from oracle import weights as OW
    from test_gpu_engine import _build_cuda_engine, _tie_band_ok
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    sd = RO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    assert OW.checksum(sd) == g["weights_checksum"], "seeded weights are not reproducible on this machine"
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    eng = _build_cuda_engine(g["model"], sd, g["gap"])
    with torch.no_grad():
        lo, labels = O.run_video(eng, [f.cuda() for f in frames], mask.cuda(), g["objs"], tuple(g["out_size"]),
                                 forced_masks=[l.float() for l in g["ref_labels"]])
    n = g["objs"] + 1
    dmax = max((a.cpu()[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(lo, g["ref_logits_lo"]))
    print(f"{name}: max |dlogit| vs the real reference = {dmax:.3e}")
    assert dmax < 1e-3, dmax
    assert _tie_band_ok(lo, g["ref_logits_lo"], labels, g["ref_labels"], tuple(g["out_size"]), n) == 0


def test_full_geometry_rs101_vs_reference_golden(golden_dir):
    """RS101-AOTL at 481x849 -> 480x854, 10 objects, gap 5 (the bank grows), teacher-forced with the reference's labels as in
    test_gpu_full_geometry.py: logits of the stored frames (every second row and column) within 1e-3; where a label differs from
    the reference's, the reference's label must score within the tie band of the engine's own top label (4 x the logit error
    + 1e-5); at most 2e-4 of all pixels differ."""
    from oracle import aot_oracle as O
    from oracle import resnest_oracle as RO
    from oracle import weights as OW
    from oracle.fixtures import load_full_labels
    from test_gpu_engine import _build_cuda_engine
    g = torch.load(os.path.join(golden_dir, "full_rs101_aotl_480p.pt"))
    sd = RO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    assert OW.checksum(sd) == g["weights_checksum"], "seeded weights are not reproducible on this machine"
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    eng = _build_cuda_engine(g["model"], sd, g["gap"])
    ref_labels = load_full_labels(g)
    with torch.no_grad():
        lo, labels = O.run_video(eng, [f.cuda() for f in frames], mask.cuda(), g["objs"], tuple(g["out_size"]),
                                 forced_masks=ref_labels)
    e0 = eng.aot_engines[0]
    assert e0.bank_len == e0.enc_hw * (1 + (g["frames"] - 1) // g["gap"])
    n, s = g["objs"] + 1, g["logit_stride"]
    dmax = 0.0
    for t in g["logit_frames"]:
        dmax = max(dmax, (lo[t - 1].cpu()[:, :n, ::s, ::s] - g["ref_logits_lo"][t][:, :n]).abs().max().item())
    print(f"rs101_aotl_480p: max |dlogit| vs the real reference = {dmax:.3e}")
    assert dmax < 1e-3, dmax
    bad = 0
    for t in range(1, g["frames"]):
        mm = labels[t - 1].cpu().to(torch.uint8) != ref_labels[t - 1].to(torch.uint8)
        if mm.any():
            up = F.interpolate(lo[t - 1].cpu()[:, :n], size=tuple(g["out_size"]), mode="bilinear", align_corners=True)
            ours = up.gather(1, labels[t - 1].cpu().long())
            theirs = up.gather(1, ref_labels[t - 1].long())
            bad += int((mm & (ours - theirs > 4 * dmax + 1e-5)).sum().item())
    assert bad == 0
    total = sum(b.numel() for b in ref_labels)
    mism = sum((a.cpu().to(torch.uint8) != b.to(torch.uint8)).sum().item() for a, b in zip(labels, ref_labels))
    assert mism <= 2e-4 * total, (mism, total)
