"""GPU: the squeeze-excite kernels (aotb_se_gate_f32, aotb_gate_scale_f32) and h_swish in the fp32 conv and depthwise conv
against float64 restatements of networks/encoders/mobilenetv3.py, the MobileNetV3-Large and ResNeSt-50 encoders against the
oracle, and the AOTL + MobileNetV3 / R50-AOTL + ResNeSt-50 engines against the real reference's goldens."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

MBV3, RS50 = "AOTL with mobilenetv3", "R50-AOTL with resnest50"
SE_WIDTHS = [(72, 24), (120, 32), (480, 120), (672, 168), (960, 240)]     # SELayer(C): _make_divisible(C // 4, 8)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _hswish64(v):
    return v * F.relu6(v + 3) / 6


def _se_ref(x, w1, b1, w2, b2):
    """SELayer.fc(avg_pool(x)) (mobilenetv3.py:61-65) in float64: x [HW, C] -> gate [C]."""
    x = x.double()
    h = torch.relu(x.mean(0) @ w1.double() + b1.double())
    return F.relu6(h @ w2.double() + b2.double() + 3) / 6


def _se_inputs(C, inter, HW, seed):
    g = _gen(seed)
    x = torch.randn(HW, C, generator=g) + 0.5 * torch.randn(C, generator=g)
    w1 = torch.randn(C, inter, generator=g) * (2.0 / C) ** 0.5
    b1 = 0.1 * torch.randn(inter, generator=g)
    w2 = torch.randn(inter, C, generator=g) * 3.0 / inter ** 0.5
    b2 = 0.5 * torch.randn(C, generator=g)
    return x, w1, b1, w2, b2


@pytest.mark.parametrize("C,inter", SE_WIDTHS)
@pytest.mark.parametrize("hw", [(1, 1), (3, 5), (31, 54), (121, 213)])
def test_se_gate_vs_float64(C, inter, hw):
    from aot_benchmark_b200 import ops
    HW = hw[0] * hw[1]
    x, w1, b1, w2, b2 = _se_inputs(C, inter, HW, seed=C + HW)
    want = _se_ref(x, w1, b1, w2, b2)
    if HW > 1:
        assert want.max().item() - want.min().item() > 0.4               # the gates spread over (0, 1)
    xd = x.cuda().view(1, hw[0], hw[1], C)
    w1d, b1d, w2d, b2d = w1.cuda(), b1.cuda(), w2.cuda(), b2.cuda()
    ws = ops.splat_workspace(C, xd.device)
    gate = torch.empty(C, device="cuda")
    ops.se_gate(xd, w1d, b1d, w2d, b2d, gate, ws)
    g1 = gate.clone()
    ops.se_gate(xd, w1d, b1d, w2d, b2d, gate, ws)
    torch.cuda.synchronize()
    assert torch.equal(g1, gate)                                            # deterministic reduction
    assert (g1.cpu().double() - want).abs().max().item() < 2e-6
    graph = torch.cuda.CUDAGraph()
    out = torch.zeros(C, device="cuda")
    with torch.cuda.graph(graph):
        ops.se_gate(xd, w1d, b1d, w2d, b2d, out, ws)
    for _ in range(2):                                                      # the counter resets itself between replays
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, g1)


def test_se_gate_channel_slice_input():
    """x as a channel slice of a wider NHWC buffer (ld > C)."""
    from aot_benchmark_b200 import ops
    C, inter, H, W = 120, 32, 9, 7
    x, w1, b1, w2, b2 = _se_inputs(C, inter, H * W, seed=5)
    big = torch.randn(1, H, W, C + 64).cuda()
    big[..., 32:32 + C] = x.view(1, H, W, C).cuda()
    gate = torch.empty(C, device="cuda")
    ops.se_gate(big[..., 32:32 + C], w1.cuda(), b1.cuda(), w2.cuda(), b2.cuda(), gate, ops.splat_workspace(C, "cuda"))
    assert (gate.cpu().double() - _se_ref(x, w1, b1, w2, b2)).abs().max().item() < 2e-6


@pytest.mark.parametrize("C", [72, 960])
@pytest.mark.parametrize("hw", [(1, 1), (31, 54), (61, 107)])
@pytest.mark.parametrize("act", ["relu", "hswish"])
@pytest.mark.parametrize("sliced", [False, True])
def test_gate_scale_vs_float64(C, hw, act, sliced):
    from aot_benchmark_b200 import ops
    H, W = hw
    g = _gen(C + H * W)
    x = 3 * torch.randn(1, H, W, C, generator=g)
    gate = torch.rand(C, generator=g)
    y = gate.double() * x.double()
    want = F.relu(y) if act == "relu" else _hswish64(y)
    code = ops.ACT_RELU if act == "relu" else ops.ACT_HSWISH
    if sliced:
        xb = torch.randn(1, H, W, C + 8).cuda()
        xb[..., 4:4 + C] = x.cuda()
        ob = torch.full((1, H, W, C + 16), float("nan"), device="cuda")
        xd, out = xb[..., 4:4 + C], ob[..., 8:8 + C]
    else:
        xd, out = x.cuda(), torch.full((1, H, W, C), float("nan"), device="cuda")
    ops.gate_scale(xd, gate.cuda(), out, act=code)
    torch.cuda.synchronize()
    assert (out.cpu().double() - want).abs().max().item() < 1e-6 * max(1.0, want.abs().max().item())
    if sliced:
        assert torch.isnan(ob[..., :8]).all() and torch.isnan(ob[..., 8 + C:]).all()


def test_hswish_is_the_reference_expression():
    """gate_scale with h_swish computes (g * x) * (relu6(g * x + 3) / 6) in fp32 with a true division: bit-identical to the
    reference's x * y followed by h_swish, written out in float32 on the GPU with explicit rounding steps."""
    from aot_benchmark_b200 import ops
    g = _gen(11)
    x = (8 * torch.randn(1, 33, 47, 960, generator=g)).cuda()
    gate = torch.rand(960, generator=g).cuda()
    out = torch.empty_like(x)
    ops.gate_scale(x, gate, out, act=ops.ACT_HSWISH)
    y = x * gate
    six = torch.full_like(y, 6.0)
    want = y * torch.div(torch.clamp(y + 3, 0, 6), six)                      # tensor / tensor: a true division
    torch.cuda.synchronize()
    assert torch.equal(out, want)


@pytest.mark.parametrize("cin,cout,k,stride,hw", [(4, 16, 3, 2, (97, 131)), (160, 960, 1, 1, (31, 54)),
                                                  (80, 480, 1, 1, (30, 53)), (24, 72, 1, 1, (61, 107))])
def test_hswish_in_simt_conv2d_vs_float64(cin, cout, k, stride, hw):
    """h_swish in the fp32 CUDA-core conv finish (weights not registered for the tensor cores)."""
    from aot_benchmark_b200 import ops
    H, W = hw
    g = _gen(cin * cout)
    x = torch.randn(1, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    b = torch.randn(cout, generator=g)
    want = _hswish64(F.conv2d(x.double(), w.double(), b.double(), stride, k // 2)).permute(0, 2, 3, 1)
    wk = w.permute(2, 3, 1, 0).reshape(k * k * cin, cout).contiguous().cuda()
    assert wk.data_ptr() not in ops._TC_WEIGHTS
    out = torch.full(tuple(want.shape), float("nan"), device="cuda")
    ops.conv2d(x.permute(0, 2, 3, 1).contiguous().cuda(), wk, b.cuda(), out, KH=k, KW=k, stride=stride, pad=k // 2,
               act=ops.ACT_HSWISH)
    torch.cuda.synchronize()
    assert (out.cpu().double() - want).abs().max().item() < 2e-5 * max(1.0, want.abs().max().item())


@pytest.mark.parametrize("C,K,stride,dil,hw", [(72, 5, 2, 1, (61, 107)), (960, 5, 1, 2, (31, 54)), (120, 5, 1, 1, (30, 53)),
                                               (240, 3, 2, 1, (61, 107)), (200, 3, 1, 1, (31, 54))])
def test_hswish_in_dwconv_vs_float64(C, K, stride, dil, hw):
    """The depthwise shapes of MobileNetV3 (5x5 stride 2, 5x5 dilation 2 pad 4, the 5x5 stride-1 row kernel, 3x3) with h_swish."""
    from aot_benchmark_b200 import ops
    H, W = hw
    pad = (K - 1) // 2 * dil
    g = _gen(C + K)
    x = torch.randn(1, C, H, W, generator=g)
    w = torch.randn(C, 1, K, K, generator=g) * (2.0 / (K * K)) ** 0.5
    b = torch.randn(C, generator=g)
    want = _hswish64(F.conv2d(x.double(), w.double(), b.double(), stride, pad, dil, C)).permute(0, 2, 3, 1)
    out = torch.full(tuple(want.shape), float("nan"), device="cuda")
    ops.dwconv(x.permute(0, 2, 3, 1).contiguous().cuda(), w.permute(2, 3, 1, 0).reshape(K * K, C).contiguous().cuda(),
               b.cuda(), out, K=K, stride=stride, pad=pad, dil=dil, act=ops.ACT_HSWISH)
    torch.cuda.synchronize()
    assert (out.cpu().double() - want).abs().max().item() < 2e-5 * max(1.0, want.abs().max().item())


def _cuda_engine(case, sd, gap):
    from aot_benchmark_b200 import build_engine, build_vos_model
    from oracle import mobilenetv3_oracle as MO
    cfg = MO.engine_config(case, "t")
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    return build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                        short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP).eval()


@pytest.mark.parametrize("case,H,W", [(MBV3, 97, 131), (MBV3, 481, 849), (RS50, 97, 131), (RS50, 161, 241)])
def test_encoder_vs_oracle(case, H, W):
    """Whole encoder + projector on the GPU vs the oracle (itself pinned to the reference's encoders), eager, captured and
    replayed, with the tolerance of test_gpu_resnest.test_encoder_vs_oracle."""
    from aot_benchmark_b200 import build_vos_model, engine, plan
    from oracle import mobilenetv3_oracle as MO
    sd = MO.build_state_dict(case, seed=0)
    cfg = MO.engine_config(case, "t")
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    img = torch.randn(1, 3, H, W, generator=_gen(3))
    with torch.no_grad():
        want = MO.encode_image(sd, MO.OracleConfig(case), img)
        enc = engine._Encoder(plan.get_plan(model), H, W)
        st = torch.cuda.current_stream().cuda_stream
        for rep in range(3):
            got = enc(img.cuda(), st)
            torch.cuda.synchronize()
            for a, b in zip(got, want):
                assert tuple(a.shape) == tuple(b.shape)
                assert (a.cpu() - b).abs().max().item() < 5e-4 * max(1.0, b.abs().max().item()), rep


@pytest.mark.parametrize("name", ["aotl_mbv3_small", "rs50_aotl_small"])
def test_engine_vs_reference_golden(name, golden_dir):
    from oracle import aot_oracle as O
    from oracle import mobilenetv3_oracle as MO
    from oracle import weights as OW
    from test_gpu_engine import _tie_band_ok
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    sd = MO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    assert OW.checksum(sd) == g["weights_checksum"], "seeded weights are not reproducible on this machine"
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    eng = _cuda_engine(g["model"], sd, g["gap"])
    with torch.no_grad():
        lo, labels = O.run_video(eng, [f.cuda() for f in frames], mask.cuda(), g["objs"], tuple(g["out_size"]),
                                 forced_masks=[l.float() for l in g["ref_labels"]])
    n = g["objs"] + 1
    dmax = max((a.cpu()[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(lo, g["ref_logits_lo"]))
    print(f"{name}: max |dlogit| vs the real reference = {dmax:.3e}")
    assert dmax < 1e-3, dmax
    assert _tie_band_ok(lo, g["ref_logits_lo"], labels, g["ref_labels"], tuple(g["out_size"]), n) == 0


def test_full_geometry_mbv3_vs_reference_golden(golden_dir):
    """AOTL + MobileNetV3 at 481x849 -> 480x854, 10 objects, gap 5 (the bank grows), teacher-forced with the reference's labels
    as test_gpu_resnest.test_full_geometry_rs101_vs_reference_golden checks RS101-AOTL."""
    from oracle import aot_oracle as O
    from oracle import mobilenetv3_oracle as MO
    from oracle import weights as OW
    from oracle.fixtures import load_full_labels
    g = torch.load(os.path.join(golden_dir, "full_aotl_mbv3_480p.pt"))
    sd = MO.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    assert OW.checksum(sd) == g["weights_checksum"], "seeded weights are not reproducible on this machine"
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    eng = _cuda_engine(g["model"], sd, g["gap"])
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
    print(f"aotl_mbv3_480p: max |dlogit| vs the real reference = {dmax:.3e}")
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


def test_kernels_without_hswish_reject_it():
    """The tensor-core conv and GroupNorm do not implement activation 5: they refuse it instead of skipping it."""
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import AotbError
    x = torch.randn(1, 8, 8, 64, device="cuda")
    wh = torch.zeros(64, 64, dtype=torch.float16, device="cuda")
    out = torch.empty(1, 8, 8, 64, device="cuda")
    with pytest.raises(AotbError, match="activation"):
        ops.conv2d_tc(x, wh, wh.clone(), None, out, act=ops.ACT_HSWISH)
    with pytest.raises(AotbError, match="activation"):
        ops.groupnorm(x.view(1, 64, 64), torch.ones(64, device="cuda"), torch.zeros(64, device="cuda"), out.view(1, 64, 64), 16,
                      ops.ACT_HSWISH, ops.groupnorm_workspace(1, 16, x.device))
