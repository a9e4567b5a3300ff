"""GPU: the halo path of the tensor-core conv (stride-1 3x3 convolutions on 8 x 16 pixel tiles, the input halo staged once
per 64-channel slice) against the chunked kernel it replaces.

  Cin = 64     one slice: the K order of both kernels is (ky, kx, ci), so the outputs are bitwise equal (same N tile, no
               split-K on either side).
  Cin >= 128   slice-major K order: only the fp32 summation order differs.  Both kernels are held to the conv law of
               DESIGN section 3.1 against float64 with the accumulation coefficient that section gives for convolutions
               with K > 256 (C_ACC_CONV = 16): the chunked kernel itself exceeds the attention sweeps' C_ACC = 4 on
               persistent tiles at K = 1152 and 2304.

Every eligible 3x3 shape of the R50-AOTL 480p frame, and maps whose width and height leave partial tiles on both edges, at
B = 1 and 3, split and single pass, with and without residual and ReLU.  Also: NaN outside the map (other channels of a
wider pixel stride, memory before and after the tensor) changes nothing; nothing is written outside the output; scaling
the weights by 2^k scales the output by 2^k bitwise (the per-channel weight normalisation)."""
import math
from types import SimpleNamespace

import pytest
import torch

from test_gpu_tc_envelope import DEV, _pack_w
from test_gpu_tc_operand_range import C_ACC, _ratio, conv_law, conv_restatement

pytestmark = pytest.mark.gpu

# H, W, Cin, Cout: the stride-1 3x3 convolutions of one R50-AOTL 481 x 849 frame: layers 1-3 (the FPN decoder's conv_16x
# has layer 3's shape), the decoder's conv_8x and conv_4x
FRAME = [(121, 213, 64, 64), (61, 107, 128, 128), (31, 54, 256, 256), (61, 107, 256, 128), (121, 213, 128, 128)]
# maps with partial 8 x 16 tiles at the right and bottom edges (and a map smaller than one tile); one more with
# Cout = 256 for the BN = 256 instantiations
EDGE_MAPS = [(1, 1), (7, 15), (9, 17), (31, 54), (37, 65), (121, 213)]
SHAPES = FRAME + [(h, w, c, c) for h, w in EDGE_MAPS for c in (64, 128) if (h, w, c, c) not in FRAME] + \
    [(37, 65, 256, 256)]
BN_CODE = {64: 1, 128: 2, 256: 3}
# fp32 accumulation coefficient of the conv law for K > 256 (DESIGN section 3.1)
C_ACC_CONV = 16.0


def _case(H, W, Cin, Cout, B, seed=0):
    from aot_benchmark_b200 import ops
    g = torch.Generator().manual_seed(seed + 31 * Cin + H * W)
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin)
    res = torch.randn(B, H, W, Cout, generator=g)
    bias = torch.randn(Cout, generator=g)
    wh, wl, ws = ops.split_fp16_scaled(_pack_w(w).to(DEV))
    four = lambda t: (t[:, :9 * Cin].double().cpu() * ws.double().cpu().view(-1, 1)).view(Cout, 3, 3, Cin) \
        .permute(0, 3, 1, 2).contiguous()
    return SimpleNamespace(x=x, w=w, res=res, bias=bias, wh=wh, wl=wl, ws=ws, Wh4=four(wh), Wl4=four(wl), K=3, stride=1,
                           pad=1, Cout=Cout)


def _run(c, split, halo, x=None, res=False, act=0, tiling=0, out=None, wscale=None):
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import lib
    x = c.x.to(DEV) if x is None else x
    B, H, W, _ = x.shape
    if out is None:
        out = torch.full((B, H, W, c.Cout), float("nan"), device=DEV)
    assert lib().aotb_set_conv_halo(halo) == 0 and lib().aotb_set_conv_tiling(tiling) == 0
    try:
        ops.conv2d_tc(x, c.wh, c.wl if split else None, c.bias.to(DEV) if res else None, out,
                      res=c.res.to(DEV) if res else None, KH=3, KW=3, stride=1, pad=1, act=act,
                      wscale=c.ws if wscale is None else wscale)
        torch.cuda.synchronize()
    finally:
        lib().aotb_set_conv_halo(1)
        lib().aotb_set_conv_tiling(0)
    return out


@pytest.mark.parametrize("fused", [False, True], ids=["plain", "res_relu"])
@pytest.mark.parametrize("split", [True, False], ids=["split", "single"])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_halo_against_chunked(shape, B, split, fused):
    H, W, Cin, Cout = shape
    c = _case(H, W, Cin, Cout, B)
    act = 1 if fused else 0
    if Cin == 64:
        for bn in (64, 128, 256):
            if Cout % bn:
                continue
            tiling = (BN_CODE[bn] << 4) | (1 << 8)           # same N tile, no split-K, on both kernels
            new = _run(c, split, 2, res=fused, act=act, tiling=tiling)
            old = _run(c, split, 0, res=fused, act=act, tiling=tiling)
            assert torch.equal(new, old), f"BN {bn}: max |diff| {(new - old).abs().max().item():.3e}"
    else:
        ref, tol = conv_law(c, c.x, split, dev=DEV)
        tol = tol + (C_ACC_CONV / C_ACC - 1) * conv_restatement(c, c.x, split, DEV)[1]   # C_ACC -> C_ACC_CONV
        if fused:
            # the finish adds bias and residual in fp32 and applies ReLU: one more rounding of the sum, and ReLU is
            # 1-Lipschitz
            bias, res = c.bias.double().to(DEV), c.res.double().to(DEV)
            pre = ref + bias + res
            tol = tol + 2.0 ** -23 * (pre.abs() + res.abs() + bias.abs())
            ref = torch.relu(pre)
        assert _ratio(_run(c, split, 0, res=fused, act=act), ref, tol) <= 1.0
        # the policy's N tile, and BN = 256 forced where Cout allows it (the policy rarely picks it for these maps)
        tilings = [0] + ([(BN_CODE[256] << 4) | (1 << 8)] if Cout % 256 == 0 else [])
        for tiling in tilings:
            new = _run(c, split, 2, res=fused, act=act, tiling=tiling)
            assert not new.isnan().any()
            assert _ratio(new, ref, tol) <= 1.0, f"tiling {tiling:#x}"


@pytest.mark.parametrize("split", [True, False], ids=["split", "single"])
@pytest.mark.parametrize("shape", [(37, 65, 64, 64), (37, 65, 128, 128)], ids=lambda s: "x".join(map(str, s)))
def test_halo_nan_outside_map_and_no_stray_writes(shape, split):
    H, W, Cin, Cout = shape
    B = 3
    c = _case(H, W, Cin, Cout, B, seed=5)
    ref = _run(c, split, 2, res=True, act=1)
    # the input inside a NaN buffer: 64 more channels per pixel, and NaN before and after the tensor
    ld, pad = Cin + 64, 4096
    buf = torch.full((2 * pad + B * H * W * ld,), float("nan"), device=DEV)
    xin = buf[pad:pad + B * H * W * ld].view(B, H, W, ld)[..., :Cin]
    xin.copy_(c.x.to(DEV))
    # the output inside a sentinel buffer: 64 more channels per pixel, and guard zones before and after
    sentinel = 1234.5
    obuf = torch.full((2 * pad + B * H * W * (Cout + 64),), sentinel, device=DEV)
    out = obuf[pad:pad + B * H * W * (Cout + 64)].view(B, H, W, Cout + 64)[..., :Cout]
    _run(c, split, 2, x=xin, res=True, act=1, out=out)
    assert torch.equal(out, ref)
    assert (obuf[:pad] == sentinel).all() and (obuf[-pad:] == sentinel).all()
    assert (obuf[pad:pad + B * H * W * (Cout + 64)].view(B, H, W, Cout + 64)[..., Cout:] == sentinel).all()


@pytest.mark.parametrize("k", [-20, -3, 5, 30])
@pytest.mark.parametrize("split", [True, False], ids=["split", "single"])
def test_halo_weight_scale_equivariance(split, k):
    from aot_benchmark_b200 import ops
    c = _case(37, 65, 128, 128, 1, seed=9)
    base = _run(c, split, 2)
    wh, wl, ws = ops.split_fp16_scaled(_pack_w(c.w * 2.0 ** k).to(DEV))
    assert torch.equal(wh, c.wh) and torch.equal(wl, c.wl)
    scaled = _run(c, split, 2, wscale=ws)
    assert torch.equal(scaled, base * 2.0 ** k)


def test_halo_setter_rejects_bad_mode():
    from aot_benchmark_b200._lib import lib
    assert lib().aotb_set_conv_halo(3) != 0
    assert lib().aotb_set_conv_halo(-1) != 0
    assert lib().aotb_set_conv_halo(1) == 0
