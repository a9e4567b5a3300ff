"""GPU: the warp-specialised tensor-core conv at every N tile.

- Without split-K the MMA order per output element (chunks, k-steps, Ah Wh / Al Wh / Ah Wl) does not depend on the N tile,
  so BN = 64, 128 and 256 give bitwise equal outputs: on shapes of an R50-AOTL frame (scaled down where large) and on the
  envelope's tiling cases.
- BN = 256 at every split-K cluster size stays within the fp32-accumulation bound of the float64 reference, is bitwise
  reproducible and writes nothing outside its output columns."""
import math

import pytest
import torch

import test_gpu_tc_envelope as EV

pytestmark = pytest.mark.gpu

DEV = EV.DEV

# B, H, W, Cin, Cout, K, stride, pad, residual ("" | "res" | "alias"), act, wide (ldin / ldout / ldres wider than C)
FRAME_CASES = [
    (1, 31, 54, 256, 256, 3, 1, 1, "", 1, False),        # layer3 3x3 at 480p (M = 1674)
    (1, 31, 54, 1024, 256, 1, 1, 0, "", 1, False),       # layer3 1x1 reduce
    (1, 30, 53, 64, 256, 1, 1, 0, "res", 1, False),      # layer1 1x1 expand with the block's residual, scaled down
    (1, 21, 27, 128, 512, 1, 1, 0, "alias", 1, True),    # layer2 1x1 expand, residual aliasing a channel slice
    (1, 300, 1, 256, 1024, 1, 1, 0, "", 2, False),       # LSTT linear 256 -> 1024 with GELU
    (1, 23, 37, 256, 256, 3, 2, 1, "res", 0, False),     # stride-2 3x3
    (1, 17, 19, 12, 256, 3, 1, 1, "res", 4, True),       # general Cin (12 x 9 = 108)
]
ALL_CASES = FRAME_CASES + EV.TILING_CASES
IDS = [f"frame{i}" for i in range(len(FRAME_CASES))] + [f"c{i}" for i in range(len(EV.TILING_CASES))]


class _Case:
    def __init__(self, case):
        from aot_benchmark_b200 import ops
        B, H, W, Cin, Cout, K, stride, pad, rmode, act, wide = case
        self.case = case
        g = torch.Generator().manual_seed(H * 197 + W * 7 + Cin + Cout)
        self.x = torch.randn(B, H, W, Cin, generator=g) * 2
        self.w = torch.randn(Cout, Cin, K, K, generator=g) / math.sqrt(Cin * K * K)
        self.b = torch.randn(Cout, generator=g)
        Ho, Wo = (H + 2 * pad - K) // stride + 1, (W + 2 * pad - K) // stride + 1
        self.r = torch.randn(B, Ho, Wo, Cout, generator=g) if rmode else None
        self.ex = 8 if wide else 0
        xg = torch.zeros(B, H, W, Cin + self.ex, device=DEV)
        xg[..., :Cin] = self.x.to(DEV)
        self.xv = xg[..., :Cin]
        self.wh, self.wl, self.ws = ops.split_fp16_scaled(EV._pack_w(self.w).to(DEV))
        self.obuf = torch.full((B, Ho, Wo, Cout + 2 * self.ex), float("nan"), device=DEV)
        self.out = self.obuf[..., self.ex:self.ex + Cout]
        self.rbuf = None
        if rmode == "res":
            self.rbuf = torch.full((B, Ho, Wo, Cout + self.ex), float("nan"), device=DEV)
            self.rbuf[..., :Cout] = self.r.to(DEV)
        self.nchunks = (K * K * Cin + 63) // 64

    def run(self, bn_code, S):
        from aot_benchmark_b200 import ops
        from aot_benchmark_b200._lib import lib
        B, H, W, Cin, Cout, K, stride, pad, rmode, act, wide = self.case
        assert lib().aotb_set_conv_tiling((bn_code << 4) | (S << 8)) == 0
        try:
            self.obuf.fill_(float("nan"))
            if rmode == "alias":
                self.out.copy_(self.r.to(DEV))
            res = self.out if rmode == "alias" else (None if self.rbuf is None else self.rbuf[..., :Cout])
            ops.conv2d_tc(self.xv, self.wh, self.wl, self.b.to(DEV), self.out, res=res, KH=K, KW=K, stride=stride,
                          pad=pad, act=act, wscale=self.ws)
            torch.cuda.synchronize()
        finally:
            lib().aotb_set_conv_tiling(0)
        return self.obuf.clone()


WIDE_CASES = [(c, i) for c, i in zip(ALL_CASES, IDS) if c[4] % 128 == 0]


@pytest.mark.parametrize("case", [c for c, _ in WIDE_CASES], ids=[i for _, i in WIDE_CASES])
def test_unsplit_outputs_equal_across_n_tiles(case):
    c = _Case(case)
    Cout, ex = case[4], c.ex
    outs = {BN: c.run(code, 1) for code, BN in ((1, 64), (2, 128), (3, 256)) if Cout % BN == 0}
    base = outs[64][..., ex:ex + Cout]
    assert not torch.isnan(base).any()
    for BN, o in outs.items():
        got = o[..., ex:ex + Cout]
        assert torch.equal(got, base), f"BN {BN} differs from BN 64: max |d| = {(got - base).abs().max().item():.3e}"
        assert torch.isnan(o[..., :ex]).all() and torch.isnan(o[..., ex + Cout:]).all(), f"BN {BN}: wrote outside its columns"


@pytest.mark.parametrize("case", [c for c in ALL_CASES if c[4] % 256 == 0],
                         ids=[i for c, i in zip(ALL_CASES, IDS) if c[4] % 256 == 0])
def test_n256_every_split(case):
    c = _Case(case)
    B, H, W, Cin, Cout, K, stride, pad, rmode, act, wide = case
    ref = EV._ref_conv(c.x, c.w, c.b, stride, pad, c.r, act)
    scale = ref.abs().max().item()
    ex = c.ex
    tried = 0
    for S in (1, 2, 4, 8):
        if S > c.nchunks:
            continue
        runs = [c.run(3, S) for _ in range(2)]
        err = (runs[0][..., ex:ex + Cout].double().cpu() - ref).abs().max().item()
        assert err < 1e-5 * max(scale, 1.0) + 1e-5, f"S {S}: err {err:.3e} (scale {scale:.2f})"
        assert torch.equal(runs[0][..., ex:ex + Cout], runs[1][..., ex:ex + Cout]), f"S {S}: not reproducible"
        for o in runs:
            assert torch.isnan(o[..., :ex]).all() and torch.isnan(o[..., ex + Cout:]).all(), f"S {S}: wrote outside its columns"
        tried += 1
    assert tried >= 1
