"""CPU: the per-output-channel power-of-two normalisation of the split-fp16 tensor-core weights (ops.split_fp16_scaled), and
a float64 model of the kernels' three-product sum that shows why it is needed: lo = fp16(w - hi) cannot go below the fp16
subnormal spacing 2^-24, so without the normalisation a small channel hits an absolute error floor."""
import numpy as np
import pytest
import torch

from aot_benchmark_b200 import ops


def _weights(K=2304, N=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(K, N, generator=g, dtype=torch.float64).mul(torch.logspace(-4, -1, N, dtype=torch.float64)).float()


def _unsplit(hi, lo, K):
    """[N, Kpad] fp16 pair -> fp64 [K, N] value carried by the split."""
    return (hi.double() + lo.double())[:, :K].t()


@pytest.mark.parametrize("K,N", [(2304, 64), (196, 128), (1024, 256)])
def test_scale_exponents(K, N):
    w = _weights(K, N, seed=K)
    w[:, 3] = 0.0
    w[:, 4] = 2.0 ** 13                                   # already in range: scale 1
    w[:, 5] = -(2.0 ** 14)                                # exactly a power of two on the boundary
    hi, lo, ws = ops.split_fp16_scaled(w)
    assert ws.dtype == torch.float32 and ws.shape == (N,)
    assert hi.shape == lo.shape == (N, (K + 63) // 64 * 64) and hi.dtype == lo.dtype == torch.float16
    m, e = np.frexp(ws.numpy())
    assert (m == 0.5).all(), "every scale is a power of two"
    assert ws[3] == 1.0 and ws[4] == 1.0 and ws[5] == 2.0
    # the normalised weights w' = w / wscale: per-channel max |w'| in [2^13, 2^14) except the zero column
    wn = w.double() / ws.double()
    amax = wn.abs().amax(0)
    nz = amax > 0
    assert ((amax[nz] >= 2.0 ** 13) & (amax[nz] < 2.0 ** 14)).all()
    assert not nz[3] and nz.sum() == N - 1
    # w' * wscale == w bitwise (fp32), and hi never overflows
    assert torch.equal(wn.float() * ws, w)
    assert torch.isfinite(hi.float()).all() and hi.float().abs().max() <= 2.0 ** 14
    # hi + lo carries w' to 2^-22 relative of each channel's maximum
    err = (_unsplit(hi, lo, K) - wn).abs().amax(0)
    assert (err[nz] <= amax[nz] * 2.0 ** -22).all()
    assert (hi[3].float() == 0).all() and (lo[3].float() == 0).all()


def test_unscaled_split_is_unchanged():
    """split_fp16_scaled of a channel already in [2^13, 2^14) is split_fp16 bit for bit (scale 1)."""
    w = _weights(640, 64) / _weights(640, 64).abs().amax(0) * 1.5 * 2.0 ** 13
    hi0, lo0 = ops.split_fp16(w)
    hi, lo, ws = ops.split_fp16_scaled(w)
    assert (ws == 1.0).all() and torch.equal(hi, hi0) and torch.equal(lo, lo0)


def _model(a, w, scaled):
    """float64 model of the tensor-core GEMM: Ah Wh + Al Wh + Ah Wl with exact products and sums, times wscale."""
    K = a.shape[1]
    ah = a.half()
    al = (a - ah.float()).half()
    if scaled:
        wh, wl, ws = ops.split_fp16_scaled(w)
    else:
        (wh, wl), ws = ops.split_fp16(w), torch.ones(w.shape[1])
    wh, wl = wh.double()[:, :K].t(), wl.double()[:, :K].t()
    acc = ah.double() @ wh + al.double() @ wh + ah.double() @ wl
    return acc * ws.double()


def test_three_product_model_small_channels():
    """Channels with rms 1e-4 .. 1e-1 (FrozenBN folding can make single channels that small): with the normalisation
    every channel is within 2e-6 of its own max |ref|; without it the smallest one is worse than 1e-5."""
    w = _weights()
    g = torch.Generator().manual_seed(1)
    a = torch.randn(128, w.shape[0], generator=g)
    ref = a.double() @ w.double()
    scale = ref.abs().amax(0)
    err_s = ((_model(a, w, True) - ref).abs().amax(0) / scale)
    err_u = ((_model(a, w, False) - ref).abs().amax(0) / scale)
    assert err_s.max() < 2e-6, err_s.max()
    assert err_u[0] > 1e-5, err_u[0]                      # rms 1e-4: the absolute floor of lo
    assert err_u[-1] < 2e-6                               # rms 1e-1: fine either way
