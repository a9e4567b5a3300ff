"""CPU: a float32 / float64 restatement of the GroupNorm statistics of csrc/norm.cu (groupnorm_stats_kernel and the finaliser
run by its last block), in the kernel's own order, and the precision it gives when a group's mean is large next to its
standard deviation.

The order modelled:
- launch: chunks = ceil(P * Cg/4 / 1024), rounded up to a multiple of 8 and clamped to [8, 64]; chunk k covers pixels
  [k * per, min(P, (k + 1) * per)) with per = ceil(P / chunks), so chunks past the end of a small map are empty;
- 256 threads per block; thread t takes float4 number t, t + 256, ... of the chunk's (pixel, channel quad) sequence and
  accumulates in fp32 s += (x + y) + (z + w) and q += fma(x, x, y*y) + fma(z, z, w*w) (nvcc fuses the first product);
- per warp, an fp32 xor butterfly over offsets 16, 8, 4, 2, 1 (lane 0's value); per block, the 8 warp sums added in order in
  fp64;
- finaliser, fp64: 8 threads per group each add chunks / 8 consecutive chunk partials in order, then an xor tree over 1, 2, 4.

The one-pass form (the kernel before the shift) sums the raw values and forms var = E[v^2] - mean^2.  The shifted form (the
kernel now) sums v - K and (v - K)^2 with K the group's first element, and forms mean = K + S/n, var = Q/n - (S/n)^2.
"""
import numpy as np
import pytest

EPS = float(np.float32(1e-5))          # the kernel passes eps as a float and widens it to double
U = 2.0 ** -23                         # fp32 unit roundoff x 2

# Output tolerance, per element (the same bound tests/test_gpu_simt_envelope.py applies to the kernel):
#   |y - y64| <= C1 * ulp(|mean|) * rstd * |gamma| + C2 * 2^-23 * ((|x - mean| * rstd + 1) * |gamma| + |beta|)
# C1 = 1: the mean is finalised in fp64 and rounded once to fp32: half an ulp, and as much again for margin;
# C2 = 8: the apply step rounds v - mean, the product with rstd and the fused gamma / beta step (half an ulp each); rstd
#         carries a few ulps from the fp32 sums of squares, and the fp32 sum of v - K gives the mean an error relative to
#         |K - mean|, a few standard deviations (the "+ 1": one standard deviation times rstd).
C1, C2 = 1.0, 8.0


def launch_chunks(P, Cg):
    chunks = -(-(P * (Cg // 4)) // 1024)
    chunks = -(-chunks // 8) * 8
    return min(max(chunks, 8), 64)


def _fma(a, b, c):
    """fp32 a * b + c with one rounding (the product of two fp32 numbers is exact in fp64)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def _thread_sums(terms, n):
    """fp32 per-thread sums of `terms` [n] (thread t adds terms t, t + 256, ...), then lane 0 of each warp's xor butterfly,
    then the block's fp64 sum of its 8 warps in order."""
    J = -(-n // 256)
    pad = np.zeros(J * 256, np.float32)
    pad[:n] = terms
    acc = np.zeros(256, np.float32)
    for j in range(J):                 # adding the zero padding is exact
        acc = acc + pad[j * 256:(j + 1) * 256]
    w = acc.reshape(8, 32)
    for o in (16, 8, 4, 2, 1):
        w = w + w[:, np.arange(32) ^ o]
    blk = 0.0
    for wi in range(8):
        blk += float(w[wi, 0])
    return blk


def model_stats(xg, shifted):
    """xg float32 [P, Cg], one (batch, group) -> (mean, rstd) as float32, computed as the kernel does."""
    P, Cg = xg.shape
    Cg4 = Cg // 4
    chunks = launch_chunks(P, Cg)
    per = -(-P // chunks)
    K = xg[0, 0] if shifted else np.float32(0.0)
    d = (xg - K).astype(np.float32).reshape(P * Cg4, 4)
    e_s = (d[:, 0] + d[:, 1]) + (d[:, 2] + d[:, 3])
    e_q = _fma(d[:, 0], d[:, 0], d[:, 1] * d[:, 1]) + _fma(d[:, 2], d[:, 2], d[:, 3] * d[:, 3])
    part = np.zeros((chunks, 2))
    for k in range(chunks):
        p0, p1 = k * per, min(P, k * per + per)
        n = max(p1 - p0, 0) * Cg4
        i0 = p0 * Cg4
        part[k] = (_thread_sums(e_s[i0:i0 + n], n), _thread_sums(e_q[i0:i0 + n], n))
    cps = chunks // 8
    sub = [[0.0, 0.0] for _ in range(8)]
    for s in range(8):
        for c in range(cps):
            sub[s][0] += part[s * cps + c, 0]
            sub[s][1] += part[s * cps + c, 1]
    for o in (1, 2, 4):
        sub = [[sub[i][0] + sub[i ^ o][0], sub[i][1] + sub[i ^ o][1]] for i in range(8)]
    ss, qq = sub[0]
    nn = float(P * Cg)
    dm = ss / nn
    var = max(qq / nn - dm * dm, 0.0)
    return np.float32(float(K) + dm), np.float32(1.0 / np.sqrt(var + EPS))


def model_apply(xg, mean, rstd, gamma, beta):
    """fp32 apply step: fma((v - mean) * rstd, gamma, beta)."""
    return _fma((xg - mean) * rstd, gamma, beta)


def reference(xg, gamma, beta):
    x = xg.astype(np.float64)
    mean = x.mean()
    rstd = 1.0 / np.sqrt(((x - mean) ** 2).mean() + EPS)
    return (x - mean) * rstd * gamma + beta, mean, rstd


def tolerance(xg, mean, rstd, gamma, beta):
    g = np.abs(gamma.astype(np.float64))
    ulp = float(np.spacing(np.float32(abs(mean))))
    return C1 * ulp * rstd * g + C2 * U * ((np.abs(xg.astype(np.float64) - mean) * rstd + 1.0) * g + np.abs(beta))


# (P, Cg): the three engine sites on the 31 x 54 / 121 x 213 maps, a map smaller than the chunk count, and one pixel
CONFIGS = [
    (1674, 32),        # FFN GroupNorm(32, 1024): 16 chunks
    (25773, 16),       # decoder conv_4x GroupNorm(8, 128): 64 chunks
    (1674, 256),       # final GroupNorm1D(512, groups=2): 64 chunks
    (5, 32),           # P < 8: three of the 8 chunks are empty
    (7, 4),            # P < 8 with one float4 per pixel
    (1, 4),            # one pixel, four channels: one thread of one chunk
    (1, 256),
]


def _case(P, Cg, offset, seed):
    rng = np.random.default_rng(seed)
    sigma = 1.5
    xg = (sigma * (rng.standard_normal((P, Cg)) + offset)).astype(np.float32)
    gamma = rng.standard_normal(Cg).astype(np.float32)
    beta = rng.standard_normal(Cg).astype(np.float32)
    return xg, gamma, beta


def _worst(xg, gamma, beta, shifted):
    """max over the group of |y - y64| / tolerance, and max |y - y64|."""
    mean, rstd = model_stats(xg, shifted)
    y = model_apply(xg, mean, rstd, gamma, beta)
    ref, m64, r64 = reference(xg, gamma, beta)
    err = np.abs(y.astype(np.float64) - ref)
    return (err / tolerance(xg, m64, r64, gamma, beta)).max(), err.max()


@pytest.mark.parametrize("P,Cg", CONFIGS)
def test_launch_rule(P, Cg):
    chunks = launch_chunks(P, Cg)
    assert chunks % 8 == 0 and 8 <= chunks <= 64
    per = -(-P // chunks)
    covered = sum(max(min(P, k * per + per) - k * per, 0) for k in range(chunks))
    assert covered == P


@pytest.mark.parametrize("offset", [0, 10, 30, 100, 1000])
@pytest.mark.parametrize("P,Cg", CONFIGS)
def test_shifted_sums_hold_the_tolerance(P, Cg, offset):
    xg, gamma, beta = _case(P, Cg, offset, seed=P * 7 + Cg + offset)
    ratio, err = _worst(xg, gamma, beta, shifted=True)
    assert ratio <= 1.0, (ratio, err)


@pytest.mark.parametrize("P,Cg", CONFIGS)
def test_one_pass_sums_hold_the_tolerance_near_zero_mean(P, Cg):
    """Without an offset the two forms are the same computation, and the tolerance is not the thing that fails below."""
    xg, gamma, beta = _case(P, Cg, 0, seed=P * 7 + Cg)
    assert _worst(xg, gamma, beta, shifted=False)[0] <= 1.0


@pytest.mark.parametrize("offset", [100, 1000])
@pytest.mark.parametrize("P,Cg", CONFIGS)
def test_one_pass_sums_fail_at_large_mean(P, Cg, offset):
    """The one-pass E[v^2] - mean^2 cancels: at mean / std = 100 and 1000 it misses the tolerance in every configuration."""
    xg, gamma, beta = _case(P, Cg, offset, seed=P * 7 + Cg + offset)
    ratio, err = _worst(xg, gamma, beta, shifted=False)
    assert ratio > 1.0, (ratio, err)


def test_shift_pivot_is_the_first_element_of_the_group():
    """With the shift equal to every value (a constant group) the sums are exactly zero: mean is the value, rstd is
    1/sqrt(eps), and the output is beta to the bit."""
    xg = np.full((1674, 32), 1234.5, np.float32)
    mean, rstd = model_stats(xg, shifted=True)
    assert mean == np.float32(1234.5) and rstd == np.float32(1.0 / np.sqrt(EPS))
    gamma, beta = np.ones(32, np.float32), np.linspace(-1, 1, 32).astype(np.float32)
    assert np.array_equal(model_apply(xg, mean, rstd, gamma, beta), beta[None, :].repeat(1674, 0))
