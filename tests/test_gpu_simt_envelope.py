"""GPU: the fp32 CUDA-core kernels at the edges of their envelope -- GroupNorm and LayerNorm (norm.cu), the SIMT attention and
its split-KV merge (attention_simt.cu), the three short-term local attention kernels (local_attn.cu) and the NHWC helpers
(elementwise.cu).  Every case compares against a float64 restatement.  Kernels that only move data or take maxima are compared
bit for bit; the others against a tolerance derived from the case's own inputs:

  normalisation   |y - y64| <= c1 * ulp(m) * rstd * |gamma| + c2 * 2^-23 * ((|x - mean| * rstd + 1) * |gamma| + |beta|)
  attention       |o - o64| <= 2^-23 * (A_FIX + A_ACC * sqrt(n_keys) + A_SCORE * sqrt(d) * S) * sum_j p_j |v_j|

with m the mean (GroupNorm) or the mean absolute value (LayerNorm) of the normalised set, S the largest sum_c |q_c k_c| / T
(+ the relative-position term) of the row, and p the float64 softmax.  The constants and where they come from are below."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
EPS = float(np.float32(1e-5))

# GroupNorm: the mean is finalised in fp64 from sums taken about the group's first element and rounded once (c1 = 1: half an
# ulp, and as much again); the apply step rounds three times and rstd carries a few ulps of the fp32 sums of squares (c2 = 8).
# tests/test_cpu_groupnorm_model.py derives both against a float32 model of the kernel's reduction order.
GN_C1, GN_C2 = 1.0, 8.0
# LayerNorm (one warp per row, fp32 two-pass): c1 = c2 = 9 + ceil(C / 128), the roundings on the way into a sum -- three per
# float4, one per step of the lane's running sum, five butterfly levels -- plus the division, rsqrtf's 2 ulps and the apply step.
LN_FIX = 9
# Attention: the value sum is a chain of fp32 FMAs over the keys (A_ACC per sqrt(key), as independent rounding errors add);
# a score error ds moves the softmax by at most 2 ds relative, and ds grows with the d-term FMA chain of the dot product and the
# rounding of q / T (A_SCORE per sqrt(d) times the magnitude S of the summands); expf, the row sum and the final 1/l cost a
# fixed few ulps (A_FIX).
A_FIX, A_ACC, A_SCORE = 8.0, 2.0, 4.0
# max |GELU'(y)| (at y = sqrt(2)); erff and the products of the GELU add a few ulps of |y|
GELU_SLOPE = 1.13

ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2


def _dev():
    return torch.device("cuda:0")


def _ulp32(t):
    """fp64 tensor -> the fp32 ulp of each |value| (as fp64)."""
    return torch.from_numpy(np.spacing(t.abs().float().numpy()).astype(np.float64))


def _act64(y, act):
    return {ACT_NONE: lambda t: t, ACT_RELU: F.relu, ACT_GELU: F.gelu}[act](y)


def _act_tol(y64, tol, act):
    """Tolerance after the activation, given the tolerance `tol` before it."""
    if act == ACT_GELU:
        return GELU_SLOPE * tol + 4 * U * y64.abs()
    return tol


def _nan_buf(*shape):
    return torch.full(shape, float("nan"), device=_dev())


# ----------------------------------------------------------------------------------------------------------------- GroupNorm
def _gn_data(B, P, C, offset, seed):
    """[B, P, C] float32: batch b is sigma_b * (z + offset_b) with different sigma and offset per batch element."""
    g = torch.Generator().manual_seed(seed)
    sig = (1.5, 0.7)
    off = (offset, -offset / 2)
    x = torch.stack([sig[b] * (torch.randn(P, C, generator=g, dtype=torch.float64) + off[b]) for b in range(B)]).float()
    return x, torch.randn(C, generator=g), torch.randn(C, generator=g)


def _gn_reference(x, G, gamma, beta, act):
    """float64 GroupNorm of float32 x [B, P, C] -> (act(y), tolerance) per element."""
    B, P, C = x.shape
    xr = x.double().view(B, P, G, C // G)
    mean = xr.mean(dim=(1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(((xr - mean) ** 2).mean(dim=(1, 3), keepdim=True) + EPS)
    ga, be = gamma.double().view(1, 1, G, C // G), beta.double().view(1, 1, G, C // G)
    y = ((xr - mean) * rstd * ga + be).view(B, P, C)
    tol = (GN_C1 * _ulp32(mean) * rstd * ga.abs()
           + GN_C2 * U * (((xr - mean).abs() * rstd + 1.0) * ga.abs() + be.abs())).view(B, P, C)
    return _act64(y, act), _act_tol(y, tol, act)


def _gn_run(x, G, gamma, beta, act, ws=None, ldx_pad=4, ldo_pad=16):
    """groupnorm on a column slice of a wider input into a column slice of a wider NaN-filled output (ldx != ldo, both > C);
    returns the slice and checks that the columns around it are untouched."""
    from aot_benchmark_b200 import ops
    d = _dev()
    B, P, C = x.shape
    xb = torch.zeros(B, P, C + 2 * ldx_pad, device=d)
    xb[:, :, ldx_pad:ldx_pad + C] = x.to(d)
    ob = _nan_buf(B, P, C + ldo_pad)
    o0 = ldo_pad // 2
    ws = ops.groupnorm_workspace(B, G, d) if ws is None else ws
    ops.groupnorm(xb[:, :, ldx_pad:ldx_pad + C], gamma.to(d), beta.to(d), ob[:, :, o0:o0 + C], G, act, ws)
    torch.cuda.synchronize()
    assert torch.isnan(ob[:, :, :o0]).all() and torch.isnan(ob[:, :, o0 + C:]).all()
    return ob[:, :, o0:o0 + C].cpu()


def _assert_within(out, ref, tol, what=""):
    err = (out.double() - ref).abs()
    assert torch.isfinite(out).all(), what
    ratio = (err / tol).max().item()
    assert ratio <= 1.0, f"{what}: max |err| {err.max().item():.3e}, worst err / tol {ratio:.3f}"


# the three engine sites: FFN GroupNorm(32, 1024) on the 31 x 54 token map, decoder conv_4x GroupNorm(8, 128) on the
# 121 x 213 map, GroupNorm1D(512, groups=2) before the decoder
GN_SITES = [(1674, 1024, 32, ACT_GELU), (25773, 128, 8, ACT_RELU), (1674, 512, 2, ACT_NONE)]


@pytest.mark.parametrize("offset", [0, 10, 100, 1000])
@pytest.mark.parametrize("P,C,G,act", GN_SITES)
def test_groupnorm_mean_offset(P, C, G, act, offset):
    """Groups whose mean is up to 1000 standard deviations from zero (the fp32 one-pass E[x^2] - mean^2 misses this tolerance
    at 100 and 1000)."""
    x, ga, be = _gn_data(2, P, C, offset, seed=P + G + offset)
    ref, tol = _gn_reference(x, G, ga, be, act)
    _assert_within(_gn_run(x, G, ga, be, act), ref, tol, f"offset {offset}")


@pytest.mark.parametrize("P,C,G", [
    (1674, 256, 1), (1674, 256, 2), (1674, 256, 8), (1674, 256, 32), (1674, 256, 64),   # Cg = 256 .. 4
    (1, 256, 8), (5, 256, 8), (1, 4, 1), (5, 128, 32),                                   # fewer pixels than chunks
    (63, 256, 8), (65, 256, 8),                                                          # 8 chunks: 8 x 8 -/+ 1 pixels
    (511, 1024, 2), (513, 1024, 2),                                                      # 64 chunks: 8 x 64 -/+ 1 pixels
    (25773, 256, 64),
])
@pytest.mark.parametrize("act", [ACT_NONE, ACT_RELU, ACT_GELU])
def test_groupnorm_shapes(P, C, G, act):
    x, ga, be = _gn_data(2, P, C, 100, seed=7 * P + G + act)
    ref, tol = _gn_reference(x, G, ga, be, act)
    _assert_within(_gn_run(x, G, ga, be, act), ref, tol, f"P {P} C {C} G {G}")


def test_groupnorm_in_place():
    """out == x, as the engine calls it: the shift is read by the statistics kernel before the apply kernel writes."""
    from aot_benchmark_b200 import ops
    d = _dev()
    x, ga, be = _gn_data(2, 1674, 1024, 1000, seed=3)
    ref, tol = _gn_reference(x, 32, ga, be, ACT_GELU)
    xg = x.to(d)
    ops.groupnorm(xg, ga.to(d), be.to(d), xg, 32, ACT_GELU, ops.groupnorm_workspace(2, 32, d))
    _assert_within(xg.cpu(), ref, tol, "in place")


def test_groupnorm_workspace_reuse():
    """One workspace, back to back across different (B, G, P): the last block's counter reset leaves it ready for the next
    shape, and every result equals that of a fresh workspace bit for bit."""
    from aot_benchmark_b200 import ops
    d = _dev()
    ws = ops.groupnorm_workspace(2, 64, d)
    seq = [(2, 5, 256, 64), (1, 25773, 128, 8), (2, 1674, 512, 2), (1, 63, 128, 32), (2, 5, 256, 64), (2, 1674, 1024, 32)]
    for i, (B, P, C, G) in enumerate(seq):
        x, ga, be = _gn_data(B, P, C, 10 * i, seed=50 + i)
        got = _gn_run(x, G, ga, be, ACT_RELU, ws=ws)
        fresh = _gn_run(x, G, ga, be, ACT_RELU)
        assert torch.equal(got, fresh), (B, P, C, G)
        ref, tol = _gn_reference(x, G, ga, be, ACT_RELU)
        _assert_within(got, ref, tol, str((B, P, C, G)))
    assert ws.view(torch.int32)[0].item() == 0                      # the launch counter is back to zero


def test_groupnorm_graph_replay_bitwise():
    from aot_benchmark_b200 import ops
    d = _dev()
    x, ga, be = _gn_data(2, 1674, 1024, 100, seed=11)
    xg, gag, beg = x.to(d), ga.to(d), be.to(d)
    ws = ops.groupnorm_workspace(2, 32, d)
    eager = torch.empty_like(xg)
    ops.groupnorm(xg, gag, beg, eager, 32, ACT_GELU, ws)
    out = torch.zeros_like(xg)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.groupnorm(xg, gag, beg, out, 32, ACT_GELU, ws)
    for _ in range(3):
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)


# ----------------------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("offset", [0, 10, 100, 1000])
@pytest.mark.parametrize("C", [4, 36, 256, 260, 1024])
def test_layernorm(C, offset):
    """37 rows (not a multiple of the 8 rows of a block), ldx / ldo / ldadd wider than C, out2 = LN + add into a column slice;
    the two-pass fp32 form holds the tolerance at every mean offset."""
    from aot_benchmark_b200 import ops
    d = _dev()
    rows = 37
    g = torch.Generator().manual_seed(C + offset)
    x = ((torch.randn(rows, C, generator=g, dtype=torch.float64) + offset) * 1.5
         + torch.linspace(-3, 3, rows, dtype=torch.float64).view(-1, 1)).float()
    ga, be = torch.randn(C, generator=g), torch.randn(C, generator=g)
    add = torch.randn(rows, C, generator=g) * 4
    x64 = x.double()
    mean = x64.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x64 - mean) ** 2).mean(1, keepdim=True) + EPS)
    ref = (x64 - mean) * rstd * ga.double() + be.double()
    c = LN_FIX + math.ceil(C / 128)
    tol = (c * _ulp32(x64.abs().mean(1, keepdim=True)) * rstd * ga.double().abs()
           + c * U * (((x64 - mean).abs() * rstd + 1.0) * ga.double().abs() + be.double().abs()))
    ref2 = ref + add.double()
    tol2 = tol + U * ref2.abs()

    xb = torch.zeros(rows, C + 8, device=d)
    xb[:, 4:4 + C] = x.to(d)
    ab = torch.zeros(rows, C + 20, device=d)
    ab[:, 16:16 + C] = add.to(d)
    ob = _nan_buf(rows, C + 12)
    ob2 = _nan_buf(rows, 2 * C + 4)
    ops.layernorm(xb[:, 4:4 + C], ga.to(d), be.to(d), ob[:, 8:8 + C], add=ab[:, 16:16 + C], out2=ob2[:, C:2 * C])
    torch.cuda.synchronize()
    assert torch.isnan(ob[:, :8]).all() and torch.isnan(ob[:, 8 + C:]).all()
    assert torch.isnan(ob2[:, :C]).all() and torch.isnan(ob2[:, 2 * C:]).all()
    _assert_within(ob[:, 8:8 + C].cpu(), ref, tol, "out")
    _assert_within(ob2[:, C:2 * C].cpu(), ref2, tol2, "out2")


# ----------------------------------------------------------------------------------------------------------- SIMT attention
def _attn_reference(Q, K, V, H, dq, dv):
    """float64 softmax(Q K^T / sqrt(dq)) V per head for float32 Q [N, H*dq], K [Tk, H*dq], V [Tk, H*dv] ->
    (out [N, H*dv], tolerance [N, H*dv])."""
    N, Tk = Q.shape[0], K.shape[0]
    T = math.sqrt(dq)
    q = Q.double().view(N, H, dq).transpose(0, 1)
    k = K.double().view(Tk, H, dq).transpose(0, 1)
    v = V.double().view(Tk, H, dv).transpose(0, 1)
    p = torch.softmax((q / T) @ k.transpose(1, 2), dim=-1)                              # [H, N, Tk]
    out = (p @ v).transpose(0, 1).reshape(N, H * dv)
    S = (q.abs() / T @ k.abs().transpose(1, 2)).amax(-1, keepdim=True)                 # [H, N, 1]
    pv = p @ v.abs()                                                                     # [H, N, dv]
    tol = U * (A_FIX + A_ACC * math.sqrt(Tk) + A_SCORE * math.sqrt(dq) * S) * pv
    return out, tol.transpose(0, 1).reshape(N, H * dv)


# (H, d_qk, d_v): the three instantiations <32, 32>, <32, 64> (d_v a multiple of 64) and <128, 256> (a multiple of 256)
ATTN_HEADS = [(8, 32, 32), (2, 32, 128), (1, 128, 512)]
EDGES = [1, 63, 64, 65, 129]


def _attn_inputs(H, dq, dv, N, Tk, qscale, seed):
    g = torch.Generator().manual_seed(seed)
    Q = torch.randn(N, H * dq, generator=g) * qscale
    K = torch.randn(Tk, H * dq, generator=g)
    V = torch.randn(Tk, H * dv, generator=g)
    return Q, K, V


def _slices(d, N, Tk, H, dq, dv, Q, K, V):
    """Q / K / V as column slices of wider buffers with different row strides, O a slice of a wider NaN-filled buffer."""
    qb = torch.zeros(N, H * dq + 12, device=d)
    kb = torch.zeros(Tk + 3, H * dq + 36, device=d)
    vb = torch.zeros(Tk + 3, H * dv + 4, device=d)
    qb[:, 8:8 + H * dq] = Q.to(d)
    kb[:Tk, 32:32 + H * dq] = K.to(d)
    vb[:Tk, 4:4 + H * dv] = V.to(d)
    return qb[:, 8:8 + H * dq], kb[:, 32:32 + H * dq], vb[:, 4:4 + H * dv]


@pytest.mark.parametrize("Tk", EDGES)
@pytest.mark.parametrize("N", EDGES)
@pytest.mark.parametrize("H,dq,dv", ATTN_HEADS)
def test_attention_edges(H, dq, dv, N, Tk):
    """N and Tk at the 64-row tile edges; every other shape with q scaled by 30, which makes the softmax near one-hot; a device
    key count overrides a different host count bit for bit."""
    from aot_benchmark_b200 import ops
    d = _dev()
    qscale = 30.0 if (EDGES.index(N) + EDGES.index(Tk)) % 2 else 1.0
    Q, K, V = _attn_inputs(H, dq, dv, N, Tk, qscale, seed=N * 1000 + Tk + dv)
    ref, tol = _attn_reference(Q, K, V, H, dq, dv)
    q, k, v = _slices(d, N, Tk, H, dq, dv, Q, K, V)
    ob = _nan_buf(N, H * dv + 8)
    ops.attention(q, k, v, ob[:, 4:4 + H * dv], H, dq, dv, Tk=Tk)
    torch.cuda.synchronize()
    assert torch.isnan(ob[:, :4]).all() and torch.isnan(ob[:, 4 + H * dv:]).all()
    _assert_within(ob[:, 4:4 + H * dv].cpu(), ref, tol, f"qscale {qscale}")
    tk_dev = torch.tensor([Tk], dtype=torch.int32, device=d)
    o2 = _nan_buf(N, H * dv)
    ops.attention(q, k, v, o2, H, dq, dv, Tk=Tk + 2, Tk_dev=tk_dev)             # host count says two more rows
    assert torch.equal(o2, ob[:, 4:4 + H * dv])


@pytest.mark.parametrize("H,dq,dv", ATTN_HEADS)
def test_attention_split_kv_with_empty_shard(H, dq, dv):
    """Split-KV partials of three shards -- the middle one empty through a device key count of 0 against a host count of 5 --
    give (O, M, L) = (0, -inf, 0) for the empty shard, and attn_merge of all three, or of one shard spanning every key, equals
    the unsplit attention."""
    from aot_benchmark_b200 import ops
    d = _dev()
    N, Tk, cut = 129, 200, 65
    Q, K, V = _attn_inputs(H, dq, dv, N, Tk, 6.0, seed=dv)
    ref, tol = _attn_reference(Q, K, V, H, dq, dv)
    q, k, v = _slices(d, N, Tk, H, dq, dv, Q, K, V)
    full = torch.empty(N, H * dv, device=d)
    ops.attention(q, k, v, full, H, dq, dv, Tk=Tk)
    R = 3
    Op = _nan_buf(R, N, H * dv)
    Mp = _nan_buf(R, H, N)
    Lp = _nan_buf(R, H, N)
    ops.attention(q, k[:cut], v[:cut], Op[0], H, dq, dv, Tk=cut, Mout=Mp[0], Lout=Lp[0])
    zero = torch.zeros(1, dtype=torch.int32, device=d)
    ops.attention(q, k[cut:], v[cut:], Op[1], H, dq, dv, Tk=5, Tk_dev=zero, Mout=Mp[1], Lout=Lp[1])
    ops.attention(q, k[cut:], v[cut:], Op[2], H, dq, dv, Tk=Tk - cut, Mout=Mp[2], Lout=Lp[2])
    torch.cuda.synchronize()
    assert torch.equal(Op[1], torch.zeros_like(Op[1]))
    assert torch.equal(Mp[1], torch.full_like(Mp[1], -math.inf)) and torch.equal(Lp[1], torch.zeros_like(Lp[1]))
    mb = _nan_buf(N, H * dv + 8)
    ops.attn_merge(Op, Mp, Lp, mb[:, 4:4 + H * dv], H, dv)
    torch.cuda.synchronize()
    assert torch.isnan(mb[:, :4]).all() and torch.isnan(mb[:, 4 + H * dv:]).all()
    merged = mb[:, 4:4 + H * dv].cpu()
    _assert_within(full.cpu(), ref, tol, "unsplit")
    # each shard within the bound of its own keys, and the merge's exp / sums / division a few ulps more
    _assert_within(merged, ref, 2 * tol, "merge of three shards")
    _assert_within(merged, full.cpu().double(), 3 * tol, "merge against unsplit")
    # one shard over every key: the merge is the unsplit normalisation done as a division
    O1, M1, L1 = torch.empty(1, N, H * dv, device=d), torch.empty(1, H, N, device=d), torch.empty(1, H, N, device=d)
    ops.attention(q, k, v, O1[0], H, dq, dv, Tk=Tk, Mout=M1[0], Lout=L1[0])
    one = torch.empty(N, H * dv, device=d)
    ops.attn_merge(O1, M1, L1, one, H, dv)
    torch.cuda.synchronize()
    assert ((one - full).abs() <= 2 * U * full.abs()).all()          # o / l against o * (1 / l)


# -------------------------------------------------------------------------------------------------------- local attention
# h and w at the 8 x 6 query tile and 15-tap window edges; every value of each appears at least once
LOCAL_HW = [(1, 1), (1, 13), (7, 5), (8, 6), (9, 7), (16, 12), (17, 13), (17, 1), (8, 13), (9, 6), (16, 5), (7, 12)]


def _local_reference(q, k, v, rkw, rkb, rv, H):
    """float64 short-term attention (oracle unfold form) of float32 NCHW inputs -> (out [hw, H*dv], tol [hw, H*dv])."""
    from oracle import aot_oracle as O
    n, c, h, w = q.shape
    dq, dv = c // H, v.shape[1] // H
    T = math.sqrt(dq)
    q64, k64, v64, w64, b64 = q.double(), k.double(), v.double(), rkw.double(), rkb.double()
    rv64 = rv.double() if rv is not None else None
    out = O.local_attention(q64, k64, v64, w64, b64, rv64, H)[:, 0]
    # softmax and score magnitudes per (query, head, tap), with the same -1e8 for taps outside the frame
    P = 225
    rel = F.conv2d(q64, w64, b64, groups=H).view(1, H, P, h * w)
    relmag = F.conv2d(q64.abs(), w64.abs(), b64.abs(), groups=H).view(1, H, P, h * w)
    ku = F.unfold(k64, 15, padding=7).view(1, H, dq, P, h * w)
    qv = (q64 / T).view(1, H, dq, h * w)
    s = torch.einsum("nhdp,nhdwp->nhwp", qv, ku) + rel
    inside = F.unfold(torch.ones(1, 1, h, w, dtype=torch.float64), 15, padding=7).view(1, 1, P, h * w)
    p = torch.softmax(s - (1 - inside) * 1e8, dim=2)
    S = (torch.einsum("nhdp,nhdwp->nhwp", qv.abs(), ku.abs()) + relmag).amax(2)         # [1, H, hw]
    vu = F.unfold(v64.abs(), 15, padding=7).view(1, H, dv, P, h * w)
    pv = torch.einsum("nhwp,nhdwp->nhdp", p, vu)                                         # [1, H, dv, hw]
    if rv64 is not None:
        pv = pv + torch.einsum("nhwp,hcw->nhcp", p, rv64.abs())
    tol = U * (A_FIX + A_ACC * math.sqrt(P) + A_SCORE * math.sqrt(dq) * S.unsqueeze(2)) * pv
    return out, tol[0].permute(2, 0, 1).reshape(h * w, H * dv)


def _engine_slices(d, tok_q, tok_k, tok_v):
    """q, k, v as column slices of one wider [hw, ...] buffer, the way the engine passes them."""
    cq, ck, cv = tok_q.shape[1], tok_k.shape[1], tok_v.shape[1]
    buf = torch.zeros(tok_q.shape[0], cq + ck + cv + 24, device=d)
    buf[:, 4:4 + cq] = tok_q.to(d)
    buf[:, 12 + cq:12 + cq + ck] = tok_k.to(d)
    buf[:, 20 + cq + ck:20 + cq + ck + cv] = tok_v.to(d)
    return buf[:, 4:4 + cq], buf[:, 12 + cq:12 + cq + ck], buf[:, 20 + cq + ck:20 + cq + ck + cv]


def _tok(t):
    return t[0].permute(1, 2, 0).reshape(t.shape[2] * t.shape[3], -1).contiguous()


def _check_slice(ob, c0, c1, ref, tol, what):
    torch.cuda.synchronize()
    assert torch.isnan(ob[:, :c0]).all() and torch.isnan(ob[:, c1:]).all(), f"{what}: wrote outside its columns"
    _assert_within(ob[:, c0:c1].cpu(), ref, tol, what)


@pytest.mark.parametrize("qscale", [1.0, 30.0])
@pytest.mark.parametrize("h,w", LOCAL_HW)
def test_local_attention_aot(h, w, qscale):
    """AOT head shape (8 heads, d = 32, relative_emb_v): the per-warp kernel and the 8 x 6 tiled kernel."""
    from aot_benchmark_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(h * 100 + w + int(qscale))
    H = 8
    q = torch.randn(1, 256, h, w, generator=g) * qscale
    k = torch.randn(1, 256, h, w, generator=g)
    v = torch.randn(1, 256, h, w, generator=g)
    rkw = torch.randn(1800, 32, 1, 1, generator=g) * 0.2
    rkb = torch.randn(1800, generator=g) * 0.1
    rv = torch.randn(8, 32, 225, generator=g) * 0.3
    ref, tol = _local_reference(q, k, v, rkw, rkb, rv, H)
    qs, ks, vs = _engine_slices(d, _tok(q), _tok(k), _tok(v))
    w2, b2 = rkw.view(1800, 32).contiguous().to(d), rkb.to(d)
    ob = _nan_buf(h * w, 256 + 40)
    ops.local_attention(qs, ks, vs, w2, b2, rv.to(d), ob[:, 16:272], h, w, H, 32, 32)
    _check_slice(ob, 16, 272, ref, tol, "per-warp")
    ob = _nan_buf(h * w, 256 + 40)
    ops.local_attention_tile(qs, ks, vs, w2, b2, rv.permute(0, 2, 1).contiguous().to(d), ob[:, 36:292], h, w, H)
    _check_slice(ob, 36, 292, ref, tol, "tile")


@pytest.mark.parametrize("qscale", [1.0, 30.0])
@pytest.mark.parametrize("h,w", LOCAL_HW)
def test_local_attention_deaot(h, w, qscale):
    """DeAOT head shape (1 head, d_att = 128, d_v = 1024, no relative_emb_v): the per-warp kernel and the gated tile kernel."""
    from aot_benchmark_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(h * 100 + w + int(qscale) + 7)
    q = torch.randn(1, 128, h, w, generator=g) * (qscale / 2)
    k = torch.randn(1, 128, h, w, generator=g)
    v = torch.randn(1, 1024, h, w, generator=g)
    rkw = torch.randn(225, 128, 1, 1, generator=g) * 0.1
    rkb = torch.randn(225, generator=g) * 0.1
    ref, tol = _local_reference(q, k, v, rkw, rkb, None, 1)
    qs, ks, vs = _engine_slices(d, _tok(q), _tok(k), _tok(v))
    w2, b2 = rkw.view(225, 128).contiguous().to(d), rkb.to(d)
    ob = _nan_buf(h * w, 1024 + 40)
    ops.local_attention(qs, ks, vs, w2, b2, None, ob[:, 8:1032], h, w, 1, 128, 1024)
    _check_slice(ob, 8, 1032, ref, tol, "per-warp")
    ob = _nan_buf(h * w, 1024 + 40)
    ops.local_gated_tile(qs, ks, vs, w2, b2, ob[:, 32:1056], h, w)
    _check_slice(ob, 32, 1056, ref, tol, "gated tile")


# ------------------------------------------------------------------------------------------------------------ elementwise
@pytest.mark.parametrize("W", [17, 18, 19])                 # Wo = W + 2 pad - 4: Wo mod 4 = 1, 2, 3 at pad 2 (and at pad 0)
@pytest.mark.parametrize("pad", [0, 2])
def test_dwconv5_row4(W, pad):
    """5x5 stride-1 depthwise conv (the row-of-4 kernel), batch 2, input and output as column slices."""
    _dwconv_case(2, 13, W, 36, 5, 1, pad, 1, seed=W + pad)


@pytest.mark.parametrize("K,stride,pad,dil", [(5, 2, 2, 1), (3, 1, 2, 2), (3, 2, 2, 2), (5, 1, 4, 2)])
def test_dwconv_generic(K, stride, pad, dil):
    _dwconv_case(2, 15, 21, 36, K, stride, pad, dil, seed=K * 10 + stride + dil)


def _dwconv_case(B, H, W, C, K, stride, pad, dil, seed):
    from aot_benchmark_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g) * 3
    wt = torch.randn(C, 1, K, K, generator=g) * 0.2
    b = torch.randn(C, generator=g)
    ref = F.conv2d(x.double(), wt.double(), b.double(), stride, pad, dil, C)
    mag = F.conv2d(x.double().abs(), wt.double().abs(), b.double().abs(), stride, pad, dil, C)
    tol = U * (K * K + 1) / 2 * mag                        # a chain of K*K fp32 FMAs from the bias
    Ho, Wo = ref.shape[2:]
    xb = torch.zeros(B, H, W, C + 12, device=d)
    xb[..., 8:8 + C] = x.permute(0, 2, 3, 1).to(d)
    ob = _nan_buf(B, Ho, Wo, C + 8)
    ops.dwconv(xb[..., 8:8 + C], wt.permute(2, 3, 1, 0).reshape(K * K, C).contiguous().to(d), b.to(d), ob[..., 4:4 + C],
               K=K, stride=stride, pad=pad, dil=dil)
    torch.cuda.synchronize()
    assert torch.isnan(ob[..., :4]).all() and torch.isnan(ob[..., 4 + C:]).all()
    _assert_within(ob[..., 4:4 + C].cpu().permute(0, 3, 1, 2), ref, tol, "dwconv")


@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("H,W,Ho,Wo", [(31, 54, 13, 20), (1, 1, 5, 7), (9, 11, 1, 1), (31, 54, 61, 107), (4, 3, 1, 9)])
def test_bilinear(H, W, Ho, Wo, align):
    """Downscale, 1-pixel input, 1-pixel output and upscale, batch 2, against F.interpolate in float64.  The kernel computes
    the source coordinate in fp32: its rounding (about max(H, W) ulps of 1) moves a weight, times the step between taps."""
    from aot_benchmark_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(H * W + Ho)
    x = torch.randn(2, 8, H, W, generator=g) * 2
    ref = F.interpolate(x.double(), size=(Ho, Wo), mode="bilinear", align_corners=align)
    out = _nan_buf(2, Ho, Wo, 8)
    ops.bilinear(x.permute(0, 2, 3, 1).contiguous().to(d), out, align)
    torch.cuda.synchronize()
    tol = U * (4 + 4 * max(H, W)) * x.abs().max().item()
    _assert_within(out.cpu().permute(0, 3, 1, 2), ref, torch.full_like(ref, tol), "bilinear")


@pytest.mark.parametrize("H,W", [(13, 17), (14, 18), (13, 18), (1, 2), (2, 1)])
def test_maxpool3x3s2(H, W):
    """Odd and even sizes, batch 2, with -inf entries (a window of -inf alone stays -inf): bit-exact."""
    from aot_benchmark_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(H * 31 + W)
    x = torch.randn(2, 8, H, W, generator=g)
    x[torch.rand(x.shape, generator=g) < 0.3] = -math.inf
    x[1, :, :3, :3] = -math.inf
    ref = F.max_pool2d(x, 3, 2, 1)
    out = _nan_buf(2, ref.shape[2], ref.shape[3], 8)
    ops.maxpool3x3s2(x.permute(0, 2, 3, 1).contiguous().to(d), out)
    assert torch.equal(out.cpu().permute(0, 3, 1, 2), ref)


@pytest.mark.parametrize("op", [0, 1, 2, 3, 4, 5])
def test_eltwise_strided(op):
    """All six ops on [rows, cols] views whose row strides all differ; copy / add / mul / fill are exact in fp32."""
    from aot_benchmark_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(op)
    rows, cols = 37, 44
    a = torch.randn(rows, cols, generator=g) * 5
    b = torch.randn(rows, cols, generator=g)
    ab = torch.zeros(rows, cols + 8, device=d)
    bb = torch.zeros(rows, cols + 20, device=d)
    ab[:, 4:4 + cols] = a.to(d)
    bb[:, 16:16 + cols] = b.to(d)
    ob = _nan_buf(rows, cols + 3)
    ops.eltwise(op, ab[:, 4:4 + cols] if op != ops.EW_FILL else None, bb[:, 16:16 + cols] if op in (1, 2, 4) else None,
                ob[:, 1:1 + cols], scalar=-2.75)
    torch.cuda.synchronize()
    assert torch.isnan(ob[:, :1]).all() and torch.isnan(ob[:, 1 + cols:]).all()
    out = ob[:, 1:1 + cols].cpu()
    exact = {0: a, 1: a + b, 2: a * b, 5: torch.full_like(a, -2.75)}
    if op in exact:
        assert torch.equal(out, exact[op])
    else:
        ref = F.silu(a.double()) * (b.double() if op == 4 else 1.0)
        _assert_within(out, ref, 4 * U * (ref.abs() + U), f"op {op}")


@pytest.mark.parametrize("C,HW", [(3, 45 * 67), (45, 33), (70, 100)])
def test_transposes(C, HW):
    """nchw_to_nhwc / nhwc_to_nchw, batch 2, C and HW not multiples of 32: bit-exact round trip."""
    from aot_benchmark_b200 import ops
    d = _dev()
    g = torch.Generator().manual_seed(C + HW)
    x = torch.randn(2, C, 1, HW, generator=g)
    nhwc = _nan_buf(2, 1, HW, C)
    ops.nchw_to_nhwc(x.to(d), nhwc)
    assert torch.equal(nhwc.cpu(), x.permute(0, 2, 3, 1))
    back = _nan_buf(2, C, 1, HW)
    ops.nhwc_to_nchw(nhwc, back)
    assert torch.equal(back.cpu(), x)
