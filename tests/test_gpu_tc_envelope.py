"""GPU: the tensor-core kernels at the edges of their envelope, against float64 references.

- Weight scale: the split-fp16 conv / linear with weights scaled by 2^k, and with channels whose rms spans 1e-4 .. 1e-1
  (FrozenBN folding makes such channels), stays within the fp32-accumulation bound in every channel, through the
  per-layer kernel and ops.conv2d / ops.linear with registered weights.
- Tiling: every N tile x split-K cluster size the conv kernel can be forced to, at M / K tails, general Cin, stride 2,
  batch 2, strided rows, an aliased residual and every activation.
- Attention: the fused long-term attention kernels (all layouts, exact and fast) at the 64 / 128 tile edges, with a
  device-resident key count under a fixed split count (empty splits), a column-slice output, poisoned padding rows, and
  closed-form cases, each in both modes.  The fast mode (S = Qh Kh, P rounded to fp16) is held to a bound derived over the
  kernel's own packed operands (attn_restatement), on the full N x Tk grid."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


# ------------------------------------------------------------------ convolutions
def _pack_w(w):  # [Cout, Cin, KH, KW] -> fp32 [K, Cout] (k = (ky, kx, ci))
    co, ci, kh, kw = w.shape
    return w.permute(2, 3, 1, 0).reshape(kh * kw * ci, co).contiguous()


def _act(y, act):
    return [lambda t: t, F.relu, lambda t: F.gelu(t), F.silu, lambda t: t.clamp(0.0, 6.0)][act](y)


def _ref_conv(x, w, b, stride, pad, res=None, act=0):
    """float64 NHWC reference: x [B, H, W, Cin], w [Cout, Cin, K, K], res like the output."""
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), None if b is None else b.double(), stride, pad)
    y = y.permute(0, 2, 3, 1)
    if res is not None:
        y = y + res.double()
    return _act(y, act)


def _conv_tc(x, w4, b, stride, pad, res=None, act=0, normalise=True, out=None):
    from aot_benchmark_b200 import ops
    wk = _pack_w(w4).to(DEV)
    if normalise:
        wh, wl, ws = ops.split_fp16_scaled(wk)
    else:
        (wh, wl), ws = ops.split_fp16(wk), None
    K = w4.shape[2]
    if out is None:
        Ho, Wo = (x.shape[1] + 2 * pad - K) // stride + 1, (x.shape[2] + 2 * pad - K) // stride + 1
        out = torch.full((x.shape[0], Ho, Wo, w4.shape[0]), float("nan"), device=DEV)
    ops.conv2d_tc(x, wh, wl, None if b is None else b.to(DEV), out, res=res, KH=K, KW=K, stride=stride, pad=pad, act=act,
                  wscale=ws)
    torch.cuda.synchronize()
    return out


def _channel_err(out, ref):
    """per output channel: max |out - ref| and max |ref| over all pixels."""
    C = ref.shape[-1]
    d = (out.double().cpu() - ref).abs().reshape(-1, C).amax(0)
    return d, ref.abs().reshape(-1, C).amax(0)


# 3x3 conv (Cin 256, Cout 128, 13 x 11 = 143 pixels: one full 128-row tile and a tail) and a 1024 -> 256 linear
WEIGHT_SHAPES = {"conv3x3": (1, 13, 11, 256, 128, 3, 1), "linear": (1, 300, 1, 1024, 256, 1, 0)}


def _weight_scale_case(kind, seed=0):
    B, H, W, Cin, Cout, K, pad = WEIGHT_SHAPES[kind]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, K, K, generator=g) / math.sqrt(Cin * K * K)
    return x, w, pad


def weight_scale_sweep(kind, normalise=True):
    """-> {k: worst per-channel max |out - ref| / max |ref|} for weights scaled by 2^k, and the outputs per k."""
    x, w, pad = _weight_scale_case(kind)
    xg = x.to(DEV)
    errs, outs = {}, {}
    for k in range(-14, 5):
        wk = w * 2.0 ** k                                    # exact
        out = _conv_tc(xg, wk, None, 1, pad, normalise=normalise)
        d, s = _channel_err(out, _ref_conv(x, wk, None, 1, pad))
        errs[k], outs[k] = (d / s).max().item(), out
    return errs, outs


@pytest.mark.parametrize("kind", ["conv3x3", "linear"])
def test_weight_scale_sweep(kind):
    """Weights scaled by 2^k, k = -14 .. 4: within 1e-5 of max |ref| in every channel at every k (without the per-channel
    normalisation the small scales are off by up to ~1e-4), and bitwise equivariant: out(w 2^k) == 2^k out(w)."""
    errs, outs = weight_scale_sweep(kind)
    bad = {k: e for k, e in errs.items() if not e < 1e-5}
    assert not bad, f"per-channel relative error above 1e-5 at 2^k: {bad}"
    for k, o in outs.items():
        assert torch.equal(o, outs[0] * 2.0 ** k), f"not equivariant at 2^{k}"


def _mixed_weights(Cout, Cin, K, g):
    """channels with rms from 1e-4 to 1e-1 (log-spaced)"""
    rms = torch.logspace(-4, -1, Cout, dtype=torch.float64)
    return (torch.randn(Cout, Cin, K, K, generator=g, dtype=torch.float64) * rms.view(-1, 1, 1, 1)).float()


@pytest.mark.parametrize("kind", ["conv3x3", "linear"])
def test_small_weight_channels(kind):
    """Channels with rms 1e-4 .. 1e-1 each stay within 1e-5 of their own max |ref|, through the kernel directly and
    through ops.conv2d / ops.linear with weights registered as the engine registers them (bit-identical to the former)."""
    from aot_benchmark_b200 import ops
    B, H, W, Cin, Cout, K, pad = WEIGHT_SHAPES[kind]
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, H, W, Cin, generator=g)
    w = _mixed_weights(Cout, Cin, K, g)
    b = torch.randn(Cout, generator=g) * 1e-3
    xg = x.to(DEV)
    ref = _ref_conv(x, w, b, 1, pad)
    out = _conv_tc(xg, w, b, 1, pad)
    d, s = _channel_err(out, ref)
    assert (d / s).max().item() < 1e-5, f"worst channel {(d / s).argmax().item()}: {(d / s).max().item():.2e}"
    wk = _pack_w(w).to(DEV)
    ops.register_tc_weights(wk, *ops.split_fp16_scaled(wk))
    try:
        out2 = torch.full_like(out, float("nan"))
        if kind == "linear":
            ops.linear(xg.view(H, Cin), wk, b.to(DEV), out2.view(H, Cout))
        else:
            ops.conv2d(xg, wk, b.to(DEV), out2, KH=K, KW=K, pad=pad)
        torch.cuda.synchronize()
    finally:
        ops._TC_WEIGHTS.pop(wk.data_ptr(), None)
    assert torch.equal(out, out2)


# B, H, W, Cin, Cout, K, stride, pad, residual ("" | "res" | "alias"), act, wide (ldin / ldout / ldres wider than C)
TILING_CASES = [
    (1, 9, 9, 64, 128, 3, 1, 1, "res", 1, False),       # 9 chunks: with S = 8, CTAs 5 .. 7 of a cluster have none
    (1, 1, 1, 64, 128, 3, 1, 1, "", 2, False),          # M = 1
    (1, 127, 1, 256, 128, 1, 1, 0, "res", 3, False),    # M = 127
    (1, 8, 16, 64, 64, 3, 1, 1, "", 4, False),          # M = 128
    (1, 3, 43, 64, 128, 3, 1, 1, "alias", 0, False),    # M = 129, residual aliasing the output
    (1, 33, 41, 4, 64, 7, 2, 3, "", 1, False),          # general Cin: 4 x 7 x 7 = 196
    (1, 17, 19, 12, 128, 3, 1, 1, "res", 4, True),      # 12 x 9 = 108
    (1, 13, 15, 36, 64, 1, 1, 0, "", 2, False),         # 36 x 1 (K < 64)
    (1, 11, 12, 100, 128, 3, 1, 1, "alias", 3, True),   # 100 x 9 = 900: 15 chunks
    (1, 9, 10, 12, 64, 7, 1, 3, "", 0, False),          # 12 x 49 = 588
    (1, 15, 17, 64, 64, 3, 2, 1, "res", 1, True),       # stride 2
    (2, 7, 9, 128, 192, 3, 1, 1, "res", 2, False),      # batch 2, Cout 192 (N tile 64 only)
    (2, 12, 13, 256, 128, 1, 2, 0, "alias", 4, True),   # batch 2, strided 1x1
]


@pytest.mark.parametrize("case", TILING_CASES, ids=[f"c{i}" for i in range(len(TILING_CASES))])
def test_conv_tiling_sweep(case):
    """Every N tile (64, 128) x split-K cluster size (1, 2, 4, 8 <= chunks) forced through aotb_set_conv_tiling: within the
    fp32-accumulation bound of the float64 reference, and bitwise reproducible."""
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import lib
    B, H, W, Cin, Cout, K, stride, pad, rmode, act, wide = case
    g = torch.Generator().manual_seed(H * 131 + Cin)
    x = torch.randn(B, H, W, Cin, generator=g) * 2
    w = torch.randn(Cout, Cin, K, K, generator=g) / math.sqrt(Cin * K * K)
    b = torch.randn(Cout, generator=g)
    Ho, Wo = (H + 2 * pad - K) // stride + 1, (W + 2 * pad - K) // stride + 1
    r = torch.randn(B, Ho, Wo, Cout, generator=g) if rmode else None
    ref = _ref_conv(x, w, b, stride, pad, r, act)
    scale = ref.abs().max().item()
    ex = 8 if wide else 0
    xg = torch.zeros(B, H, W, Cin + ex, device=DEV)
    xg[..., :Cin] = x.to(DEV)
    xv = xg[..., :Cin]
    wk = _pack_w(w).to(DEV)
    wh, wl, ws = ops.split_fp16_scaled(wk)
    obuf = torch.full((B, Ho, Wo, Cout + 2 * ex), float("nan"), device=DEV)
    out = obuf[..., ex:ex + Cout]
    rbuf = torch.full((B, Ho, Wo, Cout + ex), float("nan"), device=DEV) if rmode == "res" else None
    if rbuf is not None:
        rbuf[..., :Cout] = r.to(DEV)
    nchunks = (K * K * Cin + 63) // 64
    tried = 0
    try:
        for bn_code, BN in ((1, 64), (2, 128)):
            if Cout % BN:
                continue
            for S in (1, 2, 4, 8):
                if S > nchunks:
                    continue
                assert lib().aotb_set_conv_tiling((bn_code << 4) | (S << 8)) == 0
                runs = []
                for _ in range(2):
                    obuf.fill_(float("nan"))
                    if rmode == "alias":
                        out.copy_(r.to(DEV))
                    res = out if rmode == "alias" else (None if rbuf is None else rbuf[..., :Cout])
                    ops.conv2d_tc(xv, wh, wl, b.to(DEV), out, res=res, KH=K, KW=K, stride=stride, pad=pad, act=act,
                                  wscale=ws)
                    torch.cuda.synchronize()
                    runs.append(obuf.clone())
                err = (runs[0][..., ex:ex + Cout].double().cpu() - ref).abs().max().item()
                assert err < 1e-5 * max(scale, 1.0) + 1e-5, f"BN {BN} S {S}: err {err:.3e} (scale {scale:.2f})"
                assert torch.equal(runs[0][..., ex:ex + Cout], runs[1][..., ex:ex + Cout]), f"BN {BN} S {S}: not reproducible"
                for o in runs:
                    assert torch.isnan(o[..., :ex]).all() and torch.isnan(o[..., ex + Cout:]).all(), \
                        f"BN {BN} S {S}: wrote outside its columns"
                tried += 1
    finally:
        lib().aotb_set_conv_tiling(0)
    assert tried >= 1


# ------------------------------------------------------------------ attention
H_LT, D = 8, 32
NS = (1, 63, 64, 65, 127, 128, 129, 257)
TKS = (1, 63, 64, 65, 127, 128, 129, 255, 257)


def _attn_ref(Q, K, V, heads, d_att):
    from oracle import aot_oracle as O
    return O.multihead_attention(Q.double().cpu().unsqueeze(1), K.double().cpu().unsqueeze(1),
                                 V.double().cpu().unsqueeze(1), heads, d_att=d_att)[:, 0]


class _Attn:
    """Packed operands of one problem for the AOT kernel (gp=False: H = 8 heads x 32) or the DeAOT one (gp=True: d_qk 128,
    d_v 256), with padding rows of the packed buffers set to `qpad` (Q rows >= N) / `kvpad` (K, V rows >= Tk).  Q is divided
    by `qdiv` when packed (default T = sqrt(d_qk), as the engines pack it)."""

    def __init__(self, Q, K, V, gp, qpad=0.0, kvpad=0.0, kv_rows=None, qdiv=None):
        from aot_benchmark_b200 import ops
        self.gp, self.N, self.Tk = gp, Q.shape[0], K.shape[0]
        unit = 64 if gp else 128
        ncap = -(-self.N // (128 if gp else 256)) * (128 if gp else 256)
        kcap = (kv_rows or -(-self.Tk // unit) * unit) + unit

        def pack(x, cap, heads, pad, div=1.0):
            full = torch.full((cap, x.shape[1]), pad, device=DEV)
            full[:x.shape[0]] = x
            dst = torch.zeros(heads, cap, 64, dtype=torch.float16, device=DEV)
            ops.tc_pack_rows(full, dst, 0, div)
            return dst

        self.Qp = pack(Q, ncap, 4 if gp else H_LT, qpad, math.sqrt(128.0 if gp else 32.0) if qdiv is None else qdiv)
        self.Kp = pack(K, kcap, 4 if gp else H_LT, kvpad)
        self.Vp = pack(V, kcap, V.shape[1] // 32, kvpad)
        self.dv = V.shape[1]

    def run(self, exact=True, variant="tile", Tk=None, Tk_dev=None, splits=1, O=None):
        from aot_benchmark_b200 import ops
        N = self.N
        O = torch.full((N, self.dv), float("nan"), device=DEV) if O is None else O
        part = None
        if splits > 1:
            hp = 1 if self.gp else H_LT
            part = (torch.full((splits, N, self.dv), float("nan"), device=DEV),
                    torch.full((splits, hp, N), float("nan"), device=DEV), torch.full((splits, hp, N), float("nan"), device=DEV))
        tk = self.Tk if Tk is None else Tk
        if self.gp:
            ops.gp_attention_tc(self.Qp, self.Kp, self.Vp, N, tk, O=O, Tk_dev=Tk_dev, splits=splits, exact=exact, part=part)
        else:
            ops.lt_attention_tc(self.Qp, self.Kp, self.Vp, N, tk, O=O, Tk_dev=Tk_dev, splits=splits, exact=exact, part=part,
                                variant=variant)
        torch.cuda.synchronize()
        return O


def _qkv(N, Tk, gp, seed):
    g = torch.Generator().manual_seed(seed)
    dq = 128 if gp else 256
    return (torch.randn(N, dq, generator=g), torch.randn(Tk, dq, generator=g),
            torch.randn(Tk, 256, generator=g))


def _ref_for(Q, K, V, gp):
    return _attn_ref(Q, K, V, 1, 128) if gp else _attn_ref(Q, K, V, H_LT, D)


# The fast mode (exact bit clear) against float64 over the kernel's own operands.  With q, k, v the packed values read back
# from Qp / Kp / Vp (exact mode: S = qh kh + ql kh + qh kl, v = vh + vl; fast mode: S = qh kh, v = vh + vl), p_j = exp(s_j - m)
# against the final row max m, l = sum_j p_j and O64 = sum_j p_j v_j / l, the kernel's O differs from O64 by
#   - the rounding of P: ph (+ pl) is within eps_P p_j + 2^-25 of p_j, eps_P = 2^-11 (fast, fp16 round to nearest) or 2^-22
#     (exact, the split), and 2^-25 the half spacing of fp16 subnormals.  P is rounded against the running row max of its
#     split, which is at most m, and rescaled by exp(m_run - m) <= 1 later, so the bound holds against the final max.  The row
#     sum l is summed from the unrounded fp32 p, so P's rounding enters only the numerator: sum_j (eps_P p_j + 2^-25) |v_j| / l.
#   - fp32 arithmetic, in the form tests/test_gpu_simt_envelope.py uses for its attention: 2^-23 (A_FIX + A_ACC sqrt(Tk) +
#     A_SCORE sqrt(d_qk) S) sum_j p_j |v_j| / l, with S the row's largest sum_c |q_c k_c| (the score's FMA chain, the
#     exponent argument s log2e - m log2e rounded in fp32), A_ACC per sqrt(key) for the P V chain, A_FIX for ex2, l and 1 / l,
#     doubled with KV splits for the merge's exponentials, sums and division.
A_FIX, A_ACC, A_SCORE = 8.0, 2.0, 4.0
EPS_P = {True: 2.0 ** -22, False: 2.0 ** -11}


def unpack(P, rows, part="both"):
    """packed [H', cap, 64] fp16 operand -> float64 [rows, H' 32]: hi, lo or hi + lo of each value"""
    hi, lo = P[:, :rows, :32].double(), P[:, :rows, 32:].double()
    x = {"hi": hi, "lo": lo, "both": hi + lo}[part]
    return x.permute(1, 0, 2).reshape(rows, -1)


def attn_restatement(q, k, v, heads, exact, splits=1, qk=None):
    """float64 restatement of the kernel over its operands.  q = (qh, ql), k = (kh, kl) [rows, heads d_qk] and v [Tk, dv]
    float64 (see unpack); `qk` overrides the three (exact) or one (fast) score products.  -> (O64, bound) [N, dv]."""
    N, Tk, dv = q[0].shape[0], k[0].shape[0], v.shape[1]
    dq = q[0].shape[1] // heads
    hd = lambda x, d: x.view(x.shape[0], heads, d).transpose(0, 1)
    qh, ql, kh, kl = hd(q[0], dq), hd(q[1], dq), hd(k[0], dq), hd(k[1], dq)
    vv = hd(v, dv // heads)
    if qk is None:
        s = qh @ kh.transpose(1, 2)
        if exact:
            s = s + ql @ kh.transpose(1, 2) + qh @ kl.transpose(1, 2)
    else:
        s = qk
    sabs = (qh.abs() + ql.abs()) @ (kh.abs() + kl.abs()).transpose(1, 2) if exact else qh.abs() @ kh.abs().transpose(1, 2)
    S = sabs.amax(-1, keepdim=True)
    p = torch.exp(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    o = (p @ vv) / l
    pv = (p @ vv.abs()) / l
    fix = A_FIX * (2 if splits > 1 else 1)
    tol = (EPS_P[exact] * pv + 2.0 ** -25 * vv.abs().sum(1, keepdim=True) / l
           + 2.0 ** -23 * (fix + A_ACC * math.sqrt(Tk) + A_SCORE * math.sqrt(dq) * S) * pv)
    back = lambda x: x.transpose(0, 1).reshape(N, dv)
    return back(o), back(tol)


def packed_restatement(A, exact, Tk=None, splits=1):
    """attn_restatement over the packed buffers of an _Attn problem (Tk live keys)."""
    tk = A.Tk if Tk is None else Tk
    q = (unpack(A.Qp, A.N, "hi"), unpack(A.Qp, A.N, "lo"))
    k = (unpack(A.Kp, tk, "hi"), unpack(A.Kp, tk, "lo"))
    return attn_restatement(q, k, unpack(A.Vp, tk), 1 if A.gp else H_LT, exact, splits)


def within(O, ref, tol, what=""):
    """-> worst |O - ref| / tol (asserted below 1)"""
    r = ((O.double().to(ref.device) - ref).abs() / tol).max().item()
    assert r < 1.0, f"{what}: worst |O - O64| / bound = {r:.3f}"
    return r


ATTN_KERNELS = [("tile", False), ("groups", False), ("ahead", False), ("pair", False), ("gp", True)]
# both modes; the exact cases keep the ids they had before the fast ones were added
ATTN_MODES = [(v, gp, ex) for ex in (True, False) for v, gp in ATTN_KERNELS]
MODE_IDS = [f"{v}-{gp}" + ("" if ex else "-fast") for v, gp, ex in ATTN_MODES]


@pytest.mark.parametrize("variant,gp", ATTN_KERNELS)
@pytest.mark.parametrize("exact", [True, False])
def test_attention_tile_edges(variant, gp, exact):
    """N and Tk on both sides of the 64 / 128 tile boundaries: the exact mode against the float64 oracle, the fast mode within
    the bound over its own operands (attn_restatement) on the same full grid."""
    tol = (5e-5 if gp else 3e-5)       # d_qk 128 for the DeAOT kernel
    bad, worst = [], 0.0
    for N, Tk in [(n, t) for n in NS for t in TKS]:
        Q, K, V = _qkv(N, Tk, gp, N * 1000 + Tk)
        A = _Attn(Q.to(DEV), K.to(DEV), V.to(DEV), gp)
        O = A.run(exact=exact, variant=variant)
        if exact:
            err = (O.cpu().double() - _ref_for(Q, K, V, gp)).abs().max().item()
            if not err < tol:
                bad.append((N, Tk, err))
        else:
            ref, bound = packed_restatement(A, exact)
            r = ((O.double() - ref).abs() / bound).max().item()
            worst = max(worst, r)
            if not r < 1.0:
                bad.append((N, Tk, r))
    if not exact:
        print(f"fast {variant}: worst |O - O64| / bound {worst:.3f}")
    assert not bad, f"(N, Tk, max |dO| or |dO| / bound) out of bounds: {bad}"


@pytest.mark.parametrize("variant,gp,exact", ATTN_MODES, ids=MODE_IDS)
def test_attention_device_key_count_empty_splits(variant, gp, exact):
    """The engine fixes the split count at graph capture and reads the live key count on the device at replay, so splits
    can be empty: splits = 8 with a device count equals the host-count call bitwise and matches float64 (exact mode) or
    the restatement over the kernel's operands (fast mode)."""
    N, cap = 129, 1024
    Q, K, V = _qkv(N, cap, gp, 11)
    A = _Attn(Q.to(DEV), K.to(DEV), V.to(DEV), gp)
    for tk in (1, 65, 129, 300, 1000):                  # 1 .. 8 of the 8 splits hold keys
        dev = torch.tensor([tk], dtype=torch.int32, device=DEV)
        Od = A.run(exact=exact, variant=variant, Tk=1, Tk_dev=dev, splits=8)
        Oh = A.run(exact=exact, variant=variant, Tk=tk, splits=8)
        assert torch.equal(Od, Oh), f"Tk {tk}: device and host key counts differ"
        if exact:
            err = (Od.cpu().double() - _ref_for(Q, K[:tk], V[:tk], gp)).abs().max().item()
            assert err < 3e-5, f"Tk {tk}: max |dO| = {err:.2e}"
        else:
            within(Od, *packed_restatement(A, False, Tk=tk, splits=8), f"Tk {tk}")


@pytest.mark.parametrize("variant,gp,exact", ATTN_MODES, ids=MODE_IDS)
def test_attention_column_slice_output(variant, gp, exact):
    """O written into columns [256, 512) of an [N, 512] buffer (the engine writes into [lt_core | st_core]): equal to the
    dense result bitwise, neighbouring columns untouched; with and without KV splits."""
    N, Tk = 129, 257
    Q, K, V = _qkv(N, Tk, gp, 12)
    A = _Attn(Q.to(DEV), K.to(DEV), V.to(DEV), gp)
    for splits in (1, 3):
        dense = A.run(exact=exact, variant=variant, splits=splits)
        buf = torch.randn(N, 512, device=DEV)
        keep = buf.clone()
        A.run(exact=exact, variant=variant, splits=splits, O=buf[:, 256:])
        assert torch.equal(buf[:, 256:], dense), f"splits {splits}"
        assert torch.equal(buf[:, :256], keep[:, :256]), f"splits {splits}: columns [0, 256) changed"


@pytest.mark.parametrize("variant,gp,exact", ATTN_MODES, ids=MODE_IDS)
def test_attention_poisoned_padding(variant, gp, exact):
    """Padding rows are never read into a live result: Q rows >= N set to NaN and K / V rows in [Tk, kv_cap) set to 3e4 give
    the zero-padded result bitwise, with and without splits and a device key count."""
    for N, Tk in ((65, 63), (129, 200), (1, 129)):
        Q, K, V = _qkv(N, Tk, gp, 13 + N)
        Qd, Kd, Vd = Q.to(DEV), K.to(DEV), V.to(DEV)
        clean = _Attn(Qd, Kd, Vd, gp, kv_rows=512)
        dirty = _Attn(Qd, Kd, Vd, gp, qpad=float("nan"), kvpad=3e4, kv_rows=512)
        dev = torch.tensor([Tk], dtype=torch.int32, device=DEV)
        for kw in (dict(), dict(splits=4), dict(Tk=1, Tk_dev=dev, splits=8)):
            a, b = clean.run(exact=exact, variant=variant, **kw), dirty.run(exact=exact, variant=variant, **kw)
            assert torch.equal(a, b), f"N {N} Tk {Tk} {kw}: max |d| = {(a - b).abs().max().item()}"


@pytest.mark.parametrize("variant,gp,exact", ATTN_MODES, ids=MODE_IDS)
def test_attention_closed_forms(variant, gp, exact):
    """Q = 0: every key has the same score, so O is the column mean of V.  One key whose score leads every other by >= 100:
    O is that key's V row.  In both forms every p is exactly 1 or below 2^-140, so the fast mode is as faithful as the exact
    one, and two tighter forms catch a V rounded to fp16 (Vl dropped), which the fast mode's bound alone would not: a single
    key (Tk = 1: O = V to the split's 2^-22 and one rounding) and Q = 0 over three keys (O = their mean to a few fp32 ulps)."""
    N, Tk = 65, 200
    _, K, V = _qkv(N, Tk, gp, 14)
    Q = torch.zeros(N, K.shape[1])
    O = _Attn(Q.to(DEV), K.to(DEV), V.to(DEV), gp).run(exact=exact, variant=variant)
    mean = V.double().mean(0, keepdim=True).expand(N, -1)
    assert (O.cpu().double() - mean).abs().max().item() < 1e-5
    for tk in (1, 3):
        O = _Attn(Q.to(DEV), K[:tk].to(DEV), V[:tk].to(DEV), gp).run(exact=exact, variant=variant)
        # Tk = 1: the split (2^-22 |v| + 2^-25) and the add of the hi / lo accumulators; Tk = 3: also two sums, 1 / l and O' / l
        c = 2.0 ** -21 if tk == 1 else 2.0 ** -20
        tol = c * V[:tk].double().abs().mean(0) + 2.0 ** -25
        err = ((O.cpu().double() - V[:tk].double().mean(0)).abs() / tol).max().item()
        assert err < 1.0, f"Q = 0, Tk {tk}: |O - mean V| / ({c:.1e} mean |V| + 2^-25) = {err:.2f}"
    # key j: K[j] = c * u with a unit direction u per head / query block, queries along u; every other key orthogonal-ish
    g = torch.Generator().manual_seed(15)
    K = torch.randn(Tk, K.shape[1], generator=g) * 0.01
    hd = 128 if gp else D
    d_att = 128 if gp else D
    j = 77
    Q = torch.zeros(N, K.shape[1])
    for h in range(K.shape[1] // hd):
        u = torch.zeros(hd)
        u[h % hd] = 1.0
        K[j, h * hd:(h + 1) * hd] = u * 30.0
        Q[:, h * hd:(h + 1) * hd] = u * (110.0 * math.sqrt(d_att) / 30.0)   # score of key j: 110, of the others: < 1
    O = _Attn(Q.to(DEV), K.to(DEV), V.to(DEV), gp).run(exact=exact, variant=variant)
    assert (O.cpu() - V[j].view(1, -1)).abs().max().item() < 1e-5
