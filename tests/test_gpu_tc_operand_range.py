"""GPU: the tensor-core kernels across the magnitude of their activation and attention operands.

The split-fp16 kernels carry an fp32 operand x as hi = fp16(x), lo = fp16(x - hi); the single-pass (fp16 mode) kernels carry
hi only.  The weights are normalised per output channel, so their magnitude does not matter (tests/test_gpu_tc_envelope.py);
the other operand is split as it comes.  This module sweeps that operand over 2^-24 .. 2^13 and checks three statements:

  restatement   float64 over the values the kernel multiplies -- hi + lo of x read back from torch's CPU fp16 conversion
                (which keeps subnormals) against Ah Wh + Al Wh + Ah Wl, or fp16(x) against fp16(w 2^e) 2^-e -- is within
                C_ACC 2^-23 sum_k |x_k| |w_k| per output element over that element's taps (the fp32 accumulation; the finish
                multiplies by an exact power of two).  At the small end of the sweep hi and lo are fp16 subnormals, so this
                fails if the producer's conversion or wgmma flushed them.
  law           against the plain float64 conv, per element sum_k (R |x_k| |w_k| + 2^-25 |w_k| + 2^-25 ws |x_k|) plus the
                restatement term: R = 2^-21 for the split (x and w each within 2^-22 relative, the dropped Al Wl 2^-22),
                R = 2^-10 + 2^-21 for single pass (x and w each within 2^-11), 2^-25 the half spacing of fp16 subnormals
                (the floor of x, and of w 2^e, which the finish scales by ws = 2^-e).
  equivariance  out(x 2^a) == 2^a out(x) bitwise, wherever the halves of x 2^a stay normal fp16 (no bias, no residual).

C_ACC: the accumulator is fp32 over P ceil(K / 16) wgmma k-steps (P = 3 split, 1 single).  With n such roundings of a running
sum whose size grows like sqrt(k) t for products of size t, the rounding errors add to about 2^-24 n t sqrt(8 / 3), while
sum_k |x_k| |w_k| is about 16 n E|t|, so the ratio of the two does not grow with K.  C_ACC = 4 leaves that ratio a margin of
about 20 for round-to-nearest and covers a truncating accumulator up to n ~ 400 (K = 2304 split).

The fused attention kernels (AOT 8 heads x 32, DeAOT d_qk 128 with d_v 1024, so the value grid reaches 16 slices) in both
modes: V 2^c gives 2^c O bitwise while Vh and Vl stay normal; Q 2^a with K 2^-a gives the same O bitwise (same exact scores);
Q, K and V swept separately into the floor regime within test_gpu_tc_envelope.attn_restatement's bound over the packed values;
and the engine's own launches (N = 1674, self-attention and a memory bank, split counts from engine.lt_splits and the DeAOT
split rule, a device key count) within that bound, where fast and exact also differ by more than the exact mode's own error.

Measured on an H100 80GB HBM3 (700 W): see DESIGN.md section 3.1."""
import math
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from test_gpu_tc_envelope import DEV, H_LT, _Attn, _pack_w, attn_restatement, packed_restatement, unpack

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
C_ACC = 4.0
# The subnormal tail: at x 2^a with a <= SUB_TAIL, where every hi is an fp16 subnormal with at most 9 significant bits, the
# tensor-core result departs from the fp32-accumulation restatement by an absolute amount that does not shrink with x
# (measured on an H100: up to 18 C_ACC 2^-23 sum |x| |w| at 2^-24, halving per binade up, 1.4 at 2^-20).  There the restatement is
# held to SUB_COEF sum |x| |w|, 2^-12: still about a hundred times below what a flush to zero of the subnormal operands costs
# (tests/test_cpu_tc_operand_controls.py), so the sweep still shows that wgmma reads fp16 subnormals.
SUB_TAIL, SUB_COEF = -18, 2.0 ** -12
LAW = {True: (2.0 ** -21, 2.0 ** -25), False: (2.0 ** -10 + 2.0 ** -21, 2.0 ** -25 * (1 + 2.0 ** -10))}
FLOOR = 2.0 ** -25

# ------------------------------------------------------------------ convolutions
# B, H, W, Cin, Cout, K, stride, pad, forced tiling (aotb_set_conv_tiling), grid cap
CONV_CASES = {
    "conv3x3": (1, 13, 11, 256, 128, 3, 1, 1, 0, 0),           # M = 143: a full 128-row tile and a tail
    "linear": (1, 300, 1, 1024, 256, 1, 1, 0, 0, 0),           # 1024 -> 256
    "stem7x7": (1, 33, 41, 4, 64, 7, 2, 3, 0, 0),              # 4-channel gather: Cin % 64 != 0
    "persistent": (1, 37, 41, 64, 128, 1, 1, 0, (1 << 4) | (1 << 8), 3),   # 12 x 2 tiles of BN 64 on 3 CTAs: 8 per CTA
}
A_SCALES = list(range(-24, 14))                # randn clamped to |x| <= 7: max |x| 2^13 = 57344 < 65504


def conv_case(kind, device="cpu"):
    """-> SimpleNamespace: x (randn, |x| <= 7, float32 CPU), w [Cout, Cin, K, K] float32, the packed split weights on
    `device` and the weights the kernel multiplies by, Wh4 = fp16(w 2^e) 2^-e and Wl4, float64 [Cout, Cin, K, K]."""
    from aot_benchmark_b200 import ops
    B, H, W, Cin, Cout, K, stride, pad, tiling, cap = CONV_CASES[kind]
    g = torch.Generator().manual_seed(Cin * 7 + K)
    x = torch.randn(B, H, W, Cin, generator=g).clamp(-7.0, 7.0)
    w = torch.randn(Cout, Cin, K, K, generator=g) / math.sqrt(Cin * K * K)
    wh, wl, ws = ops.split_fp16_scaled(_pack_w(w).to(device))
    four = lambda t: (t[:, :K * K * Cin].double().cpu() * ws.double().cpu().view(-1, 1)).view(Cout, K, K, Cin) \
        .permute(0, 3, 1, 2).contiguous()
    return SimpleNamespace(kind=kind, x=x, w=w, wh=wh, wl=wl, ws=ws, Wh4=four(wh), Wl4=four(wl), K=K, stride=stride,
                           pad=pad, tiling=tiling, cap=cap, Cout=Cout)


def conv64(x, w, c):
    """float64 NHWC conv of x [B, H, W, Cin] with w [Cout, Cin, K, K] on x's device."""
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().to(x.device), None, c.stride, c.pad)
    return y.permute(0, 2, 3, 1)


def split_x(x):
    """hi = fp16(x), lo = fp16(x - hi) by torch's CPU conversion (round to nearest, subnormals kept), as float64."""
    hi = x.cpu().float().half()
    lo = (x.cpu().float() - hi.float()).half()
    return hi.double(), lo.double()


def restatement_coef(a):
    """The restatement bound's coefficient of sum |x| |w| at activation scale 2^a (see the module docstring)."""
    return C_ACC * U if a > SUB_TAIL else SUB_COEF


def conv_restatement(c, x, split, dev="cpu", hi=None, lo=None, a=0):
    """float64 over the kernel's operands -> (ref, bound) [B, Ho, Wo, Cout] on `dev` (hi / lo override the split of x; `a`
    is the scale of x, which selects the coefficient)."""
    h, l = split_x(x)
    h, l = (h if hi is None else hi).to(dev), (l if lo is None else lo).to(dev)
    if split:
        ref = conv64(h + l, c.Wh4, c) + conv64(h, c.Wl4, c)
        sabs = conv64(h.abs() + l.abs(), c.Wh4.abs(), c) + conv64(h.abs(), c.Wl4.abs(), c)
    else:
        ref = conv64(h, c.Wh4, c)
        sabs = conv64(h.abs(), c.Wh4.abs(), c)
    return ref, restatement_coef(a) * sabs


def conv_law(c, x, split, dev="cpu", a=0):
    """plain float64 conv -> (ref, bound) with the operand terms of DESIGN section 3.1 plus the restatement term."""
    R, fl = LAW[split]
    xd = x.double().to(dev)
    ref = conv64(xd, c.w, c)
    wabs = c.w.double().abs()
    tol = (R * conv64(xd.abs(), wabs, c) + fl * conv64(torch.ones_like(xd), wabs, c)
           + FLOOR * c.ws.double().to(dev) * conv64(xd.abs(), torch.ones_like(wabs), c))
    return ref, tol + conv_restatement(c, x, split, dev, a=a)[1]


def run_conv(c, x, split, act=0):
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import lib
    B, H, W, _ = x.shape
    Ho, Wo = (H + 2 * c.pad - c.K) // c.stride + 1, (W + 2 * c.pad - c.K) // c.stride + 1
    out = torch.full((B, Ho, Wo, c.Cout), float("nan"), device=DEV)
    assert lib().aotb_set_conv_tiling(c.tiling) == 0 and lib().aotb_set_conv_grid_cap(c.cap) == 0
    try:
        ops.conv2d_tc(x.to(DEV), c.wh, c.wl if split else None, None, out, KH=c.K, KW=c.K, stride=c.stride, pad=c.pad,
                      act=act, wscale=c.ws)
        torch.cuda.synchronize()
    finally:
        lib().aotb_set_conv_tiling(0)
        lib().aotb_set_conv_grid_cap(0)
    return out


def _ratio(out, ref, tol):
    return ((out.double().to(ref.device) - ref).abs() / tol).max().item()


MODES = [True, False]
MODE_IDS = ["split", "single"]


@pytest.mark.parametrize("split", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("kind", list(CONV_CASES))
def test_conv_activation_scale_sweep(kind, split):
    """x 2^a, a = -24 .. 13: within the restatement bound (its subnormal-tail form at a <= SUB_TAIL) and within the law at
    every scale (worst ratios printed)."""
    c = conv_case(kind, DEV)
    worst_r = worst_l = worst_t = 0.0
    bad = []
    for a in A_SCALES:
        x = c.x * 2.0 ** a                                   # exact
        out = run_conv(c, x, split)
        rr = _ratio(out, *conv_restatement(c, x, split, DEV, a=a))
        rl = _ratio(out, *conv_law(c, x, split, DEV, a=a))
        worst_l = max(worst_l, rl)
        if a <= SUB_TAIL:
            worst_t = max(worst_t, rr)
        else:
            worst_r = max(worst_r, rr)
        if not (rr < 1.0 and rl < 1.0):
            bad.append((a, rr, rl))
    print(f"{kind} {MODE_IDS[MODES.index(split)]}: worst err / bound: restatement {worst_r:.3f} (a > {SUB_TAIL}), "
          f"{worst_t:.3f} (a <= {SUB_TAIL}), law {worst_l:.3f}")
    assert not bad, f"(a, restatement ratio, law ratio) out of bounds: {bad}"


def exact_pairs(shape, seed, lo_exp=-12):
    """fp32 x = hi + lo with hi in +-[1, 2) and lo in +-[2^lo_exp, 2^(lo_exp + 1)), both fp16, so fp16(x) = hi and
    fp16(x - hi) = lo exactly (|lo| < ulp(hi) / 2 = 2^-11, and x needs 23 significant bits)."""
    g = torch.Generator().manual_seed(seed)
    sign = torch.randint(0, 2, shape, generator=g).float() * 2 - 1
    hi = ((1 + torch.rand(shape, generator=g)) * sign).half().clamp(-1.999, 1.999).half()
    lo = ((1 + 0.99 * torch.rand(shape, generator=g)) * 2.0 ** lo_exp * sign).half()     # the sign of hi: x stays in hi's binade
    x = hi.float() + lo.float()
    assert torch.equal(x.double(), hi.double() + lo.double())
    assert torch.equal(x.half(), hi) and torch.equal((x - x.half().float()).half(), lo)
    return x


@pytest.mark.parametrize("split", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("kind", list(CONV_CASES))
def test_conv_activation_scale_equivariance(kind, split):
    """out(x 2^a) == 2^a out(x) bitwise, act none and ReLU: split mode on exact hi + lo pairs for a = -2 .. 15 (lo 2^a stays
    normal, hi 2^a <= 65504), single pass on fp16 values for a = -14 .. 15 (hi 2^a normal)."""
    c = conv_case(kind, DEV)
    x = exact_pairs(c.x.shape, 5) if split else exact_pairs(c.x.shape, 5).half().float()
    window = range(-2, 16) if split else range(-14, 16)
    for act in (0, 1):
        base = run_conv(c, x, split, act)
        assert torch.isfinite(base).all()
        for a in window:
            o = run_conv(c, x * 2.0 ** a, split, act)
            assert torch.equal(o, base * 2.0 ** a), f"act {act}: not equivariant at 2^{a}"


def top_edge_input(shape, seed):
    """|x| uniform up to 65519.99, an eighth of the elements in [65504, 65520) (fp16(x) = 65504, x - 65504 < 16), and the
    two ends themselves."""
    g = torch.Generator().manual_seed(seed)
    sgn = torch.randint(0, 2, shape, generator=g).float() * 2 - 1
    mag = torch.rand(shape, generator=g) * 65519.99
    edge = torch.rand(shape, generator=g) < 0.125
    mag = torch.where(edge, 65504.0 + torch.rand(shape, generator=g) * 15.99, mag)
    x = (sgn * mag).view(-1)
    x[0], x[1], x[2] = 65504.0, -65519.99, 65519.99
    x = x.view(shape)
    assert x.abs().max().item() < 65520 and torch.isfinite(x.half()).all()
    return x


@pytest.mark.parametrize("split", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("kind", list(CONV_CASES))
def test_conv_top_edge(kind, split):
    """|x| up to 65519.99 (hi = 65504 at the top, lo <= 16): finite, within the restatement bound and the law."""
    c = conv_case(kind, DEV)
    x = top_edge_input(c.x.shape, 6)
    out = run_conv(c, x, split)
    assert torch.isfinite(out).all()
    rr = _ratio(out, *conv_restatement(c, x, split, DEV))
    rl = _ratio(out, *conv_law(c, x, split, DEV))
    print(f"{kind} {MODE_IDS[MODES.index(split)]} top edge: restatement {rr:.3f}, law {rl:.3f}")
    assert rr < 1.0 and rl < 1.0, (rr, rl)


# ------------------------------------------------------------------ attention
ATTN = [(False, 256), (True, 1024)]           # (DeAOT kernel, d_v): AOT 8 heads x 32; DeAOT d_qk 128, d_v 1024
ATTN_IDS = ["aot", "deaot_dv1024"]
EXACT_IDS = ["exact", "fast"]


def attn_inputs(N, Tk, gp, dv, seed):
    g = torch.Generator().manual_seed(seed)
    dq = 128 if gp else 256
    return (torch.randn(N, dq, generator=g), torch.randn(Tk, dq, generator=g),
            torch.randn(Tk, dv, generator=g).clamp(-7.0, 7.0))


def _run_attn(Q, K, V, gp, exact, splits=1, qdiv=None, **kw):
    A = _Attn(Q.to(DEV), K.to(DEV), V.to(DEV), gp, qdiv=qdiv)
    part = dict(splits=splits)
    return A, A.run(exact=exact, **part, **kw)


@pytest.mark.parametrize("exact", [True, False], ids=EXACT_IDS)
@pytest.mark.parametrize("gp,dv", ATTN, ids=ATTN_IDS)
def test_attention_value_scale_equivariance(gp, dv, exact):
    """V 2^c, c = -2 .. 15, on exact hi + lo pairs (Vh and Vl normal throughout): O(V 2^c) == 2^c O(V) bitwise, with and
    without KV splits (V enters only through P [Vh | Vl] and the merge is linear in O)."""
    N, Tk = 129, 257
    Q, K, _ = attn_inputs(N, Tk, gp, dv, 21)
    V = exact_pairs((Tk, dv), 22)
    for splits in (1, 3):
        _, base = _run_attn(Q, K, V, gp, exact, splits)
        for c in range(-2, 16):
            _, o = _run_attn(Q, K, V * 2.0 ** c, gp, exact, splits)
            assert torch.equal(o, base * 2.0 ** c), f"splits {splits}: not equivariant at V 2^{c}"


@pytest.mark.parametrize("exact", [True, False], ids=EXACT_IDS)
@pytest.mark.parametrize("gp,dv", ATTN, ids=ATTN_IDS)
def test_attention_query_key_exchange(gp, dv, exact):
    """Q 2^a with K 2^-a (Q packed without the 1/T, so the scaling is exact): the same scores, so the same O bitwise, with
    and without KV splits.  Exact mode on hi + lo pairs for a = -2 .. 2 (every half of both stays normal), fast mode on the
    hi halves, which are all it reads, for a = -14 .. 14."""
    N, Tk = 129, 257
    _, _, V = attn_inputs(N, Tk, gp, dv, 23)
    dq = 128 if gp else 256
    Q, K = exact_pairs((N, dq), 24), exact_pairs((Tk, dq), 25)
    window = range(-2, 3) if exact else range(-14, 15)
    for splits in (1, 3):
        _, base = _run_attn(Q, K, V, gp, exact, splits, qdiv=1.0)
        assert torch.isfinite(base).all()
        for a in window:
            _, o = _run_attn(Q * 2.0 ** a, K * 2.0 ** -a, V, gp, exact, splits, qdiv=1.0)
            assert torch.equal(o, base), f"splits {splits}: Q 2^{a}, K 2^{-a} changed O"


# (operand, scales): Q is the raw feature, divided by T = sqrt(d_qk) when packed (scale 0 is the engine's magnitude)
SWEEPS = {"Q": list(range(-24, 5, 2)), "K": list(range(-24, 5, 2)), "V": list(range(-24, 14, 2)) + [13]}


def sweep_restatement(q, k, v, heads, exact, splits, op, s):
    """attn_restatement's (O64, bound), plus SUB_COEF sum_j p_j |v_j| / l in V's subnormal tail (see SUB_TAIL: the P V
    product shows the same tail as the conv)."""
    ref, tol = attn_restatement(q, k, v, heads, exact, splits)
    if op == "V" and s <= SUB_TAIL:
        tol = tol + SUB_COEF * attn_restatement(q, k, v.abs(), heads, exact, splits)[0]
    return ref, tol


def sweep_inputs(op, s, gp, dv, seed=26):
    N, Tk = 129, 257
    Q, K, V = attn_inputs(N, Tk, gp, dv, seed)
    f = 2.0 ** s
    return (Q * f, K, V) if op == "Q" else (Q, K * f, V) if op == "K" else (Q, K, V * f)


@pytest.mark.parametrize("op", list(SWEEPS))
@pytest.mark.parametrize("exact", [True, False], ids=EXACT_IDS)
@pytest.mark.parametrize("gp,dv", ATTN, ids=ATTN_IDS)
def test_attention_operand_scale_sweep(gp, dv, exact, op):
    """Q, K or V scaled by 2^s down into the fp16 subnormals: within sweep_restatement's bound over the packed values at
    every scale (splits 1 and 3 alternating)."""
    worst, bad = 0.0, []
    for i, s in enumerate(SWEEPS[op]):
        splits = 1 + 2 * (i % 2)
        A, O = _run_attn(*sweep_inputs(op, s, gp, dv), gp, exact, splits)
        q = (unpack(A.Qp, A.N, "hi"), unpack(A.Qp, A.N, "lo"))
        k = (unpack(A.Kp, A.Tk, "hi"), unpack(A.Kp, A.Tk, "lo"))
        r = _ratio(O, *sweep_restatement(q, k, unpack(A.Vp, A.Tk), 1 if gp else H_LT, exact, splits, op, s))
        worst = max(worst, r)
        if not r < 1.0:
            bad.append((s, r))
    print(f"{'deaot' if gp else 'aot'} {EXACT_IDS[0 if exact else 1]} {op} sweep: worst err / bound {worst:.3f}")
    assert not bad, f"(scale, err / bound) out of bounds: {bad}"


def gp_splits(N, Tk):
    """The DeAOT engine's split rule for the fused kernel (C = 256)."""
    from aot_benchmark_b200.engine import DeAOTEngine
    stub = SimpleNamespace(enc_hw=N, _plan=lambda: SimpleNamespace(C=256))
    return DeAOTEngine._gp_splits(stub, Tk)


ENGINE_N = 1674                    # 481 x 849 at stride 16: 31 x 54 tokens
ENGINE_TK = [ENGINE_N, 2 * ENGINE_N + 37]       # self-attention (Tk = N); a bank of two frames and a partial third


@pytest.mark.parametrize("Tk", ENGINE_TK, ids=["self", "bank"])
@pytest.mark.parametrize("gp,dv", ATTN, ids=ATTN_IDS)
def test_attention_engine_launches(gp, dv, Tk):
    """The engine's launches at N = 1674: the split count it takes (engine.lt_splits / the DeAOT rule), the live key count
    on the device under a larger bank capacity.  Both modes within attn_restatement's bound; fast and exact differ by more
    than four times the exact mode's own worst error, so the fast mode really drops the lo terms."""
    from aot_benchmark_b200.engine import lt_splits
    N = ENGINE_N
    splits = gp_splits(N, Tk) if gp else lt_splits(N, H_LT, Tk, variant="tile")
    Q, K, V = attn_inputs(N, Tk, gp, dv, 27)
    A = _Attn(Q.to(DEV), K.to(DEV), V.to(DEV), gp, kv_rows=3 * N)
    dev = torch.tensor([Tk], dtype=torch.int32, device=DEV)
    outs, errs = {}, {}
    for exact in (True, False):
        outs[exact] = A.run(exact=exact, Tk=Tk, Tk_dev=dev, splits=splits)
        ref, tol = packed_restatement(A, exact, Tk=Tk, splits=splits)
        errs[exact] = (outs[exact].double() - ref).abs().max().item()
        r = _ratio(outs[exact], ref, tol)
        print(f"{'deaot' if gp else 'aot'} N {N} Tk {Tk} splits {splits} {EXACT_IDS[0 if exact else 1]}: "
              f"worst err / bound {r:.3f}, max err {errs[exact]:.2e}")
        assert r < 1.0, (exact, r)
    diff = (outs[True] - outs[False]).abs().max().item()
    print(f"  max |fast - exact| {diff:.2e}")
    assert diff > 4 * errs[True], (diff, errs[True])
