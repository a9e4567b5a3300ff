"""CPU: negative controls for the bounds of tests/test_gpu_tc_operand_range.py and the fast-mode attention bounds of
tests/test_gpu_tc_envelope.py.

Each control restates, in float64, a plausible precision slip of a tensor-core kernel -- fp16 subnormals flushed to zero, the
single-pass rounding done toward zero, V rounded to fp16, Q divided by T after its split -- and shows that the slipped result
lies outside the GPU test's bound on that test's own inputs.  Where a bound cannot see a slip, the control says so and checks
that too.  No GPU is needed: the cases, references and bounds are the GPU modules' own, and the packed attention operands are
built with torch's CPU fp16 conversion, which rounds to nearest and keeps subnormals as the packing kernel does."""
import math

import pytest
import torch

import test_gpu_tc_envelope as EV
import test_gpu_tc_operand_range as OR

SUB = 2.0 ** -14          # smallest normal fp16


def _exceeds(mut, ref, tol):
    return ((mut - ref).abs() / tol).max().item()


def _flush(t):
    return torch.where(t.abs() < SUB, torch.zeros_like(t), t)


def _fp16_rz(x):
    """fp32 -> fp16 rounded toward zero (as float64): the mantissa truncated to 10 bits, or to a multiple of 2^-24 in the
    subnormal range."""
    x = x.float()
    bits = x.view(torch.int32) & ~((1 << 13) - 1)
    normal = bits.view(torch.float32).double()
    sub = torch.trunc(x.double() * 2.0 ** 24) * 2.0 ** -24
    r = torch.where(x.abs() >= SUB, normal, sub)
    assert (r.abs() <= x.double().abs()).all() and torch.equal(r.half().double(), r)
    return r


# ------------------------------------------------------------------ conv / linear
@pytest.mark.parametrize("kind", ["conv3x3", "linear"])
@pytest.mark.parametrize("slip,split,a", [("lo_flushed", True, -8), ("hi_lo_flushed", True, -20),
                                          ("hi_flushed", False, -16), ("round_toward_zero", False, 0)])
def test_conv_restatement_catches(kind, slip, split, a):
    """At the GPU sweep's own scales: a flushed subnormal lo (x 2^-8: hi normal, lo subnormal), flushed hi and lo
    (x 2^-20), a flushed single-pass hi (x 2^-16) and single-pass rounding toward zero (x 2^0) each land outside the
    restatement bound."""
    assert a in OR.A_SCALES
    c = OR.conv_case(kind)
    x = c.x * 2.0 ** a
    ref, tol = OR.conv_restatement(c, x, split, a=a)
    hi, lo = OR.split_x(x)
    if slip == "lo_flushed":
        assert (lo.abs() < SUB).all() and (lo != 0).any()
        mhi, mlo = hi, _flush(lo)
    elif slip == "hi_lo_flushed":
        mhi, mlo = _flush(hi), _flush(lo)
    elif slip == "hi_flushed":
        mhi, mlo = _flush(hi), lo
    else:
        mhi, mlo = _fp16_rz(x), lo
    mut, _ = OR.conv_restatement(c, x, split, hi=mhi, lo=mlo, a=a)
    r = _exceeds(mut, ref, tol)
    print(f"{kind} {slip}: worst err / bound {r:.1f}")
    assert r > 1.0, f"{slip} on {kind}: worst err / bound only {r:.3f}"


def test_conv_law_is_the_restatement_plus_operand_terms():
    """The law bound contains the restatement's, and the restatement's reference lies within the law (the operand terms
    cover the split and the weight rounding), at the small, middle and top scales."""
    for kind in ("conv3x3", "stem7x7"):
        c = OR.conv_case(kind)
        for split in (True, False):
            for a in (-24, -8, 0, 13):
                x = c.x * 2.0 ** a
                ref, tol = OR.conv_restatement(c, x, split, a=a)
                law, ltol = OR.conv_law(c, x, split, a=a)
                assert (ltol >= tol).all()
                assert _exceeds(ref, law, ltol - tol) < 1.0, (kind, split, a)


# ------------------------------------------------------------------ attention
def _pack(x, div=1.0):
    """(hi, lo) float64 of fp32 x / div as the packing kernel splits it."""
    y = x.float() / torch.tensor(div, dtype=torch.float32)
    hi = y.half()
    return hi.double(), (y - hi.float()).half().double()


def _problem(Q, K, V, gp):
    T = math.sqrt(128.0 if gp else 32.0)
    q, k, v = _pack(Q, T), _pack(K), _pack(V)
    return q, k, v[0] + v[1], (1 if gp else EV.H_LT)


@pytest.mark.parametrize("gp,dv", OR.ATTN, ids=OR.ATTN_IDS)
@pytest.mark.parametrize("op,s,exact,caught", [("Q", -2, True, True), ("Q", -12, True, True), ("V", -20, False, True),
                                               ("K", -6, True, False), ("Q", -12, False, False)])
def test_attention_subnormal_flush(gp, dv, op, s, exact, caught):
    """The GPU sweep's own inputs with the subnormal halves of one operand flushed to zero:
    - exact mode, Q 2^-2 (Q / T below 2^-3: lo subnormal, hi normal): lo flushed is outside attn_restatement's bound;
    - exact mode, Q 2^-12 (Q / T below 2^-14: hi subnormal too): hi and lo flushed is outside it;
    - fast mode, V 2^-20 (Vh subnormal): flushed is outside it.
    Not caught, and checked to be inside: K lo flushed at K 2^-6 (exact mode), and Q hi flushed at Q 2^-12 (fast mode).  With
    Q at the engine's magnitude the scores stay well below 1, so a 2^-12 relative change of small keys, or the loss of scores
    of size 2^-14, moves O by less than the bound's fp32 term (exact) or P's own 2^-11 rounding (fast).  A flushing wgmma
    would still show in the other rows, since the tensor core cannot tell which operand a subnormal came from."""
    assert s in OR.SWEEPS[op]
    Q, K, V = OR.sweep_inputs(op, s, gp, dv)
    q, k, v, heads = _problem(Q, K, V, gp)
    ref, tol = OR.sweep_restatement(q, k, v, heads, exact, 1, op, s)
    if op == "Q":
        q = (_flush(q[0]), _flush(q[1]))
    elif op == "K":
        k = (k[0], _flush(k[1]))
    else:
        vh, vl = _pack(V)
        v = _flush(vh) + _flush(vl)
    mut, _ = EV.attn_restatement(q, k, v, heads, exact)
    r = _exceeds(mut, ref, tol)
    print(f"{'deaot' if gp else 'aot'} {'exact' if exact else 'fast'} {op} 2^{s} flushed: worst err / bound {r:.2f}")
    assert (r > 1.0) == caught, r


@pytest.mark.parametrize("gp", [False, True], ids=["aot", "deaot"])
def test_vl_dropped_caught_by_closed_forms_only(gp):
    """V rounded to fp16 (Vl dropped) in the fast mode: the single-key and three-key closed forms of
    test_attention_closed_forms catch it; the fast-mode bound on the tile-edge grid does not (the P rounding it allows,
    2^-11 p_j |v_j|, exceeds the 2^-12 |v_j| of a dropped Vl), which is why the closed forms are there."""
    _, K, V = EV._qkv(65, 200, gp, 14)
    for tk in (1, 3):
        c = 2.0 ** -21 if tk == 1 else 2.0 ** -20
        tol = c * V[:tk].double().abs().mean(0) + 2.0 ** -25
        mut = V[:tk].half().double().mean(0)
        r = _exceeds(mut, V[:tk].double().mean(0), tol)
        assert r > 1.0, (tk, r)
    N, Tk = 129, 257
    Q, K, V = EV._qkv(N, Tk, gp, N * 1000 + Tk)
    q, k, v, heads = _problem(Q, K, V, gp)
    ref, tol = EV.attn_restatement(q, k, v, heads, False)
    mut, _ = EV.attn_restatement(q, k, _pack(V)[0], heads, False)
    assert _exceeds(mut, ref, tol) < 1.0


def _divide_after_split(Q, T):
    hi, lo = _pack(Q)
    return (hi.float() / torch.tensor(T, dtype=torch.float32)).half().double(), \
        (lo.float() / torch.tensor(T, dtype=torch.float32)).half().double()


@pytest.mark.parametrize("gp", [False, True], ids=["aot", "deaot"])
def test_q_divided_after_split(gp):
    """Q split first and each half divided by T afterwards: hi' = fp16(hi / T) carries up to 2^-12 relative error that
    lo' = fp16(lo / T) no longer compensates.  The restatement reads the packed values back, so it cannot see a packing slip;
    the exact mode's check against the unrounded float64 oracle (test_attention_tile_edges, 3e-5 / 5e-5) is what sees it,
    on each of these grid points."""
    T = math.sqrt(128.0 if gp else 32.0)
    tol = 5e-5 if gp else 3e-5
    caught = []
    for N, Tk in ((129, 63), (129, 257), (257, 129)):
        Q, K, V = EV._qkv(N, Tk, gp, N * 1000 + Tk)
        _, k, v, heads = _problem(Q, K, V, gp)
        mut, _ = EV.attn_restatement(_divide_after_split(Q, T), k, v, heads, True)
        err = (mut - EV._ref_for(Q, K, V, gp)).abs().max().item()
        caught.append(err / tol)
    print(f"{'deaot' if gp else 'aot'} Q divided after the split: err / tol {caught}")
    assert min(caught) > 1.0, caught
