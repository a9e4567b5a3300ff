"""CPU: negative controls for the law of the tensor-core local attention (tests/test_gpu_local_attn_tc_range.py local_law,
the bound of tests/test_gpu_local_attn_tc.py).

Each control restates in float64 the kernel with one plausible slip -- q divided by T after its split, P rounded to fp16 in
P V or in P relv, relv rounded to fp16, fp16 subnormals flushed in the K or V split, the padding tap dx = 15 given a finite
score, the right-edge mask off by one -- and shows that the slipped output lies outside the law on the GPU module's own
inputs (its operand sweep at the scale named).  No GPU is needed: the law runs on the CPU, and torch's CPU fp16 conversion
rounds to nearest and keeps subnormals, as the kernel's cvt does."""
import pytest
import torch
import torch.nn.functional as F

import test_gpu_local_attn_tc_range as LR

H, D, C = LR.H, LR.D, LR.C
SUB = 2.0 ** -14          # smallest normal fp16
T32 = torch.sqrt(torch.tensor(32.0))        # sqrtf(32), as the kernel's T
MAP = LR.SWEEP_MAPS[1]


def _split(x):
    """(hi, lo) float64 of fp32 x split as the kernel's cvt does."""
    hi = x.float().half()
    return hi.double(), (x.float() - hi.float()).half().double()


def _flush(t):
    return torch.where(t.abs() < SUB, torch.zeros_like(t), t)


def _taps(x, h, w, ncol, right=8):
    """x [c, h, w + 8 - right] -> [c, 15, ncol, h, w]: x at (y + dy - 7, x + dx - 7), zero outside (the halo)."""
    xp = F.pad(x, (8, right, 7, 7))
    return torch.stack([torch.stack([xp[:, dy:dy + h, dx + 1:dx + 1 + w] for dx in range(ncol)], 1) for dy in range(15)], 1)


def local64(x, slip=None):
    """float64 restatement of local_attn_mma_kernel over inputs {q, k, v, relk_w, relk_b, relv} (local_law's layout), the
    operands exact except where `slip` changes them -> [hw, H*D]."""
    q, k, v = (x[nm][0].double() for nm in ("q", "k", "v"))
    h, w = q.shape[1], q.shape[2]
    n = h * w
    qs = (x["q"][0].float() / T32).double()                         # q / T in fp32 before the split
    relv = x["relv"].double()
    if slip == "q_divided_after_split":
        hi, lo = _split(x["q"][0])
        qs = (hi.float() / T32).half().double() + (lo.float() / T32).half().double()
    elif slip == "k_flushed":
        k = sum(_flush(t) for t in _split(x["k"][0]))
    elif slip == "v_flushed":
        v = sum(_flush(t) for t in _split(x["v"][0]))
    elif slip == "relv_fp16":
        relv = x["relv"].half().double()
    ncol = 16 if slip == "pad_tap_finite" else 15                   # tap dx = 15: key and value at x + 8
    kt = _taps(k, h, w, ncol).reshape(H, D, 15, ncol, n)
    vt = _taps(v, h, w, ncol).reshape(H, D, 15, ncol, n)
    ones = torch.ones(1, h, w + (1 if slip == "mask_right_edge_le_w" else 0), dtype=torch.float64)
    inside = _taps(ones, h, w, ncol, right=7 if slip == "mask_right_edge_le_w" else 8).reshape(1, 15, ncol, n)
    rel = F.conv2d(q[None], x["relk_w"].double(), x["relk_b"].double(), groups=H).view(H, 15, 15, n)
    rv = relv.view(H, D, 15, 15)
    if ncol == 16:                                                  # the padding tap's relk_w, bias and relv are zero
        rel, rv = F.pad(rel, (0, 0, 0, 1)), F.pad(rv, (0, 1))
    s = torch.einsum("hdn,hdyxn->hyxn", qs.reshape(H, D, n), kt) + rel - (1 - inside) * 1e8
    p = torch.exp(s - s.amax((1, 2), keepdim=True))
    l = p.sum((1, 2))
    p_v = p.float().half().double() if slip == "p_fp16_in_pv" else p
    p_r = p.float().half().double() if slip == "p_fp16_in_prelv" else p
    o = (torch.einsum("hyxn,hdyxn->hdn", p_v, vt) + torch.einsum("hyxn,hdyx->hdn", p_r, rv)) / l.unsqueeze(1)
    return o.permute(2, 0, 1).reshape(n, C)


def _ratio(x, slip):
    ref, tol = LR.local_law(x["q"], x["k"], x["v"], x["relk_w"], x["relk_b"], x["relv"], "cpu")
    return LR.ratio(local64(x, slip), ref, tol)


def test_restatement_without_slip_is_inside():
    """The restatement itself, without a slip, lies well inside the law (it differs from the oracle only by q / T in fp32)."""
    for op, s in (("q", 0), ("k", -16), ("v", -14), ("q", 5)):
        r = _ratio(LR.sweep_inputs(op, s, *MAP), None)
        print(f"no slip, {op} 2^{s}: err / bound {r:.3f}")
        assert r < 0.1, (op, s, r)


# slip, swept operand and scale (one of the GPU sweep's), caught by the law.  P rounded in P relv is caught once relv
# carries the output (2^8; at its base magnitude 0.3 the rounding, 2^-12 p_j |relv_j|, stays below the 2^-25 floor of
# the 225 taps' |u_j|).
CONTROLS = [("q_divided_after_split", "q", 0), ("q_divided_after_split", "q", 5), ("p_fp16_in_pv", "v", 0),
            ("p_fp16_in_prelv", "relv", 8), ("relv_fp16", "relv", 0), ("v_flushed", "v", -16), ("v_flushed", "v", -14),
            ("pad_tap_finite", "q", 0), ("mask_right_edge_le_w", "q", 0)]


@pytest.mark.parametrize("slip,op,s", CONTROLS, ids=[f"{c[0]}-{c[1]}{c[2]}" for c in CONTROLS])
def test_slip_is_outside_the_law(slip, op, s):
    assert s in (LR.B_SCALES if op == "relk_b" else LR.S_SCALES)
    x = LR.sweep_inputs(op, s, *MAP)
    r = _ratio(x, slip)
    print(f"{slip} ({op} 2^{s}, {MAP[0]}x{MAP[1]}): worst err / bound {r:.1f}")
    assert r > 1.0, f"{slip}: worst err / bound only {r:.3f}"


def test_k_flush_is_below_the_law():
    """fp16 subnormals of k flushed (hi and lo, k 2^-14 .. 2^-16): NOT caught, and checked to be inside.  With q at its base
    magnitude the whole dot product (q / T) . k is then about 2^-15, below the score allowance the law gives the fp32 sum of
    the relative-key term (2^-23 (8 + 4 sqrt(32)) sum |q| |relk_w| ~ 2^-16 per tap).  A flushing mma.sync would still show
    in the V sweep (caught above) and in P, whose lo halves are subnormal at every scale: the tensor core cannot tell which
    operand a subnormal came from."""
    for s in (-16, -14):
        r = _ratio(LR.sweep_inputs("k", s, *MAP), "k_flushed")
        print(f"k_flushed (k 2^{s}): worst err / bound {r:.3f} (below the law)")
        assert r < 1.0, (s, r)
