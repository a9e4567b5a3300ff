"""GPU: the fp32 implicit-GEMM conv / linear (csrc/conv_igemm.cu) at the edges of its envelope, against float64.

conv2d_dispatch picks one of seven tile instantiations <BM, BN, TM, TN, AVEC, BVEC> from the operands' alignment, Cin, Cout
and the grid size, each with an h_swish twin.  `_igemm_variant` restates that rule; the case table reaches all seven, each
also with h_swish (checked when this module is imported), and a profiler test confirms that the rule names the kernel that
actually ran.  A variant is forced on a fixed problem with misaligned views: an input starting 1 float into its buffer
clears AVEC, weights at storage offset 1 clear BVEC, an output with ldout % 4 != 0 takes the scalar store.

Every variant computes one fmaf per k with k ascending from 0 and adds bias, residual and activation in the same order, so
the variants, the two store paths and repeated launches agree bit for bit, and scaling x, bias and residual by 2^k scales
the output exactly.  Against float64 every output stays within

  |y - y64| <= 2^-23 * (C_FIX + C_ACC * sqrt(K)) * mag,     mag = conv(|x|, |w|) + |b| + |res|   (float64)

- C_ACC = 2: the k-loop is a chain of K fp32 FMAs, each rounding by at most half an ulp of the running sum (<= mag / 2);
  independent roundings grow as sqrt(K), and 2 covers a 4-sigma excursion of that walk with room to spare.
- C_FIX = 3: the bias add, the residual add and the final rounding, one ulp of mag each.
- After an activation, slope * tol + 4 * 2^-23 * |pre-activation|: the slopes are 1 (ReLU, ReLU6), 1.13 (GELU, at
  sqrt(2)), 1.1 (SiLU) and 1.5 (h_swish, at 3); erff / expf / the h_sigmoid division add a few ulps.

tests/test_cpu_envelope_controls.py shows on the CPU that this bound catches a window shifted by one pixel, a dropped last
K chunk, a missing bias and a residual read from the next pixel on every case below."""
import math
import re

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
U = 2.0 ** -23
C_FIX, C_ACC = 3.0, 2.0
SLOPE = {0: 1.0, 1: 1.0, 2: 1.13, 3: 1.1, 4: 1.0, 5: 1.5}
ACT_NAMES = ("none", "relu", "gelu", "silu", "relu6", "hswish")


# ------------------------------------------------------------------ the dispatch rule
def _cdiv(a, b):
    return (a + b - 1) // b


def _igemm_variant(M, Cin, Cout, KH, KW, ldin, in_aligned, w_aligned):
    """conv2d_dispatch (csrc/conv_igemm.cu) restated: -> (BM, BN, TM, TN, AVEC, BVEC).  in_aligned / w_aligned: the input /
    weight base pointer is 16-byte aligned."""
    avec = in_aligned and ldin % 4 == 0 and Cin % 4 == 0 and (KH * KW == 1 or Cin % 16 == 0)
    bvec = Cout % 4 == 0 and w_aligned

    def ctas(bm, bn):
        return _cdiv(M, bm) * _cdiv(Cout, bn)

    if avec and bvec:
        if Cout >= 128 and ctas(128, 128) >= 132:
            return (128, 128, 8, 8, True, True)
        if Cout >= 64 and ctas(128, 64) >= 132:
            return (128, 64, 8, 4, True, True)
        return (64, 64, 4, 4, True, True)
    if avec:
        return (128, 32, 8, 2, True, False)
    if bvec:
        return (128, 64, 8, 4, False, True) if ctas(128, 64) >= 132 else (64, 64, 4, 4, False, True)
    return (128, 32, 8, 2, False, False)


ALL_VARIANTS = {(128, 128, 8, 8, True, True), (128, 64, 8, 4, True, True), (64, 64, 4, 4, True, True),
                (128, 32, 8, 2, True, False), (128, 64, 8, 4, False, True), (64, 64, 4, 4, False, True),
                (128, 32, 8, 2, False, False)}


# ------------------------------------------------------------------ cases
def _case(B, H, W, Cin, Cout, k=1, stride=1, pad=0, dil=1, act=0, res=None, bias=True, x=(0, 0), w=0, out=(0, 0)):
    """x / out / res = (shift, extra): the tensor starts `shift` floats into a flat buffer and its pixel stride is C + extra;
    res = "alias" makes the residual the output itself; w = storage offset of the [K, Cout] weights."""
    return dict(B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=k, stride=stride, pad=pad, dil=dil, act=act, res=res, bias=bias,
                x=x, w=w, out=out)


def _out_hw(c):
    e = c["dil"] * (c["k"] - 1) + 1
    return (c["H"] + 2 * c["pad"] - e) // c["stride"] + 1, (c["W"] + 2 * c["pad"] - e) // c["stride"] + 1


def _variant(c):
    Ho, Wo = _out_hw(c)
    return _igemm_variant(c["B"] * Ho * Wo, c["Cin"], c["Cout"], c["k"], c["k"], c["Cin"] + c["x"][1], c["x"][0] % 4 == 0,
                          c["w"] % 4 == 0)


CONV_CASES = [
    # M tails at the 64-row tile (vector A and B; vector A, scalar B with Cout 11)
    *[_case(1, M, 1, 40, 64, act=i % 6, res=(0, 0) if i % 2 else None) for i, M in enumerate((1, 63, 64, 65, 127, 128, 129))],
    *[_case(1, M, 1, 40, 11, act=(i + 3) % 6) for i, M in enumerate((1, 63, 64, 65, 127, 128, 129))],
    # the 132-CTA thresholds and M tails at the 128-row tiles
    _case(1, 8320, 1, 24, 72, act=1), _case(1, 8321, 1, 24, 72, act=5),                     # <64,64> | <128,64>
    _case(1, 8320, 1, 32, 256, act=0), _case(1, 8321, 1, 32, 256, act=5, res=(0, 0)),         # <128,64> | <128,128>
    _case(1, 8447, 1, 32, 256, act=2), _case(1, 8448, 1, 32, 256, act=1), _case(1, 8449, 1, 32, 196, act=3),
    _case(1, 8320, 1, 24, 128, act=0, x=(1, 0)), _case(1, 8321, 1, 24, 128, act=5, x=(1, 0)),   # scalar A: <64,64> | <128,64>
    _case(1, 8321, 1, 24, 72, act=4, x=(1, 0), res=(0, 0)),
    # Cout tails on a 3x3 (K = 144, K % 16 = 0)
    *[_case(1, 17, 23, 16, co, k=3, pad=1, act=i % 6, res=(0, 0) if i % 3 == 0 else None)
      for i, co in enumerate((11, 33, 65, 130, 190, 32, 64, 128, 256))],
    # K % 16 in {0, 3, 8}: pointwise Cin 32 / 19 / 24; MobileNetV3's pointwise widths (Cin % 16 != 0)
    _case(1, 31, 54, 32, 64, act=1), _case(1, 31, 54, 19, 64, act=0), _case(1, 31, 54, 24, 64, act=5),
    _case(1, 31, 54, 24, 72, act=5), _case(1, 31, 54, 40, 120, act=5), _case(1, 31, 54, 72, 24, act=0, res=(0, 0)),
    _case(1, 31, 54, 120, 480, act=5), _case(1, 16, 27, 184, 80, act=0, res=(0, 0)), _case(1, 16, 27, 200, 80, act=5),
    # 3x3 with vector A (Cin 32) and scalar A (Cin 24, K % 16 = 8); dilation 2, stride 2, batch 2
    _case(1, 23, 29, 32, 64, k=3, pad=1, act=1), _case(1, 23, 29, 24, 64, k=3, pad=1, act=5),
    _case(1, 23, 29, 32, 64, k=3, pad=2, dil=2, act=2), _case(1, 33, 47, 16, 48, k=3, stride=2, pad=1, act=3),
    _case(2, 19, 21, 32, 96, k=3, pad=1, act=4, res=(0, 0)), _case(2, 20, 20, 24, 40, k=3, stride=2, pad=1, act=5),
    # the 7x7 stride-2 stem (Cin 3 and 4; scalar A) at both sides of the scalar-A CTA threshold, and the MobileNetV3 stem
    _case(1, 97, 131, 3, 64, k=7, stride=2, pad=3, act=1), _case(1, 97, 131, 4, 64, k=7, stride=2, pad=3, act=1),
    _case(1, 259, 259, 4, 64, k=7, stride=2, pad=3, act=1), _case(1, 97, 131, 3, 16, k=3, stride=2, pad=1, act=5),
    # the dense ID-bank conv of probability masks: 17x17 / stride 16 / pad 8, Cin 11
    _case(1, 161, 241, 11, 256, k=17, stride=16, pad=8), _case(1, 33, 49, 11, 256, k=17, stride=16, pad=8, act=2),
    # column slices of wider NaN-filled buffers (aligned and misaligned), residual aliasing the output, no bias
    _case(1, 21, 27, 32, 64, k=3, pad=1, act=1, x=(4, 12), out=(8, 16), res=(16, 4)),
    _case(1, 21, 27, 32, 64, k=3, pad=1, act=2, x=(3, 5), out=(1, 3), res=(2, 6)),
    _case(1, 30, 53, 64, 256, act=1, x=(32, 64), out=(4, 36), res="alias"),
    _case(1, 30, 53, 24, 36, act=5, x=(8, 8), out=(5, 7), res="alias", w=1),
    _case(1, 30, 53, 40, 64, act=0, bias=False), _case(1, 9, 11, 19, 11, k=3, pad=1, act=5, bias=False, res=(1, 1)),
    # misaligned weights (scalar B) and both operands scalar
    _case(1, 31, 54, 32, 64, act=3, w=1), _case(1, 31, 54, 32, 64, act=5, w=1, x=(1, 0)),
    _case(1, 31, 54, 19, 11, act=5), _case(1, 13, 17, 24, 33, k=3, pad=1, act=4, x=(1, 0), w=3),
]
CONV_IDS = [f"c{i}-{c['B']}x{c['H']}x{c['W']}x{c['Cin']}-{c['Cout']}-k{c['k']}-{ACT_NAMES[c['act']]}"
            for i, c in enumerate(CONV_CASES)]

# (M, K, N, act, residual) through ops.linear: "res" a separate residual, "alias" the residual accumulated in place
LINEAR_CASES = [(1674, 256, 1024, 2, None), (1674, 1024, 256, 0, "alias"), (1, 256, 1024, 1, "res"), (1674, 256, 11, 0, None),
                (1, 40, 11, 5, None)]


def _covered():
    seen, seen_hs = set(), set()
    for c in CONV_CASES:
        v = _variant(c)
        seen.add(v)
        if c["act"] == 5:
            seen_hs.add(v)
    return seen, seen_hs


_SEEN, _SEEN_HS = _covered()
assert _SEEN == ALL_VARIANTS, f"case table misses {sorted(ALL_VARIANTS - _SEEN)}"
assert _SEEN_HS == ALL_VARIANTS, f"case table misses h_swish on {sorted(ALL_VARIANTS - _SEEN_HS)}"


# ------------------------------------------------------------------ inputs and the float64 reference
def case_inputs(c, seed=None):
    """-> x [B, H, W, Cin], w [Cout, Cin, k, k], b [Cout] or None, res [B, Ho, Wo, Cout] or None (float32, CPU)."""
    g = torch.Generator().manual_seed(seed if seed is not None else c["H"] * 131 + c["W"] * 7 + c["Cin"] * 3 + c["Cout"])
    Ho, Wo = _out_hw(c)
    k = c["k"]
    x = torch.randn(c["B"], c["H"], c["W"], c["Cin"], generator=g) * 2
    w = torch.randn(c["Cout"], c["Cin"], k, k, generator=g) / math.sqrt(c["Cin"] * k * k)
    b = torch.randn(c["Cout"], generator=g) if c["bias"] else None
    res = torch.randn(c["B"], Ho, Wo, c["Cout"], generator=g) if c["res"] is not None else None
    return x, w, b, res


def act64(y, act):
    return {0: lambda t: t, 1: F.relu, 2: F.gelu, 3: F.silu, 4: lambda t: t.clamp(0.0, 6.0),
            5: lambda t: t * (t + 3).clamp(0.0, 6.0) / 6}[act](y)


def conv_reference(x, w, b, res, stride, pad, dil, act):
    """float64 act(conv(x, w) + b + res) of float32 NHWC x and [Cout, Cin, k, k] w -> (y, tol), NHWC."""
    def conv(xx, ww, bb):
        return F.conv2d(xx.double().permute(0, 3, 1, 2), ww.double(), None if bb is None else bb.double(), stride, pad,
                        dil).permute(0, 2, 3, 1)

    pre = conv(x, w, b)
    mag = conv(x.abs(), w.abs(), None if b is None else b.abs())
    if res is not None:
        pre = pre + res.double()
        mag = mag + res.double().abs()
    K = w.shape[1] * w.shape[2] * w.shape[3]
    tol = U * (C_FIX + C_ACC * math.sqrt(K)) * mag
    if act != 0:
        tol = SLOPE[act] * tol + 4 * U * pre.abs()
    return act64(pre, act), tol


def pack_w(w):  # [Cout, Cin, KH, KW] -> [K, Cout] (k = (ky, kx, ci))
    co, ci, kh, kw = w.shape
    return w.permute(2, 3, 1, 0).reshape(kh * kw * ci, co).contiguous()


def worst_ratio(out, ref, tol):
    """max |out - ref| / tol (an exact element counts 0 even where tol is 0)."""
    assert torch.isfinite(out).all()
    err = (out.double() - ref).abs()
    return torch.where(err == 0, torch.zeros_like(err), err / tol).max().item()


# ------------------------------------------------------------------ placing operands in device buffers
def _place(t, shift, extra, fill=float("nan")):
    """t [..., C] -> (flat buffer, view): the view holds t, starts `shift` floats into a flat device buffer filled with `fill`
    and has pixel stride C + extra."""
    C = t.shape[-1]
    ld = C + extra
    n = t.numel() // C
    buf = torch.full((shift + n * ld + 8,), fill, device=DEV)
    view = buf[shift:shift + n * ld].view(*t.shape[:-1], ld)[..., :C]
    view.copy_(t.to(DEV))
    return buf, view


def _place_w(wk, offset):
    buf = torch.full((offset + wk.numel() + 8,), float("nan"), device=DEV)
    view = buf[offset:offset + wk.numel()].view(wk.shape)
    view.copy_(wk.to(DEV))
    return view


def _assert_untouched(buf, view, what):
    rest = buf.clone()
    rest.as_strided(view.shape, view.stride(), view.storage_offset()).fill_(float("nan"))
    assert torch.isnan(rest).all(), f"{what}: wrote outside its view"


def run_case(c, x, w, b, res, act=None, out_layout=None, w_offset=None, x_layout=None):
    """Runs ops.conv2d on the case's layout (overridable) -> output float32 [B, Ho, Wo, Cout] on the CPU."""
    from aot_benchmark_b200 import ops
    act = c["act"] if act is None else act
    xs, xe = c["x"] if x_layout is None else x_layout
    os_, oe = c["out"] if out_layout is None else out_layout
    _, xv = _place(x, xs, xe)
    wk = _place_w(pack_w(w), c["w"] if w_offset is None else w_offset)
    assert wk.data_ptr() not in ops._TC_WEIGHTS
    Ho, Wo = _out_hw(c)
    shape = (c["B"], Ho, Wo, c["Cout"])
    obuf, ov = _place(torch.zeros(shape), os_, oe)
    ov.fill_(float("nan"))
    rv = None
    if res is not None:
        if c["res"] == "alias":
            ov.copy_(res.to(DEV))
            rv = ov
        else:
            _, rv = _place(res, *c["res"])
    k = c["k"]
    ops.conv2d(xv, wk, None if b is None else b.to(DEV), ov, res=rv, KH=k, KW=k, stride=c["stride"], pad=c["pad"],
               dil=c["dil"], act=act)
    torch.cuda.synchronize()
    _assert_untouched(obuf, ov, "conv2d")
    return ov.cpu()


# ------------------------------------------------------------------ tests
@pytest.mark.parametrize("c", CONV_CASES, ids=CONV_IDS)
def test_conv_vs_float64(c):
    x, w, b, res = case_inputs(c)
    ref, tol = conv_reference(x, w, b, res, c["stride"], c["pad"], c["dil"], c["act"])
    out = run_case(c, x, w, b, res)
    r = worst_ratio(out, ref, tol)
    print(f"variant {_variant(c)}: worst err / tol {r:.3f}")
    assert r <= 1.0, f"variant {_variant(c)}: worst err / tol {r:.3f}"


def linear_inputs(M, K, N, rmode):
    """-> x [M, K], w [N, K], b [N], res [M, N] or None (float32, CPU)."""
    g = torch.Generator().manual_seed(M + K + N)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g) * 3 if rmode else None
    return x, w, b, res


@pytest.mark.parametrize("M,K,N,act,rmode", LINEAR_CASES)
def test_linear_vs_float64(M, K, N, act, rmode):
    """ops.linear (weights not registered for the tensor cores): the LSTT shapes, an in-place residual, M = 1 and N = 11."""
    from aot_benchmark_b200 import ops
    x, w, b, res = linear_inputs(M, K, N, rmode)
    ref, tol = conv_reference(x.view(1, M, 1, K), w.view(N, K, 1, 1), b, None if res is None else res.view(1, M, 1, N),
                              1, 0, 1, act)
    wk = w.t().contiguous().to(DEV)
    assert wk.data_ptr() not in ops._TC_WEIGHTS
    obuf, out = _place(torch.zeros(M, N), 4, 4 if N % 4 else 0)
    out.fill_(float("nan"))
    rv = None
    if rmode == "alias":
        out.copy_(res.to(DEV))
        rv = out
    elif rmode == "res":
        rv = res.to(DEV)
    ops.linear(x.to(DEV), wk, b.to(DEV), out, res=rv, act=act)
    torch.cuda.synchronize()
    _assert_untouched(obuf, out, "linear")
    r = worst_ratio(out.cpu().view(1, M, 1, N), ref, tol)
    print(f"linear {M}x{K}->{N}: worst err / tol {r:.3f}")
    assert r <= 1.0, r


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "conv_igemm_kernel" in e.name]


_NAME = re.compile(r"conv_igemm_kernel<\s*(\d+),\s*(\d+),\s*(\d+),\s*(\d+),\s*(true|false),\s*(true|false)"
                   r"(?:,\s*(true|false))?\s*>")


def _one_case_per_variant():
    """The first case of each variant, plus one with h_swish."""
    picked, hs = {}, {}
    for c in CONV_CASES:
        v = _variant(c)
        (hs if c["act"] == 5 else picked).setdefault(v, c)
    return [picked[v] for v in sorted(picked)] + [hs[v] for v in sorted(hs)]


def test_dispatch_mirror_names_the_launched_kernel():
    """One case per variant (and per variant with h_swish) under torch.profiler: the launched kernel's template arguments are
    what _igemm_variant says, and the h_swish twin runs exactly when act = 5."""
    seen = set()
    for c in _one_case_per_variant():
        x, w, b, res = case_inputs(c)
        names = _kernel_names(lambda: run_case(c, x, w, b, res))
        assert len(names) == 1, names
        m = _NAME.search(names[0])
        assert m, names[0]
        got = tuple(int(m.group(i)) for i in range(1, 5)) + (m.group(5) == "true", m.group(6) == "true")
        assert got == _variant(c), (names[0], c)
        assert (m.group(7) == "true") == (c["act"] == 5), names[0]
        seen.add((got, c["act"] == 5))
    print("profiler saw:", sorted(seen))
    assert {v for v, _ in seen} == ALL_VARIANTS


# fixed problems, each run under every alignment layout: (input shift, weight offset) x (output pixel stride % 4 == 0 or not)
FIXED = [_case(1, 13, 17, 32, 64, k=3, pad=1, res=(0, 0)),          # small grid: <64,64> / <128,32> variants
         _case(1, 8321, 1, 32, 256, res=(0, 0)),                     # large grid: <128,128> / <128,64> / <128,32>
         _case(2, 11, 9, 16, 36, k=3, stride=2, pad=1, res=(0, 0))]   # Cout 36: a partial N tile in every variant
LAYOUTS = [((0, 0), 0), ((1, 0), 0), ((0, 0), 1), ((1, 0), 1)]


@pytest.mark.parametrize("fi", range(len(FIXED)))
def test_variants_bitwise_equal(fi):
    """All alignment variants, with the vector and scalar stores, and a repeated launch give the same bits; act = 5 equals
    h_swish written in float32 (true division) on the act = 0 output."""
    c = FIXED[fi]
    x, w, b, res = case_inputs(c, seed=fi)
    base = run_case(c, x, w, b, res, act=0)
    variants = set()
    for xl, wo in LAYOUTS:
        for ol in ((0, 0), (1, 3)):                                  # ovec on, ovec off
            cc = dict(c, x=xl, w=wo)
            variants.add(_variant(cc))
            out = run_case(cc, x, w, b, res, act=0, out_layout=ol)
            assert torch.equal(out, base), (xl, wo, ol, _variant(cc))
    assert len(variants) == 4
    assert torch.equal(run_case(c, x, w, b, res, act=0), base)
    hs = run_case(c, x, w, b, res, act=5)
    y = base.to(DEV)
    want = y * torch.div(torch.clamp(y + 3, 0, 6), torch.full_like(y, 6.0))
    assert torch.equal(hs, want.cpu())
    ref, tol = conv_reference(x, w, b, res, c["stride"], c["pad"], c["dil"], 0)
    assert worst_ratio(base, ref, tol) <= 1.0


@pytest.mark.parametrize("k", [-40, -20, -10, 10, 20, 40])
@pytest.mark.parametrize("act", [0, 1])
def test_power_of_two_scale_equivariance(k, act):
    """x, bias and residual scaled by 2^k: every variant's output is exactly 2^k times the unscaled output."""
    s = 2.0 ** k
    for fi in (0, 2):
        c = FIXED[fi]
        x, w, b, res = case_inputs(c, seed=fi)
        for xl, wo in LAYOUTS:
            cc = dict(c, x=xl, w=wo)
            base = run_case(cc, x, w, b, res, act=act)
            scaled = run_case(cc, x * s, w, b * s, res * s, act=act)
            assert torch.equal(scaled, base * s), (k, act, _variant(cc))
