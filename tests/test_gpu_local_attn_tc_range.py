"""GPU: the tensor-core short-term local attention (local_attn_mma_kernel, AOT head shape) across operand magnitude, at its
window and map edges, in the engines' own launches, and the batched entry points (one launch over several videos) against
float64.

local_law is the split-fp16 law of tests/test_gpu_local_attn_tc.py (DESIGN 3.2), over arbitrary q, k, v, relative_emb_k
weights and bias and relative_emb_v, on any device; tests/test_cpu_local_attn_tc_controls.py shows on this module's inputs
that plausible slips of the kernel land outside it.

  operand sweep    q, k, v, relk_w and relv scaled one at a time by 2^s, s = -24 .. 13 (randn clamped to |x| <= 7, the
                   others at the magnitudes of test_gpu_local_attn_tc), relk_b up to 2^6 (the bias dominates the softmax),
                   at two maps with partial 8-row and 16-column tiles: finite and within the law at every scale.  Below
                   2^-14 every hi of the swept operand is an fp16 subnormal, so a tensor core that flushed them would be
                   caught there (the controls measure by how much).
  top edge         q, k, v or relv with |x| up to 65519.99 (hi = 65504): finite and within the law.
  exchange         q 2^a with k 2^-a and relk_w 2^-a (relk_b unchanged), a = -2 .. 2, on operands whose halves -- and those
                   of fl32(q / T) -- stay normal fp16 (or zero) throughout: the same output bit for bit.  Every product
                   pairs a half of one operand with a half of its partner, so a half paired with the wrong operand, or a
                   term that does not scale with its operands, breaks it.
  poison           q, k, v as row and column slices of NaN buffers: bitwise the clean output, nothing written outside out.
  engine launches  every local_attention_tc call of R50-AOTL (31 x 54) and SwinB-AOTL (37 x 65), fp32, and R50-AOTL fp16.
  batched          local_attention_tc_batched over n maps of their own content: each within the law and bitwise the
                   one-video launch, rows and columns past the last map untouched; lt_attention_tc_batched at the
                   multi-video engine's size (n = 8, N = 1674), bank and self-attention forms, within
                   test_gpu_tc_envelope.attn_restatement's bound per problem and bitwise the one-video launch.

Measured on an H100 80GB HBM3 (700 W): see DESIGN.md section 3.2."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
H, D, P = 8, 32, 225
C = H * D
SWEEP_MAPS = [(13, 22), (9, 17)]           # partial 8-row and 16-column tiles
S_SCALES = list(range(-24, 14))            # randn clamped to |x| <= 7: max 7 2^13 = 57344 < 65504
B_SCALES = list(range(-24, 7, 3))          # relative_emb_k bias: 0.1 randn 2^6 dominates the scores
BASE = {"q": 1.0, "k": 1.0, "v": 1.0, "relk_w": 0.2, "relk_b": 0.1, "relv": 0.3}
NAMES = list(BASE)


def _dev():
    return torch.device("cuda:0")


# ------------------------------------------------------------------ the law
def local_law(q, k, v, rkw, rkb, rv, dev):
    """float64 oracle output [hw, H*D] and the split-fp16 bound of tests/test_gpu_local_attn_tc.py, both on `dev`, for
    q, k, v [1, H*D, h, w], rkw [H*225, D, 1, 1], rkb [H*225], rv [H, D, 225].  Per (query, head), with S_j the magnitude of
    tap j's score and F_j the operands under the 2^-25 floor:
      ds = max_j 2^-21 S_j + 2^-25 F_j + 2^-23 (8 + 4 sqrt(32)) S_j
      |o - o64| <= (2 ds + 2^-21 + 2^-23 (8 + 2 sqrt(225))) sum_j p_j |u_j| + 2^-25 sum_j |u_j|,  |u_j| = |v_j| + |relv_j|."""
    from oracle import aot_oracle as O
    h, w = q.shape[2], q.shape[3]
    T = math.sqrt(D)
    q64, k64, v64, w64, b64, rv64 = (t.to(dev, torch.float64) for t in (q, k, v, rkw, rkb, rv))
    out = O.local_attention(q64, k64, v64, w64, b64, rv64, H)[:, 0]
    n = h * w
    rel = F.conv2d(q64, w64, b64, groups=H).view(H, P, n)
    relmag = F.conv2d(q64.abs(), w64.abs(), b64.abs(), groups=H).view(H, P, n)
    relfl = F.conv2d(q64.abs(), torch.ones_like(w64), None, groups=H).view(H, P, n) + w64.abs().sum((1, 2, 3)).view(H, P, 1)
    ku = F.unfold(k64, 15, padding=7).view(H, D, P, n)
    qv = (q64 / T).view(H, D, n)
    s = torch.einsum("hdn,hdpn->hpn", qv, ku) + rel
    inside = F.unfold(torch.ones(1, 1, h, w, dtype=torch.float64, device=dev), 15, padding=7).view(1, P, n)
    p = torch.softmax(s - (1 - inside) * 1e8, dim=1)
    S = torch.einsum("hdn,hdpn->hpn", qv.abs(), ku.abs()) + relmag
    Fl = qv.abs().sum(1, keepdim=True) + ku.abs().sum(1) + relfl
    ds = ((2 ** -21 + U * (8 + 4 * math.sqrt(D))) * S + 2 ** -25 * Fl).amax(1)                  # [H, n]
    vu = F.unfold(v64.abs(), 15, padding=7).view(H, D, P, n) + rv64.abs().unsqueeze(-1)          # |u_j| per channel
    pu = torch.einsum("hpn,hdpn->hdn", p, vu)
    tol = (2 * ds.unsqueeze(1) + 2 ** -21 + U * (8 + 2 * math.sqrt(P))) * pu + 2 ** -25 * vu.sum(2)
    return out, tol.permute(2, 0, 1).reshape(n, H * D)


def law_tokens(qt, kt, vt, w2, b2, rvt, h, w, dev):
    """local_law over the kernel's own arguments: q, k, v [hw, H*D] tokens, relk_w [H*225, D], relk_b [H*225] and
    relv_t [H, 225, D]."""
    m = lambda t: t.double().t().reshape(1, C, h, w)
    return local_law(m(qt), m(kt), m(vt), w2.view(H * P, D, 1, 1), b2, rvt.permute(0, 2, 1), dev)


def ratio(out, ref, tol):
    return ((out.double().to(ref.device) - ref).abs() / tol).max().item()


# ------------------------------------------------------------------ inputs and launches
def base_inputs(h, w, seed, clamp=False):
    """{name: tensor} at the magnitudes of test_gpu_local_attn_tc (randn clamped to |x| <= 7 when `clamp`)."""
    g = torch.Generator().manual_seed(seed)
    shapes = {"q": (1, C, h, w), "k": (1, C, h, w), "v": (1, C, h, w), "relk_w": (H * P, D, 1, 1), "relk_b": (H * P,),
              "relv": (H, D, P)}
    r = lambda s: torch.randn(*s, generator=g).clamp(-7.0, 7.0) if clamp else torch.randn(*s, generator=g)
    return {nm: r(shapes[nm]) * BASE[nm] for nm in NAMES}


def sweep_inputs(op, s, h, w, seed=None):
    """base_inputs (clamped) with operand `op` scaled by 2^s (exact)."""
    x = base_inputs(h, w, h * 100 + w if seed is None else seed, clamp=True)
    x[op] = x[op] * 2.0 ** s
    return x


def tok(t):
    return t[0].permute(1, 2, 0).reshape(t.shape[2] * t.shape[3], -1).contiguous()


def kernel_args(x, dev):
    """q, k, v tokens [hw, H*D] and relk_w [H*225, D], relk_b, relv_t [H, 225, D] on `dev`."""
    return (tok(x["q"]).to(dev), tok(x["k"]).to(dev), tok(x["v"]).to(dev), x["relk_w"].view(H * P, D).contiguous().to(dev),
            x["relk_b"].to(dev), x["relv"].permute(0, 2, 1).contiguous().to(dev))


def run_local(qt, kt, vt, w2, b2, rvt, h, w, c0=36):
    """ops.local_attention_tc into columns [c0, c0 + H*D) of a NaN buffer; asserts nothing was written outside them."""
    from aot_benchmark_b200 import ops
    ob = torch.full((h * w, C + 40), float("nan"), device=_dev())
    ops.local_attention_tc(qt, kt, vt, w2, b2, rvt, ob[:, c0:c0 + C], h, w, H)
    torch.cuda.synchronize()
    assert torch.isnan(ob[:, :c0]).all() and torch.isnan(ob[:, c0 + C:]).all(), "wrote outside its columns"
    return ob[:, c0:c0 + C]


def _law_run(x, h, w):
    d = _dev()
    args = kernel_args(x, d)
    out = run_local(*args, h, w)
    return out, local_law(x["q"], x["k"], x["v"], x["relk_w"], x["relk_b"], x["relv"], d)


# ------------------------------------------------------------------ operand sweep and top edge
@pytest.mark.parametrize("op", NAMES)
@pytest.mark.parametrize("h,w", SWEEP_MAPS)
def test_operand_scale_sweep(h, w, op):
    """One operand at 2^s (relk_b up to 2^6): finite and within local_law at every scale.  The worst ratio is printed for
    the scales where the swept operand's hi halves are fp16 subnormals (s <= -14) and above."""
    worst = {True: 0.0, False: 0.0}
    bad = []
    for s in (B_SCALES if op == "relk_b" else S_SCALES):
        out, (ref, tol) = _law_run(sweep_inputs(op, s, h, w), h, w)
        r = ratio(out, ref, tol)
        worst[s <= -14] = max(worst[s <= -14], r)
        if not (torch.isfinite(out).all() and r <= 1.0):
            bad.append((s, r))
    print(f"{h}x{w} {op} sweep: worst err / bound {worst[True]:.3f} (s <= -14), {worst[False]:.3f} (s > -14)")
    assert not bad, f"(scale, err / bound) out of bounds: {bad}"


@pytest.mark.parametrize("op", ["q", "k", "v", "relv"])
def test_top_edge(op):
    """q, k, v or relv replaced by top_edge_input (|x| < 65520, hi = 65504 at the top): finite, within local_law."""
    from test_gpu_tc_operand_range import top_edge_input
    h, w = 13, 22
    x = base_inputs(h, w, 5)
    x[op] = top_edge_input(x[op].shape, 6)
    out, (ref, tol) = _law_run(x, h, w)
    assert torch.isfinite(out).all()
    r = ratio(out, ref, tol)
    print(f"{op} top edge: worst err / bound {r:.3f}")
    assert r <= 1.0, r


# ------------------------------------------------------------------ exchange equivariance
EXCHANGE = range(-2, 3)


def exchange_q(shape, seed):
    """fp32 q whose halves stay normal fp16 (or lo zero) under 2^a, a in EXCHANGE, and whose fl32(q / T) is an fp16 value
    (zero lo) in +-[2^-3, 2^-2): q = fl32(h T) for fp16 h, kept where fl32(q / T) == h (IEEE division, T = sqrtf(32))
    and q - fp16(q) is 0 or at least 2^-12."""
    g = torch.Generator().manual_seed(seed)
    T = torch.sqrt(torch.tensor(32.0))
    n = math.prod(shape)
    sign = torch.randint(0, 2, (10 * n,), generator=g).float() * 2 - 1
    hv = ((1 + torch.rand(10 * n, generator=g)) * 0.125 * sign).half().float()
    q = hv * T
    r = q - q.half().float()
    ok = (q / T == hv) & ((r == 0) | (r.abs() >= 2.0 ** -12)) & (hv.abs() >= 0.125)
    assert ok.sum().item() >= n, ok.sum().item()
    return q[ok][:n].view(shape)


def _split(x):
    hi = x.half()
    return hi.float(), (x - hi.float()).half().float()


def _check_exchange_halves(q, k, rkw):
    """Every half the kernel multiplies -- of q, fl32(q / T), k and relk_w -- scales exactly with its operand."""
    T = torch.sqrt(torch.tensor(32.0))
    for a in EXCHANGE:
        f = 2.0 ** a
        for x0, x, s in ((q, q * f, f), (q / T, q * f / T, f), (k, k / f, 1 / f), (rkw, rkw / f, 1 / f)):
            (h0, l0), (h1, l1) = _split(x0), _split(x)
            assert torch.equal(h1, h0 * s) and torch.equal(l1, l0 * s), a
            assert h1.abs().max().item() <= 65504, a


@pytest.mark.parametrize("h,w", SWEEP_MAPS)
def test_exchange_equivariance(h, w):
    """q 2^a, k 2^-a, relk_w 2^-a, relk_b unchanged: every score product is the same, so the output is bitwise the same.
    relk_w has two non-zero channels per tap in sixteen, so the scores stay O(1) and the softmax is not one-hot."""
    from test_gpu_tc_operand_range import exact_pairs
    x = base_inputs(h, w, 31)
    q = exchange_q((1, C, h, w), 32)
    k = exact_pairs((1, C, h, w), 33)
    g = torch.Generator().manual_seed(34)
    rkw = exact_pairs((H * P, D, 1, 1), 35) * (torch.rand(H * P, D, 1, 1, generator=g) < 1 / 16).float()
    _check_exchange_halves(q, k, rkw)
    d = _dev()
    outs = {}
    for a in EXCHANGE:
        x.update(q=q * 2.0 ** a, k=k * 2.0 ** -a, relk_w=rkw * 2.0 ** -a)
        outs[a] = run_local(*kernel_args(x, d), h, w).clone()
        assert torch.isfinite(outs[a]).all()
    x.update(q=q, k=k, relk_w=rkw)
    ref, tol = local_law(x["q"], x["k"], x["v"], x["relk_w"], x["relk_b"], x["relv"], d)
    print(f"{h}x{w} exchange: worst err / bound {ratio(outs[0], ref, tol):.3f}")
    assert ratio(outs[0], ref, tol) <= 1.0
    for a in EXCHANGE:
        assert torch.equal(outs[a], outs[0]), f"q 2^{a}, k and relk_w 2^{-a} changed the output"


# ------------------------------------------------------------------ poisoned surroundings
def _in_nan(t, r0=37, c0=8):
    """t [rows, cols] as the slice [r0, r0 + rows) x [c0, c0 + cols) of a NaN buffer with rows and columns on every side."""
    buf = torch.full((t.shape[0] + r0 + 41, t.shape[1] + c0 + 24), float("nan"), device=t.device)
    buf[r0:r0 + t.shape[0], c0:c0 + t.shape[1]] = t
    return buf[r0:r0 + t.shape[0], c0:c0 + t.shape[1]]


@pytest.mark.parametrize("h,w", [(13, 22), (9, 17), (3, 1), (31, 54)])
def test_poisoned_surroundings(h, w):
    """q, k and v as slices of NaN buffers (NaN rows before and after the map, NaN columns beside it): bitwise the clean
    output, and out's own buffer keeps its NaN rows and columns."""
    from aot_benchmark_b200 import ops
    x = base_inputs(h, w, 41)
    qt, kt, vt, w2, b2, rvt = kernel_args(x, _dev())
    clean = run_local(qt, kt, vt, w2, b2, rvt, h, w).clone()
    ob = _in_nan(torch.full((h * w, C), float("nan"), device=_dev()), 29, 12)
    ops.local_attention_tc(_in_nan(qt), _in_nan(kt, 5, 4), _in_nan(vt, 61, 16), w2, b2, rvt, ob, h, w, H)
    torch.cuda.synchronize()
    assert torch.equal(ob, clean)
    base = ob._base
    inside = torch.zeros_like(base, dtype=torch.bool)
    inside[29:29 + h * w, 12:12 + C] = True
    assert torch.isnan(base[~inside]).all(), "wrote outside out"


# ------------------------------------------------------------------ engine launches
ENGINES = [("r50_aotl", (481, 849), (31, 54), "fp32"), ("r50_aotl", (481, 849), (31, 54), "fp16"),
           ("swinb_aotl", (592, 1040), (37, 65), "fp32")]


@pytest.mark.parametrize("model,size,hw,precision", ENGINES, ids=["r50_aotl", "r50_aotl-fp16", "swinb_aotl"])
def test_engine_launches(monkeypatch, model, size, hw, precision):
    """A reference frame and two propagated frames on random weights, graphs off: every local_attention_tc call the engine
    makes is within local_law on its own arguments (in fp16 mode the local kernel is the same split-fp16 kernel, on
    operands from fp16-mode convolutions)."""
    from aot_benchmark_b200 import engine, ops
    from oracle import aot_oracle as O
    from oracle import weights as OW
    import fp16_support as F16
    monkeypatch.setattr(engine, "USE_GRAPHS", False)
    calls = []
    orig = ops.local_attention_tc

    def record(q, k, v, relk_w, relk_b, relv_t, out, h, w, Hh, stream=None):
        r = orig(q, k, v, relk_w, relk_b, relv_t, out, h, w, Hh, stream=stream)
        torch.cuda.synchronize()
        calls.append(tuple(t.clone() for t in (q, k, v, relk_w, relk_b, relv_t, out)) + (h, w, Hh))
        return r

    monkeypatch.setattr(ops, "local_attention_tc", record)
    sd = OW.build_state_dict(model, seed=3)
    eng = F16.build_engine(model, sd, 1, precision, device="cuda")
    frames, mask = O.synthetic_video(3, *size, 3, seed=5)
    with torch.no_grad():
        O.run_video(eng, [f.cuda() for f in frames], mask.cuda(), 3, size)
    torch.cuda.synchronize()
    assert len(calls) >= 6, len(calls)
    worst = 0.0
    for q, k, v, w2, b2, rvt, out, h, w, Hh in calls:
        assert (h, w) == hw and Hh == H
        assert torch.isfinite(out).all()
        r = ratio(out, *law_tokens(q, k, v, w2, b2, rvt, h, w, _dev()))
        worst = max(worst, r)
        assert r <= 1.0, r
    print(f"{model} {precision}: {len(calls)} local_attention_tc calls at {hw[0]}x{hw[1]}, worst err / bound {worst:.3f}")


# ------------------------------------------------------------------ batched local attention
BATCH_MAPS = [(3, 1), (5, 40), (9, 17), (31, 54), (37, 65)]


@pytest.mark.parametrize("n", [1, 2, 5, 8])
@pytest.mark.parametrize("h,w", BATCH_MAPS)
def test_local_batched_vs_float64(h, w, n):
    """n maps stacked along the rows, each its own content (map n // 2 with q at scale 30): each map within local_law and
    bitwise the one-video launch on its rows; rows and columns past the last map stay NaN."""
    from aot_benchmark_b200 import ops
    d = _dev()
    m = h * w
    xs = []
    for b in range(n):
        x = base_inputs(h, w, 1000 * n + 10 * b + h)
        if b == n // 2:
            x["q"] = x["q"] * 30.0
        xs.append(x)
    shared = {nm: xs[0][nm] for nm in ("relk_w", "relk_b", "relv")}
    for x in xs:
        x.update(shared)
    cat = lambda nm: torch.cat([tok(x[nm]) for x in xs]).to(d)
    q, k, v = _in_nan(cat("q")), _in_nan(cat("k")), _in_nan(cat("v"))
    _, _, _, w2, b2, rvt = kernel_args(xs[0], d)
    ob = torch.full((n * m + 29, C + 44), float("nan"), device=d)
    out = ob[:n * m, 4:4 + C]
    ops.local_attention_tc_batched(q, k, v, w2, b2, rvt, out, h, w, H, n)
    torch.cuda.synchronize()
    assert torch.isnan(ob[n * m:]).all() and torch.isnan(ob[:, :4]).all() and torch.isnan(ob[:, 4 + C:]).all(), \
        "wrote outside out"
    worst = 0.0
    for b, x in enumerate(xs):
        rows = slice(b * m, (b + 1) * m)
        one = run_local(q[rows], k[rows], v[rows], w2, b2, rvt, h, w)
        assert torch.equal(out[rows], one), b
        r = ratio(out[rows], *local_law(x["q"], x["k"], x["v"], x["relk_w"], x["relk_b"], x["relv"], d))
        worst = max(worst, r)
        assert r <= 1.0, (b, r)
    print(f"batched local {h}x{w} n {n}: worst err / bound {worst:.3f}")


# ------------------------------------------------------------------ batched long-term attention at the engine's size
LT_N, LT_M, LT_VIDEOS = 1674, 3, 8


@pytest.mark.parametrize("form", ["bank", "self"])
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
def test_lt_batched_engine_size(form, exact):
    """lt_attention_tc_batched as MultiVideoInferEngine runs it: n = 8 problems of N = 1674 queries (q_stride = N), keys
    from a pooled bank (kv_stride = M N, M = 3, live counts from one frame to a full bank, splits = lt_splits(n N, 8,
    max live)) or the problems' own frames (Tk = kv_stride = N, splits = lt_splits(n N, 8, N)).  Each problem within
    attn_restatement's bound over its packed operands and bitwise its one-video lt_attention_tc launch."""
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200.engine import lt_splits
    from test_gpu_tc_envelope import attn_restatement, unpack
    d = _dev()
    n, N = LT_VIDEOS, LT_N
    g = torch.Generator(device=d).manual_seed(51 + exact)
    if form == "bank":
        kvs = LT_M * N
        live = [N + (b * (kvs - N)) // (n - 1) for b in range(n)]
        tk_dev = torch.tensor(live, dtype=torch.int32, device=d)
        splits = lt_splits(n * N, H, max(live))
    else:
        kvs, live, tk_dev = N, [N] * n, None
        splits = lt_splits(n * N, H, N)

    def packed(rows, div=1.0, scale=1.0):
        x = torch.randn(rows, C, device=d, generator=g) * scale
        p = torch.zeros(H, rows, 64, dtype=torch.float16, device=d)
        ops.tc_pack_rows(x, p, 0, div)
        return p

    Qp = packed(n * N + 256, math.sqrt(D), 3.0)
    Kp, Vp = packed(n * kvs), packed(n * kvs)
    part = lambda rows: tuple(torch.full(s, float("nan"), device=d)
                              for s in ((splits, rows, C), (splits, H, rows), (splits, H, rows))) if splits > 1 else None
    O = torch.full((n * N, C), float("nan"), device=d)
    ops.lt_attention_tc_batched(Qp, N, Kp, Vp, kvs, n, N, Tk=0 if tk_dev is not None else N, Tk_dev=tk_dev, O=O,
                                splits=splits, exact=exact, part=part(n * N))
    torch.cuda.synchronize()
    worst = 0.0
    qcap = -(-N // 256) * 256
    for b in range(n):
        q = torch.zeros(H, qcap, 64, dtype=torch.float16, device=d)
        q[:, :N] = Qp[:, b * N:(b + 1) * N]
        k, v = Kp[:, b * kvs:(b + 1) * kvs].contiguous(), Vp[:, b * kvs:(b + 1) * kvs].contiguous()
        want = torch.full((N, C), float("nan"), device=d)
        ops.lt_attention_tc(q, k, v, N, N if tk_dev is None else 0, O=want,
                            Tk_dev=None if tk_dev is None else tk_dev[b:b + 1], splits=splits, exact=exact, part=part(N),
                            variant="tile")
        torch.cuda.synchronize()
        ob = O[b * N:(b + 1) * N]
        assert torch.equal(ob, want), b
        ref, tol = attn_restatement((unpack(q, N, "hi"), unpack(q, N, "lo")),
                                    (unpack(k, live[b], "hi"), unpack(k, live[b], "lo")), unpack(v, live[b]), H, exact,
                                    splits)
        r = ratio(ob, ref, tol)
        worst = max(worst, r)
        assert r < 1.0, (b, live[b], r)
    print(f"batched lt {form} {'exact' if exact else 'fast'}: n {n} N {N} live {live[0]}..{live[-1]} splits {splits}: "
          f"worst err / bound {worst:.3f}")
