"""GPU: mask in, labels out -- the ID embedding, logit post-processing, label-map and bank kernels of csrc/idbank.cu and
label_to_u8 (csrc/io_side.cu) -- against float64 or exact restatements, at the shapes, ids and label edges where they can go
wrong.  Kernels that only move or compare data are checked bit for bit; the others within these bounds:

  ID embedding, gather    |e - e64| <= 2^-23 (E_FIX + E_ACC sqrt(n + 1)) mag,  mag = conv(onehot, |W|) + |b|, n valid taps
  ID embedding, runs      the same over the 2 x runs table reads (mag = sum of |table rows read| + |b|), plus half an fp32
                          ulp of each table entry read: the prefix table is summed in float64 and stored in fp32
  + fused LayerNorm       |gamma| rstd (t + mean t + |y - mean| rstd^2 mean(|y - mean| (t + mean t)))
                          + LN_C 2^-23 ((|y - mean| rstd + 1) |gamma| + |beta|) + LN_C ulp(mean |y|) rstd |gamma|
  bilinear upsample       2^-23 (4 S + (2 h + 1) Dy + (2 w + 1) Dx)
  soft aggregation        (eps p / p_cl + 2^-23) / (1 - p_cl) + 2^-23 (1 + |logit|)

- E_ACC = 2, E_FIX = 2: the gather is a chain of n fp32 adds (roundings growing as sqrt(n)) and the bias add.
- LN_C = 11: the two-pass block LayerNorm of C = 256 rounds as the warp LayerNorm of tests/test_gpu_simt_envelope.py (9 + 2).
- Bilinear: S = sum of tap weight x |tap| (four products, three sums); the source coordinate is computed in fp32 and is off
  by at most 2 h ulps of 1 (resp. w), which moves the weights by as much, times the step Dy (Dx) between neighbouring
  low-res taps around the sample (the cells on either side included, as a rounding can cross a cell boundary).
- Aggregation: p = softmax probability before the clamp, p_cl after it.  fp32 p has relative error eps = 2^-23 (S_FIX +
  |v - m| / 2 + sum_j p_j |v_j - m| / 2): S_FIX = 10 covers expf, the 11-term sum and the division, the |v - m| terms the
  rounding of the shifted logits.  logit(p) = log(p / (1 - p)) has slope 1 / (p (1 - p)), so a relative error eps of p
  becomes eps / (1 - p): the bound grows as p -> 1, and the fp32 clamp constant 1 - 1e-5 (off by up to half an ulp of 1)
  adds 2^-23 / (1 - p_cl).  The background probability multiplies E softmax outputs: eps_bg = sum_e eps_e + E 2^-23.

tests/test_cpu_envelope_controls.py shows on the CPU that these bounds catch a run ending one tap early, a flipped
align_corners and a background taken from the last engine only, and that round-instead-of-floor changes a nearest resize."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
U = 2.0 ** -23
EPS = float(np.float32(1e-5))
E_FIX, E_ACC = 2.0, 2.0
LN_C = 11.0
S_FIX = 10.0
NID = 11
STRIDE = 16


def _ulp32(t):
    """float64 tensor -> the fp32 ulp of each |value| (as float64)."""
    return torch.from_numpy(np.spacing(t.abs().float().numpy()).astype(np.float64))


def _worst(out, ref, tol):
    assert torch.isfinite(out).all()
    err = (out.double() - ref).abs()
    return torch.where(err == 0, torch.zeros_like(err), err / tol).max().item()


# ================================================================== ID embedding
GEOMS = [(17, 8), (16, 0)]                    # (ksize, pad) at stride 16: align_corners True / False
SIZES = [(17, 17), (33, 49), (161, 241), (481, 849)]
PATTERNS = ["blocky", "per_pixel", "background", "one_object", "foreign_ids", "no_match"]
ID_CASES = [(g, s, p) for g in GEOMS for s in SIZES[:3] for p in PATTERNS] + \
           [(g, SIZES[3], p) for g in GEOMS for p in ("blocky", "per_pixel")]


def make_mask(pattern, Hm, Wm, seed=0):
    """float32 [Hm, Wm] label map.  per_pixel: every tap its own random id (up to 17 runs per window row); foreign_ids: ids
    11, 255 and -1 in a blocky map; no_match: 2.5 and NaN among per-pixel ids (they match no id)."""
    g = torch.Generator().manual_seed(seed + Hm * 7 + Wm)
    if pattern in ("blocky", "foreign_ids"):
        m = torch.randint(0, NID, (1, 1, (Hm + 11) // 12, (Wm + 8) // 9), generator=g).float()
        m = F.interpolate(m, size=(Hm, Wm), mode="nearest")[0, 0]
        if pattern == "foreign_ids":
            sel = torch.rand(Hm, Wm, generator=g)
            m[sel < 0.3] = 11.0
            m[(sel >= 0.3) & (sel < 0.4)] = 255.0
            m[(sel >= 0.4) & (sel < 0.5)] = -1.0
        return m.contiguous()
    if pattern in ("per_pixel", "no_match"):
        # random ids, each different from its left neighbour: 17 runs in every full window row
        steps = torch.randint(1, NID, (Hm, Wm), generator=g)
        m = ((torch.randint(0, NID, (Hm, 1), generator=g) + steps.cumsum(1)) % NID).float()
        if pattern == "no_match":
            sel = torch.rand(Hm, Wm, generator=g)
            m[sel < 0.3] = 2.5
            m[(sel >= 0.3) & (sel < 0.4)] = float("nan")
        return m
    m = torch.zeros(Hm, Wm)
    if pattern == "one_object":
        yy, xx = torch.meshgrid(torch.arange(Hm, dtype=torch.float64), torch.arange(Wm, dtype=torch.float64), indexing="ij")
        inside = ((yy - Hm * 0.45) / (Hm * 0.3)) ** 2 + ((xx - Wm * 0.55) / (Wm * 0.25)) ** 2 <= 1
        m[inside] = 1.0
    return m


def id_weights(C, k, seed=0):
    """The ID-bank weights as model.py initialises them (row norm k^-2, bit-reproducible Gaussian) at the calibrated x100
    scale of oracle/weights.py, and a bias like nn.Conv2d's: -> w [C, 11, k, k], b [C]."""
    import inspect

    from oracle import weights as OW
    scale = inspect.signature(OW.build_state_dict).parameters["id_scale"].default
    g = torch.Generator().manual_seed(seed + 100 * k + C)
    fan_in = NID * k * k
    w = torch.randn(C, NID, k, k, generator=g) * (float(k) ** -2 / math.sqrt(fan_in)) * scale
    b = (torch.rand(C, generator=g) * 2 - 1) / math.sqrt(fan_in)
    return w, b


def prefix_table(w):
    """Exclusive prefix sums along kx, summed in float64 and stored in fp32: [k, k + 1, 11, C]."""
    k = w.shape[2]
    t = w.double().permute(2, 3, 1, 0)
    pre = torch.zeros(k, k + 1, t.shape[2], t.shape[3], dtype=torch.float64)
    pre[:, 1:] = torch.cumsum(t, dim=1)
    return pre.float()


def _window_ids(mask, k, pad):
    """-> ids [P, k, k] int64 of each output pixel's window (-1: outside the frame or no id), and (ho, wo)."""
    Hm, Wm = mask.shape
    valid = (mask == mask.round()) & (mask >= 0) & (mask < NID)                 # NaN compares false
    ids = torch.where(valid, mask.nan_to_num(0.0), torch.full_like(mask, -1.0)).double()
    ho, wo = (Hm + 2 * pad - k) // STRIDE + 1, (Wm + 2 * pad - k) // STRIDE + 1
    padded = F.pad(ids.view(1, 1, Hm, Wm), (pad, pad, pad, pad), value=-1.0)
    win = F.unfold(padded, k, stride=STRIDE)                                    # [1, k*k, ho*wo]
    win = win.view(k, k, ho * wo).permute(2, 0, 1)
    return win.long(), (ho, wo)


def run_table_counts(mask, k, pad, end_shift=0, start_weight=1.0):
    """Count matrix S [P, k * (k + 1) * 11]: how often each prefix-table row (ky, j, id) is read for each output pixel (a
    run [a, b) of id reads rows (ky, a, id) and (ky, b, id)).  With start_weight = -1, S @ table is the runs form of the
    embedding (before the bias); end_shift moves every run end (the controls' slip)."""
    ids, (ho, wo) = _window_ids(mask, k, pad)
    P = ids.shape[0]
    minus2 = torch.full((P, k, 1), -2, dtype=torch.long)
    prev = torch.cat([minus2, ids[:, :, :-1]], dim=2)
    nxt = torch.cat([ids[:, :, 1:], minus2], dim=2)
    kx = torch.arange(k).view(1, 1, k).expand(P, k, k)
    ky = torch.arange(k).view(1, k, 1).expand(P, k, k)
    idc = ids.clamp(min=0)
    start = (ids != prev) & (ids >= 0)
    end = (ids != nxt) & (ids >= 0)
    S = torch.zeros(P, k * (k + 1) * NID, dtype=torch.float64)
    pix = torch.arange(P).view(P, 1, 1).expand(P, k, k)
    for sel, j, wgt in ((start, kx, start_weight), (end, kx + 1 + end_shift, 1.0)):
        col = ((ky * (k + 1) + j) * NID + idc)[sel]
        S.index_put_((pix[sel], col), torch.full((col.numel(),), wgt, dtype=torch.float64), accumulate=True)
    return S


def _ln64(y, ga, be):
    mean = y.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((y - mean) ** 2).mean(1, keepdim=True) + EPS)
    return (y - mean) * rstd * ga + be, mean, rstd


def ln_tolerance(y, t, ga, be):
    """Tolerance after the fused LayerNorm of float64 pre-values y [P, C] known to within t [P, C]."""
    ga, be = ga.double().view(1, -1), be.double().view(1, -1)
    _, mean, rstd = _ln64(y, ga, be)
    d = (y - mean).abs()
    tm = t + t.mean(1, keepdim=True)
    drel = rstd ** 2 * (d * tm).mean(1, keepdim=True)
    return (ga.abs() * rstd * (tm + d * drel) + LN_C * U * ((d * rstd + 1.0) * ga.abs() + be.abs())
            + LN_C * _ulp32(y.abs().mean(1, keepdim=True)) * rstd * ga.abs())


def id_reference(mask, w, b, pad, wp=None):
    """float64 dense conv of the one-hot mask -> (y [P, C], gather tolerance [P, C], runs tolerance [P, C] if wp)."""
    k, C = w.shape[2], w.shape[0]
    onehot = (mask.view(1, 1, *mask.shape) == torch.arange(NID, dtype=torch.float32).view(1, -1, 1, 1)).double()
    y = F.conv2d(onehot, w.double(), b.double(), STRIDE, pad)[0].permute(1, 2, 0).reshape(-1, C)
    mag = F.conv2d(onehot, w.double().abs(), b.double().abs(), STRIDE, pad)[0].permute(1, 2, 0).reshape(-1, C)
    n = F.conv2d(onehot.sum(1, keepdim=True), torch.ones(1, 1, k, k, dtype=torch.float64), None, STRIDE, pad).view(-1, 1)
    tol = U * (E_FIX + E_ACC * torch.sqrt(n + 1)) * mag
    if wp is None:
        return y, tol, None
    S = run_table_counts(mask, k, pad)
    wp64 = wp.double().reshape(-1, C)
    reads = S.sum(1, keepdim=True)
    tol_runs = S @ (0.5 * _ulp32(wp64)) + U * (E_FIX + E_ACC * torch.sqrt(reads + 1)) * (S @ wp64.abs() + b.double().abs())
    return y, tol, tol_runs


def _out_slice(P, C):
    """out [P, C] as a column slice of a wider NaN-filled buffer (the kernels take a row stride)."""
    buf = torch.full((P, C + 12), float("nan"), device=DEV)
    return buf, buf[:, 8:8 + C]


def _check_slice(buf, C):
    assert torch.isnan(buf[:, :8]).all() and torch.isnan(buf[:, 8 + C:]).all(), "wrote outside its columns"


def _run_id(kind, mask, table, b, C, k, pad, ln=None):
    from aot_benchmark_b200 import ops
    ho, wo = (mask.shape[0] + 2 * pad - k) // STRIDE + 1, (mask.shape[1] + 2 * pad - k) // STRIDE + 1
    buf, out = _out_slice(ho * wo, C)
    fn = ops.id_embed if kind == "gather" else ops.id_embed_runs
    fn(mask.to(DEV), table.to(DEV), b.to(DEV), out, C, NID, k, STRIDE, pad,
       ln_gamma=None if ln is None else ln[0].to(DEV), ln_beta=None if ln is None else ln[1].to(DEV))
    torch.cuda.synchronize()
    _check_slice(buf, C)
    return out.cpu()


def _pack(w):
    co, ci, kh, kw = w.shape
    return w.permute(2, 3, 1, 0).reshape(kh * kw * ci, co).contiguous()


def _check_id_embed(mask, w, b, k, pad, wp, what):
    C = w.shape[0]
    y, tol, tol_runs = id_reference(mask, w, b, pad, wp)
    g = torch.Generator().manual_seed(k)
    ga, be = torch.randn(C, generator=g), torch.randn(C, generator=g) * 0.5
    y_ln, _, _ = _ln64(y, ga.double(), be.double())
    worst = {}
    for kind, table, t in (("gather", _pack(w), tol), ("runs", wp, tol_runs)):
        worst[kind] = _worst(_run_id(kind, mask, table, b, C, k, pad), y, t)
        worst[kind + "+LN"] = _worst(_run_id(kind, mask, table, b, C, k, pad, ln=(ga, be)), y_ln,
                                     ln_tolerance(y, t, ga, be))
    print(what, {kk: round(v, 3) for kk, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("geom,size,pattern", ID_CASES,
                         ids=[f"k{g[0]}-{s[0]}x{s[1]}-{p}" for g, s, p in ID_CASES])
def test_id_embed_vs_float64(geom, size, pattern):
    """id_embed (gather) and id_embed_runs (prefix table), each with and without the fused LayerNorm (C = 256)."""
    k, pad = geom
    mask = make_mask(pattern, *size)
    w, b = id_weights(256, k)
    _check_id_embed(mask, w, b, k, pad, prefix_table(w), f"k{k} {size} {pattern}")


def test_id_embed_runs_worst_case_reaches_17_runs_per_row():
    """The per-pixel pattern fills every window row with 17 runs (578 table reads per pixel), the kernel's bound."""
    mask = make_mask("per_pixel", 161, 241)
    S = run_table_counts(mask, 17, 8)
    assert S.sum(1).max().item() == 2 * 17 * 17


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("pattern", ["blocky", "per_pixel", "foreign_ids"])
def test_id_embed_c128_vs_float64(geom, pattern):
    """The gather kernel at C = 128 (no fused LayerNorm: that needs C = 256)."""
    k, pad = geom
    mask = make_mask(pattern, 161, 241)
    w, b = id_weights(128, k)
    y, tol, _ = id_reference(mask, w, b, pad)
    r = _worst(_run_id("gather", mask, _pack(w), b, 128, k, pad), y, tol)
    print(f"C 128 k{k} {pattern}: worst err / tol {r:.3f}")
    assert r <= 1.0


@pytest.mark.parametrize("align", [True, False])
def test_id_embed_runs_with_the_plan_table(align):
    """The prefix table and packed weights exactly as plan.py builds them (Plan._idbank), not a test-side cumsum."""
    from aot_benchmark_b200 import plan

    class _IdBankOnly(plan.Plan):
        def __init__(self, sd, align_corners):
            self.sd, self.align_corners = sd, align_corners
            self._idbank()

    k = 17 if align else 16
    w, b = id_weights(256, k, seed=5)
    P = _IdBankOnly({"patch_wise_id_bank.weight": w, "patch_wise_id_bank.bias": b}, align)
    assert (P.id_k, P.id_pad) == (k, 8 if align else 0)
    mask = make_mask("per_pixel", 161, 241, seed=3)
    y, tol, tol_runs = id_reference(mask, w, b, P.id_pad, P.id_wp)
    r = _worst(_run_id("runs", mask, P.id_wp, P.id_b, 256, k, P.id_pad), y, tol_runs)
    r2 = _worst(_run_id("gather", mask, P.id_wt, P.id_b, 256, k, P.id_pad), y, tol)
    print(f"plan table k{k}: worst err / tol runs {r:.3f}, gather {r2:.3f}")
    assert r <= 1.0 and r2 <= 1.0


# ================================================================== logits: mask, upsample, argmax
# (h, w) low-res -> (Ho, Wo): x4 (the 480p decoder output), a non-integer ratio, identity, a downsample, a 1x1 output, 1xN
# and Nx1 inputs, one input pixel
LOGIT_SIZES = [((121, 213), (481, 849)), ((37, 53), (100, 150)), ((31, 17), (31, 17)), ((41, 61), (20, 30)),
               ((7, 9), (1, 1)), ((1, 9), (4, 33)), ((9, 1), (33, 4)), ((1, 1), (5, 7))]


def bilinear_taps(n_in, n_out, align):
    """PyTorch's source index rule, in float64: -> (i0, i1, l1) per output index."""
    dst = torch.arange(n_out, dtype=torch.float64)
    if align:
        src = dst * ((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0)
    else:
        src = ((dst + 0.5) * (n_in / n_out) - 0.5).clamp(min=0.0)
    i0 = src.floor().long().clamp(max=n_in - 1)
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    return i0, i1, (src - i0).clamp(0.0, 1.0)


def _step_max(lo, dim):
    """max |difference between neighbouring taps along dim (2: y, 3: x)| over the 3x3 cells around each low-res position."""
    n = lo.shape[dim]
    if n == 1:
        return torch.zeros_like(lo)
    d = (lo.narrow(dim, 1, n - 1) - lo.narrow(dim, 0, n - 1)).abs()
    d = F.pad(d, (0, 1) if dim == 3 else (0, 0, 0, 1))
    return F.max_pool2d(d, 3, 1, 1)


def bilinear_reference(lo, Ho, Wo, align):
    """float64 bilinear upsample of lo [1, NC, h, w] -> (value, tolerance) [1, NC, Ho, Wo]."""
    lo = lo.double()
    h, w = lo.shape[-2:]
    y0, y1, ly = bilinear_taps(h, Ho, align)
    x0, x1, lx = bilinear_taps(w, Wo, align)
    ly, lx = ly.view(-1, 1), lx.view(1, -1)
    hy, hx = 1 - ly, 1 - lx

    def at(t, yi, xi):
        return t[:, :, yi][:, :, :, xi]

    val = hy * (hx * at(lo, y0, x0) + lx * at(lo, y0, x1)) + ly * (hx * at(lo, y1, x0) + lx * at(lo, y1, x1))
    a = lo.abs()
    S = hy * (hx * at(a, y0, x0) + lx * at(a, y0, x1)) + ly * (hx * at(a, y1, x0) + lx * at(a, y1, x1))
    Dy, Dx = at(_step_max(lo, 2), y0, x0), at(_step_max(lo, 3), y0, x0)
    return val, U * (4 * S + (2 * h + 1) * Dy + (2 * w + 1) * Dx)


def logit_inputs(h, w, seed=0):
    g = torch.Generator().manual_seed(seed + 31 * h + w)
    return torch.randn(1, NID, h, w, generator=g) * 4


def masked_lowres(lg, obj):
    lo = lg.clone()
    lo[:, obj + 1:] = -1e10
    return lo


def _objs(h):
    return range(NID) if h < 100 else (0, 3, 10)


@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("sizes", LOGIT_SIZES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in LOGIT_SIZES])
def test_logits_postproc_vs_float64(sizes, align):
    """Low-res masking bit for bit for obj_num 0..10; the upsample within the bilinear bound; masked channels stay at
    -1e10 (to 4 ulps)."""
    from aot_benchmark_b200 import ops
    (h, w), (Ho, Wo) = sizes
    lg = logit_inputs(h, w)
    lg_nhwc = lg[0].permute(1, 2, 0).contiguous().to(DEV)
    lo = torch.empty(1, NID, h, w, device=DEV)
    out = torch.empty(1, NID, Ho, Wo, device=DEV)
    worst = 0.0
    for obj in _objs(h):
        ops.logits_postproc(lg_nhwc, lo, out, obj, align)
        torch.cuda.synchronize()
        want_lo = masked_lowres(lg, obj)
        assert torch.equal(lo.cpu(), want_lo), obj
        ref, tol = bilinear_reference(want_lo, Ho, Wo, align)
        o = out.cpu()
        worst = max(worst, _worst(o[:, :obj + 1], ref[:, :obj + 1], tol[:, :obj + 1]))
        assert (o[:, obj + 1:].double() <= -1e10 * (1 - 4 * U)).all()
        assert (o[:, obj + 1:].double() >= -1e10 * (1 + 4 * U)).all()
    print(f"{sizes} align {align}: worst err / tol {worst:.3f}")
    assert worst <= 1.0


def test_bilinear_reference_is_f_interpolate():
    """The float64 restatement used for the bounds equals F.interpolate in float64."""
    for (h, w), (Ho, Wo) in LOGIT_SIZES:
        lo = logit_inputs(h, w).double()
        for align in (True, False):
            val, _ = bilinear_reference(lo, Ho, Wo, align)
            want = F.interpolate(lo, size=(Ho, Wo), mode="bilinear", align_corners=align)
            assert (val - want).abs().max().item() <= 1e-12 * lo.abs().max().item()


def argmax_certain(ref, tol):
    """float64 argmax and where it is certain: the top value's lower bound exceeds every other channel's upper bound."""
    top = ref.argmax(1, keepdim=True)
    lower = ref.gather(1, top) - tol.gather(1, top)
    upper = (ref + tol).scatter(1, top, -math.inf)
    return top[:, 0], lower[:, 0] > upper.amax(1)


@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("sizes", LOGIT_SIZES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in LOGIT_SIZES])
def test_logits_argmax_vs_float64(sizes, align):
    """Where the float64 top-two gap exceeds the bilinear bound the label is the float64 argmax; no label exceeds obj_num."""
    from aot_benchmark_b200 import ops
    (h, w), (Ho, Wo) = sizes
    lg = logit_inputs(h, w, seed=1)
    label = torch.full((1, Ho, Wo), float("nan"), device=DEV)
    unsure = 0
    for obj in _objs(h):
        lo = masked_lowres(lg, obj)
        ops.logits_argmax(lo.to(DEV), label, align)
        torch.cuda.synchronize()
        lab = label.cpu()
        assert (lab == lab.round()).all() and lab.min().item() >= 0 and lab.max().item() <= obj
        ref, tol = bilinear_reference(lo, Ho, Wo, align)
        top, certain = argmax_certain(ref, tol)
        assert torch.equal(lab[certain], top[certain].float()), obj
        unsure += (~certain).sum().item()
    print(f"{sizes} align {align}: {unsure} pixels within the bound of a tie")


def test_logits_argmax_duplicate_channel_lower_index_wins():
    """Channels 3 and 5 hold the same, dominant values: every label is 3, as torch.argmax picks the first maximum."""
    from aot_benchmark_b200 import ops
    lo = logit_inputs(37, 53, seed=2)
    lo[:, 3] = lo[:, 1] + 50
    lo[:, 5] = lo[:, 3]
    for align in (True, False):
        label = torch.empty(1, 100, 150, device=DEV)
        ops.logits_argmax(lo.to(DEV), label, align)
        torch.cuda.synchronize()
        assert (label == 3).all()


# ================================================================== nearest resize
NEAREST_SIZES = [((480, 854), (1080, 1920)), ((1080, 1920), (480, 854)), ((37, 53), (74, 106)), ((31, 54), (31, 54)),
                 ((97, 131), (149, 211)), ((211, 149), (97, 131)), ((1, 1), (5, 7)), ((5, 7), (1, 1)), ((74, 106), (37, 53))]


@pytest.mark.parametrize("sizes", NEAREST_SIZES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in NEAREST_SIZES])
def test_nearest_resize_bitwise(sizes):
    """Every source pixel holds a distinct value, so any index slip shows."""
    from aot_benchmark_b200 import ops
    (H, W), (Ho, Wo) = sizes
    x = torch.arange(H * W, dtype=torch.float32).view(1, 1, H, W)
    out = torch.full((1, 1, Ho, Wo), float("nan"), device=DEV)
    ops.nearest_resize(x.to(DEV), out)
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), F.interpolate(x, size=(Ho, Wo), mode="nearest"))


# ================================================================== soft aggregation and label separation
MAX_OBJ = 10


def aggregation_inputs(E, H=37, W=53, seed=0):
    """E logit maps [1, 11, H, W]: random pixels, plus rows with saturated softmaxes (a channel 100 above the rest), equal
    logits, the background 100 above (all engines: bg -> 1, the upper clamp) or 100 below (the lower clamp), and from
    engine 1 on, masked -1e10 channels."""
    g = torch.Generator().manual_seed(seed + E)
    maps = []
    for e in range(E):
        t = torch.randn(1, 1 + MAX_OBJ, H, W, generator=g) * 4
        for r in range(5):
            t[:, (r + e) % (1 + MAX_OBJ), r] += 100.0
        t[:, :, 5:8] = t[:, :1, 5:8]
        t[:, 0, 8:11] += 100.0
        t[:, 0, 11:14] -= 100.0
        if e >= 1:
            t[:, 1 + (e * 3) % MAX_OBJ:] = -1e10
        maps.append(t)
    return maps


def _softmax_eps(v):
    """float64 softmax p of float32 logits v [1, NC, HW...] and the relative error bound eps of its fp32 evaluation."""
    v = v.double()
    m = v.amax(1, keepdim=True)
    p = torch.softmax(v, dim=1)
    dv = (v - m).abs()
    eps = U * (S_FIX + 0.5 * dv + 0.5 * (p * dv).nan_to_num(0.0).sum(1, keepdim=True))
    return p, eps


def _logit_tol(p, eps):
    pc = p.clamp(1e-5, 1 - 1e-5)
    out = torch.log(pc / (1 - pc))
    return out, (eps * p / pc + U) / (1 - pc) + U * (1 + out.abs())


def aggregation_reference(maps, bg_from=None):
    """float64 soft_logit_aggregation -> (out [1, 1 + E * 10, H, W], tol).  bg_from: engines whose background enters the
    product (default all; the controls' slip uses the last one only)."""
    E = len(maps)
    ps, eps = zip(*[_softmax_eps(t) for t in maps])
    idx = range(E) if bg_from is None else bg_from
    bg = torch.ones_like(ps[0][:, :1])
    for e in idx:
        bg = bg * ps[e][:, :1]
    eps_bg = sum(eps[e][:, :1] for e in idx) + len(idx) * U
    outs, tols = zip(*([_logit_tol(bg, eps_bg)] + [_logit_tol(ps[e][:, 1:], eps[e][:, 1:]) for e in range(E)]))
    return torch.cat(outs, 1), torch.cat(tols, 1)


@pytest.mark.parametrize("E", range(1, 9))
def test_soft_logit_aggregation_vs_float64(E):
    from aot_benchmark_b200 import ops
    maps = aggregation_inputs(E)
    H, W = maps[0].shape[-2:]
    out = torch.full((1, 1 + E * MAX_OBJ, H, W), float("nan"), device=DEV)
    ops.soft_logit_aggregation([t.to(DEV) for t in maps], out, MAX_OBJ)
    torch.cuda.synchronize()
    ref, tol = aggregation_reference(maps)
    r = _worst(out.cpu(), ref, tol)
    print(f"E {E}: worst err / tol {r:.3f}")
    assert r <= 1.0


def test_soft_logit_aggregation_refuses_unsupported():
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import AotbError
    maps = [t.to(DEV) for t in aggregation_inputs(8)]
    with pytest.raises(AotbError):
        ops.soft_logit_aggregation(maps + [maps[0]], torch.empty(1, 91, 37, 53, device=DEV), MAX_OBJ)
    five = [t[:, :6].contiguous() for t in maps[:2]]
    with pytest.raises(AotbError):
        ops.soft_logit_aggregation(five, torch.empty(1, 11, 37, 53, device=DEV), 5)


@pytest.mark.parametrize("E", range(1, 9))
def test_separate_labels_bitwise(E):
    """Ids at every engine boundary (10k, 10k + 1), beyond E * 10, negative, non-integer and NaN."""
    from aot_benchmark_b200 import ops
    special = [10.0 * k for k in range(E + 2)] + [10.0 * k + 1 for k in range(E + 2)] + \
              [0.5, 1.5, 9.5, 10.5, 10.999, -1.0, 255.0, float(E * MAX_OBJ + 1), float("nan")]
    g = torch.Generator().manual_seed(E)
    m = torch.cat([torch.tensor(special), torch.randint(0, E * MAX_OBJ + 5, (1000,), generator=g).float()])
    out = torch.full((E, m.numel()), float("nan"), device=DEV)
    ops.separate_labels(m.to(DEV), out, MAX_OBJ)
    torch.cuda.synchronize()
    for e in range(E):
        lo, hi = float(e * MAX_OBJ + 1), float((e + 1) * MAX_OBJ)
        fg = (m >= lo) & (m <= hi)
        want = torch.where(fg, m - lo + 1.0, torch.zeros_like(m))
        assert torch.equal(out[e].cpu(), want), e


# ================================================================== bank append and label_to_u8
@pytest.mark.parametrize("cols", [256, 1024])
@pytest.mark.parametrize("rows,offset,device_offset", [(37, 0, False), (37, 100, True), (1674, 1000, False),
                                                       (37, 2963, False), (37, 2963, True), (1674, 1326, True)])
def test_bank_append(rows, offset, device_offset, cols):
    """Host and device offsets, the last rows of the bank, a column-slice source, a row count that is not a multiple of
    the block; everything outside the target rows and columns untouched."""
    from aot_benchmark_b200 import ops
    cap = 3000
    g = torch.Generator().manual_seed(rows + offset + cols)
    src_full = torch.randn(rows, cols + 264, generator=g).to(DEV)
    src = src_full[:, 132:132 + cols]
    bank = torch.full((cap, cols + 8), float("nan"), device=DEV)
    if device_offset:
        ops.bank_append(src, bank, 7, offset_dev=torch.tensor([offset], dtype=torch.int32, device=DEV))
    else:
        ops.bank_append(src, bank, offset)
    torch.cuda.synchronize()
    assert torch.equal(bank[offset:offset + rows, :cols], src)
    rest = bank.clone()
    rest[offset:offset + rows, :cols] = float("nan")
    assert torch.isnan(rest).all()


def test_label_to_u8_bitwise():
    from aot_benchmark_b200 import ops
    lab = torch.arange(256, dtype=torch.float32).repeat(7)[torch.randperm(256 * 7, generator=torch.Generator().manual_seed(0))]
    out = torch.zeros(lab.numel(), dtype=torch.uint8, device=DEV)
    ops.label_to_u8(lab.to(DEV), out)
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), lab.to(torch.uint8))


# ================================================================== wrapper checks
def test_wrappers_refuse_strided_or_mismatched_operands():
    """Operands the kernels would read as dense although they are not, or whose shapes disagree, raise AotbError."""
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import AotbError
    d = DEV
    h, w = 9, 13
    lg = torch.randn(h, w, 16, device=d)
    lo = torch.empty(1, NID, h, w, device=d)
    out = torch.empty(1, NID, 20, 30, device=d)
    ops.logits_postproc(lg[..., :NID].contiguous(), lo, out, 3, True)             # the dense form runs
    bad_postproc = [
        (lg[..., :NID], lo, out),                                                    # channel slice of the logits
        (lg[..., :NID].contiguous(), torch.empty(1, 10, h, w, device=d), out),       # lowres NC
        (lg[..., :NID].contiguous(), torch.empty(1, NID, h + 1, w, device=d), out),  # lowres h
        (lg[..., :NID].contiguous(), torch.empty(1, NID, h, w + 1, device=d), out),  # lowres w
        (lg[..., :NID].contiguous(), lo, torch.empty(1, 10, 20, 30, device=d)),      # out NC
        (lg[..., :NID].contiguous(), lo, torch.empty(1, NID, 20, 32, device=d)[..., :30]),   # padded out rows
        (lg[..., :NID].contiguous(), torch.empty(1, NID, h, w + 3, device=d)[..., :w], out),  # padded lowres rows
    ]
    for a, b, c in bad_postproc:
        with pytest.raises(AotbError):
            ops.logits_postproc(a, b, c, 3, True)
    for a, b in ((torch.empty(1, NID, h, w + 4, device=d)[..., :w], torch.empty(1, 20, 30, device=d)),
                 (lo, torch.empty(1, 20, 32, device=d)[..., :30])):
        with pytest.raises(AotbError):
            ops.logits_argmax(a, b, True)
    for a, b in ((torch.empty(1, 1, 20, 32, device=d)[..., :30], torch.empty(1, 1, 10, 15, device=d)),
                 (torch.empty(1, 1, 20, 30, device=d), torch.empty(1, 1, 10, 16, device=d)[..., :15])):
        with pytest.raises(AotbError):
            ops.nearest_resize(a, b)

    wgt, b = id_weights(256, 17)
    wt, wp, bd = _pack(wgt).to(d), prefix_table(wgt).to(d), b.to(d)
    mask = torch.zeros(33, 53, device=d)
    ok = torch.empty(3 * 4, 256, device=d)                                            # ho x wo = 3 x 4 for a 33 x 49 mask
    ops.id_embed(mask[:, :49].contiguous(), wt, bd, ok, 256, NID, 17, STRIDE, 8)
    ops.id_embed_runs(mask[:, :49].contiguous(), wp, bd, ok, 256, NID, 17, STRIDE, 8)
    for fn, table in ((ops.id_embed, wt), (ops.id_embed_runs, wp)):
        for m, t, o in ((mask[:, :49], table, ok),                                    # mask a column slice
                        (mask[:, :49].contiguous(), table, torch.empty(12, 128, device=d)),   # out channel count
                        (mask[:, :49].contiguous(), table, torch.empty(13, 256, device=d)),   # out rows
                        (mask[:, :49].contiguous(), table[:-1], ok)):                 # table shape
            with pytest.raises(AotbError):
                fn(m, t, bd, o, 256, NID, 17, STRIDE, 8)
    with pytest.raises(AotbError):
        ops.id_embed_runs(mask[:, :49].contiguous(), wp.view(17, 18 * NID, 256), bd, ok, 256, NID, 17, STRIDE, 8)

    bank = torch.zeros(100, 256, device=d)
    src = torch.zeros(30, 256, device=d)
    ops.bank_append(src, bank, 70)                                                    # the last rows fit
    for s, off in ((src, 71), (src, -1), (torch.zeros(30, 260, device=d), 0), (torch.zeros(101, 256, device=d), 0)):
        with pytest.raises(AotbError):
            ops.bank_append(s, bank, off)
    with pytest.raises(AotbError):
        ops.bank_append(torch.zeros(30, 260, device=d), bank, 0, offset_dev=torch.zeros(1, dtype=torch.int32, device=d))
