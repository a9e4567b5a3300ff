"""CPU: negative controls for the bounds of tests/test_gpu_igemm_envelope.py, tests/test_gpu_mask_logit_envelope.py and
tests/test_gpu_window_envelope.py.

Each control restates, in float64, a plausible indexing slip of a kernel and shows that the slipped result lies outside the
GPU test's tolerance on that test's own cases, so the tolerance is tight enough to catch the slip.  Where a slip cannot
change a case's result (a nearest resize between equal sizes, one engine's background), the control says so and checks it.
No GPU is needed: the references and inputs are the GPU modules' own."""
import math

import pytest
import torch
import torch.nn.functional as F

import test_gpu_igemm_envelope as IG
import test_gpu_mask_logit_envelope as ML
import test_gpu_window_envelope as WE
from oracle import aot_oracle as O


def _exceeds(mut, ref, tol):
    return ((mut - ref).abs() / tol).max().item()


# ------------------------------------------------------------------ fp32 implicit-GEMM conv / linear
def _conv_problems():
    """(name, x, w, b, res, stride, pad, dil, act) for every conv and linear case of the GPU module."""
    for i, c in enumerate(IG.CONV_CASES):
        x, w, b, res = IG.case_inputs(c)
        yield IG.CONV_IDS[i], x, w, b, res, c["stride"], c["pad"], c["dil"], c["act"]
    for M, K, N, act, rmode in IG.LINEAR_CASES:
        x, w, b, res = IG.linear_inputs(M, K, N, rmode)
        yield (f"linear{M}x{K}-{N}", x.view(1, M, 1, K), w.view(N, K, 1, 1), b,
               None if res is None else res.view(1, M, 1, N), 1, 0, 1, act)


def _shift_one_pixel(x):
    """The window read one pixel to the right (one row down for a one-column input): out-of-frame taps read zero."""
    xs = torch.zeros_like(x)
    if x.shape[2] > 1:
        xs[:, :, :-1] = x[:, :, 1:]
    else:
        xs[:, :-1] = x[:, 1:]
    return xs


def _drop_last_chunk(w):
    """Weights with the rows of the last 16-deep K chunk (k = (ky, kx, ci)) zeroed: that chunk never accumulated."""
    co, ci, kh, kw = w.shape
    wk = IG.pack_w(w)
    K = wk.shape[0]
    wk[16 * ((K - 1) // 16):] = 0
    return wk.view(kh, kw, ci, co).permute(3, 2, 0, 1).contiguous()


def _res_next_pixel(res):
    B, Ho, Wo, C = res.shape
    return torch.roll(res.reshape(-1, C), -1, 0).view(B, Ho, Wo, C)


@pytest.mark.parametrize("slip", ["window_shift", "drop_last_k_chunk", "no_bias", "residual_next_pixel"])
def test_conv_tolerance_catches(slip):
    checked = 0
    for name, x, w, b, res, stride, pad, dil, act in _conv_problems():
        if (slip == "no_bias" and b is None) or (slip == "residual_next_pixel" and (res is None or res.numel() == res.shape[-1])):
            continue                                              # no bias / no residual / one pixel: nothing to slip
        ref, tol = IG.conv_reference(x, w, b, res, stride, pad, dil, act)
        args = dict(x=x, w=w, b=b, res=res)
        if slip == "window_shift":
            args["x"] = _shift_one_pixel(x)
        elif slip == "drop_last_k_chunk":
            args["w"] = _drop_last_chunk(w)
        elif slip == "no_bias":
            args["b"] = None
        else:
            args["res"] = _res_next_pixel(res)
        mut, _ = IG.conv_reference(args["x"], args["w"], args["b"], args["res"], stride, pad, dil, act)
        r = _exceeds(mut, ref, tol)
        assert r > 1.0, f"{slip} on {name}: worst err / tol only {r:.3f}"
        checked += 1
    assert checked >= 10


# ------------------------------------------------------------------ ID embedding: a run ending one tap early
def test_runs_model_is_the_dense_conv():
    """The run-table model behind the runs tolerance (and the slip below) reproduces the dense conv exactly in float64."""
    for (k, pad), size, pattern in ML.ID_CASES[::3]:
        mask = ML.make_mask(pattern, *size)
        w, b = ML.id_weights(256, k)
        y, _, _ = ML.id_reference(mask, w, b, pad)
        t = w.double().permute(2, 3, 1, 0)
        pre = torch.zeros(k, k + 1, ML.NID, 256, dtype=torch.float64)
        pre[:, 1:] = torch.cumsum(t, dim=1)
        S = ML.run_table_counts(mask, k, pad, start_weight=-1.0)
        assert (S @ pre.reshape(-1, 256) + b.double() - y).abs().max().item() <= 1e-12


@pytest.mark.parametrize("geom", ML.GEOMS)
def test_id_runs_tolerance_catches_a_run_ending_one_tap_early(geom):
    for g, size, pattern in ML.ID_CASES:
        if g != geom:
            continue
        k, pad = geom
        mask = ML.make_mask(pattern, *size)
        w, b = ML.id_weights(256, k)
        wp = ML.prefix_table(w)
        y, _, tol_runs = ML.id_reference(mask, w, b, pad, wp)
        S = ML.run_table_counts(mask, k, pad, end_shift=-1, start_weight=-1.0)
        mut = S @ wp.double().reshape(-1, 256) + b.double()
        r = _exceeds(mut, y, tol_runs)
        assert r > 1.0, f"{size} {pattern}: worst err / tol only {r:.3f}"


# ------------------------------------------------------------------ bilinear upsample: align_corners flipped
def _taps_move(h, w, Ho, Wo):
    return any(not all(torch.equal(a, b) for a, b in zip(ML.bilinear_taps(n, m, True), ML.bilinear_taps(n, m, False)))
               for n, m in ((h, Ho), (w, Wo)) if n > 1)


def test_upsample_tolerance_catches_flipped_align_corners():
    immune = []
    for (h, w), (Ho, Wo) in ML.LOGIT_SIZES:
        lo = ML.masked_lowres(ML.logit_inputs(h, w), 10)
        if not _taps_move(h, w, Ho, Wo):
            immune.append(((h, w), (Ho, Wo)))
            continue
        for align in (True, False):
            ref, tol = ML.bilinear_reference(lo, Ho, Wo, align)
            mut, _ = ML.bilinear_reference(lo, Ho, Wo, not align)
            r = _exceeds(mut, ref, tol)
            assert r > 1.0, f"{(h, w)} -> {(Ho, Wo)} align {align}: worst err / tol only {r:.3f}"
    # equal sizes, and a single input pixel, sample the same taps either way
    assert immune == [((31, 17), (31, 17)), ((1, 1), (5, 7))]


# ------------------------------------------------------------------ nearest resize: round instead of floor
def _nearest_round(x, Ho, Wo):
    H, W = x.shape[-2:]
    iy = torch.floor(torch.arange(Ho, dtype=torch.float32) * (H / Ho) + 0.5).long().clamp(max=H - 1)
    ix = torch.floor(torch.arange(Wo, dtype=torch.float32) * (W / Wo) + 0.5).long().clamp(max=W - 1)
    return x[..., iy, :][..., ix]


def test_nearest_bitwise_check_catches_round_instead_of_floor():
    immune = []
    for (H, W), (Ho, Wo) in ML.NEAREST_SIZES:
        x = torch.arange(H * W, dtype=torch.float32).view(1, 1, H, W)
        if torch.equal(_nearest_round(x, Ho, Wo), F.interpolate(x, size=(Ho, Wo), mode="nearest")):
            immune.append(((H, W), (Ho, Wo)))
    # identity and integer downsampling factors land on whole source indices; one source pixel has nothing to slip to
    assert immune == [((31, 54), (31, 54)), ((1, 1), (5, 7)), ((5, 7), (1, 1)), ((74, 106), (37, 53))]


# ------------------------------------------------------------------ soft aggregation: background of the last engine only
@pytest.mark.parametrize("E", range(2, 9))
def test_aggregation_tolerance_catches_last_engine_background(E):
    maps = ML.aggregation_inputs(E)
    ref, tol = ML.aggregation_reference(maps)
    mut, _ = ML.aggregation_reference(maps, bg_from=[E - 1])
    r = _exceeds(mut, ref, tol)
    assert r > 1.0, f"E {E}: worst err / tol only {r:.3f}"
    assert math.isfinite(r)


# ------------------------------------------------------------------ Swin window attention
def _bands(n, shift, off=0):
    """Region of each row (column) of the shifted padded map: [0, n-7) -> 0, [n-7, n-shift) -> 1, [n-shift, n) -> 2, with
    the second boundary moved by `off`."""
    r = torch.zeros(n, dtype=torch.long)
    r[n - WE.WS:n - shift + off] = 1
    r[n - shift + off:] = 2
    return r


def _mask(reg):
    """Region ids [Hp, Wp] of the shifted padded map -> the additive [nW, 49, 49] mask, -100 between regions."""
    Hp, Wp = reg.shape
    r = reg.view(Hp // WE.WS, WE.WS, Wp // WE.WS, WE.WS).permute(0, 2, 1, 3).reshape(-1, WE.T)
    return torch.where(r[:, :, None] != r[:, None, :], -100.0, 0.0).double()


def _padding_meets_real_tokens(H, W, shift, reg):
    """Whether some padded token shares a window and a shift region with a real token.  If none does, every padded key is
    masked for every real query (or there is no padding) and no padding slip can move a real row by more than e^-100."""
    Hp, Wp = reg.shape
    pad = torch.ones(Hp, Wp, dtype=torch.bool)
    pad[:H, :W] = False
    pad = torch.roll(pad, (-shift, -shift), (0, 1))
    win = (torch.arange(Hp) // WE.WS)[:, None] * (Wp // WE.WS) + (torch.arange(Wp) // WE.WS)[None, :]
    key = win * 9 + reg
    return bool(set(key[pad].tolist()) & set(key[~pad].tolist()))


def _window_slip(slip, case, qkv, qkv_bias, relb):
    """float64 window attention with one slip -> (output, whether the slip can change this case; None: it depends on
    the draw)."""
    H, W, heads, shift, dist = case
    C = heads * WE.D
    Hp, Wp = WE._padded(H), WE._padded(W)
    args = dict(qkv=qkv, qkv_bias=qkv_bias, relb=relb, H=H, W=W, heads=heads, shift=shift)
    reg = _bands(Hp, shift)[:, None] * 3 + _bands(Wp, shift)[None, :]
    if shift:
        assert torch.equal(_mask(reg), O.swin_shift_mask(Hp, Wp, WE.WS, shift, torch.float64))
    if slip == "region_from_unshifted_position":
        args["mask"] = _mask(torch.roll(reg, (-shift, -shift), (0, 1)))
        applies = shift > 0
    elif slip == "region_boundary_off_by_one":
        args["mask"] = _mask(_bands(Hp, shift, -1)[:, None] * 3 + _bands(Wp, shift, -1)[None, :]) if shift else None
        applies = shift > 0
    elif slip == "mask_minus_inf":
        args["mask"] = _mask(reg).masked_fill(_mask(reg) != 0, -math.inf) if shift else None
        applies = dist == "mask_sharp"
        if dist == "sharp" and shift:                         # a masked key may or may not outscore the row by chance
            applies = None
    elif slip == "padded_tokens_dropped":
        args["drop_pad"] = True
        applies = _padding_meets_real_tokens(H, W, shift, reg)
    elif slip == "padded_kv_zero":
        args["qkv_bias"] = torch.cat([qkv_bias[:C], torch.zeros(2 * C)])
        applies = _padding_meets_real_tokens(H, W, shift, reg)
    elif slip == "rel_bias_transposed":
        args["relb"] = relb.transpose(1, 2)
        applies = True
    elif slip == "shift_wrong_direction":
        args["roll"] = -1
        applies = shift > 0
    else:
        assert slip == "scale_after_bias"                       # (q.k + b) * scale = q * scale . k + b * scale
        args["relb"] = relb * WE.SCALE
        applies = True
    return WE.window_reference(**args)[0], applies


WINDOW_SLIPS = ["region_from_unshifted_position", "region_boundary_off_by_one", "mask_minus_inf", "padded_tokens_dropped",
                "padded_kv_zero", "rel_bias_transposed", "shift_wrong_direction", "scale_after_bias"]


@pytest.mark.parametrize("slip", WINDOW_SLIPS)
def test_window_tolerance_catches(slip):
    """Every case the slip can change is caught.  Where it cannot, the slipped result is the reference to within a weight of
    e^-100: a shift slip at shift 0; a padding slip on a map of whole windows, or where every padded token sits in a shift
    region of its own (14 x 20 at shift 6, 2 x 9 at shift 2); a -inf mask where every masked key scores about 100 below
    its row, which holds for the normal and large-bias draws.  The mask-sharp cases are built to expose the -inf mask; in
    the sharp draws a masked key outscores its row only by chance, so those are not asserted either way."""
    caught = 0
    for case, cid in zip(WE.CASES, WE.CASE_IDS):
        qkv, qkv_bias, relb = WE.case_inputs(*case)
        ref, tol = WE.window_reference(qkv, qkv_bias, relb, *case[:4])
        mut, applies = _window_slip(slip, case, qkv, qkv_bias, relb)
        r = _exceeds(mut, ref, tol)
        if applies:
            assert r > 1.0, f"{slip} on {cid}: worst err / tol only {r:.3f}"
            caught += 1
        elif applies is not None:
            assert r < 1e-20, f"{slip} on {cid}: the slip should not apply, yet err / tol is {r:.3e}"
    assert caught >= 10


@pytest.mark.parametrize("H,W,heads,shift", [(7, 7, 2, 0), (7, 7, 2, 3), (9, 13, 1, 3), (12, 5, 2, 0), (12, 5, 2, 3),
                                             (3, 16, 1, 3)])
def test_window_reference_is_the_oracle_swin_block(H, W, heads, shift):
    """A Swin block built around the float64 window reference -- LayerNorm, the qkv Linear, the window reference, proj and
    the residual, then the MLP -- is oracle.aot_oracle.swin_block, which the goldens pin to the reference's
    SwinTransformer."""
    g = torch.Generator().manual_seed(H * 100 + W + shift)
    C = heads * WE.D

    def rnd(*shape, s=1.0):
        return torch.randn(*shape, generator=g, dtype=torch.float64) * s

    sd = {"norm1.weight": 1 + rnd(C, s=0.1), "norm1.bias": rnd(C, s=0.1),
          "attn.qkv.weight": rnd(3 * C, C, s=C ** -0.5), "attn.qkv.bias": rnd(3 * C),
          "attn.relative_position_bias_table": rnd((2 * WE.WS - 1) ** 2, heads),
          "attn.proj.weight": rnd(C, C, s=C ** -0.5), "attn.proj.bias": rnd(C, s=0.1),
          "norm2.weight": 1 + rnd(C, s=0.1), "norm2.bias": rnd(C, s=0.1),
          "mlp.fc1.weight": rnd(4 * C, C, s=C ** -0.5), "mlp.fc1.bias": rnd(4 * C, s=0.1),
          "mlp.fc2.weight": rnd(C, 4 * C, s=(4 * C) ** -0.5), "mlp.fc2.bias": rnd(C, s=0.1)}
    x = rnd(H * W, C)
    want = O.swin_block(sd, "", x, H, W, heads, WE.WS, shift)
    qkv = O._lin(O._ln(x, sd, "norm1"), sd, "attn.qkv")
    relb = WE.relative_bias(sd["attn.relative_position_bias_table"])
    o, _ = WE.window_reference(qkv, sd["attn.qkv.bias"], relb, H, W, heads, shift)
    y = x + O._lin(o, sd, "attn.proj")
    got = y + O._lin(F.gelu(O._lin(O._ln(y, sd, "norm2"), sd, "mlp.fc1")), sd, "mlp.fc2")
    assert ((got - want).abs().max() / want.abs().max()).item() <= 1e-12
