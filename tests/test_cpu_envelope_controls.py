"""CPU: negative controls for the bounds of tests/test_gpu_igemm_envelope.py and tests/test_gpu_mask_logit_envelope.py.

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
