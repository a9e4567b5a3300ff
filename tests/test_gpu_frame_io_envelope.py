"""The frame preprocessing kernel (preprocess_bgr_u8_kernel, csrc/io_side.cu) against oracle.io_side, bit for bit.

The kernel evaluates cv2's INTER_CUBIC resampling in the order oracle.io_side.resize_cubic does: per output pixel, four
fp32 products summed left to right along x, then four along y, with no contraction.  It then evaluates numpy's
normalisation statements as oracle.io_side.to_tensor does: v / 255 in fp32, then - mean and / std in fp64, each rounded to
fp32.  Both round the same operations in the same order, so the kernel must equal the oracle in every bit, at any size,
including outputs larger than the kernel's grid of 132 * 16 blocks of 256 threads (540,672 pixels).

Bitwise agreement could hide a mistake both make, so a CPU test compares the oracle with a float64 evaluation of the same
operation (Keys cubic taps with A = -0.75 in float64, each weight from its own polynomial) within a few ulps.  The tap
tables the engine uploads (io_side._cubic_taps) are checked on the CPU to be the oracle's, bit for bit.
"""
import functools
import os

import numpy as np
import pytest
import torch

from oracle import io_side as IO

DEV = torch.device("cuda:0")
U = 2.0 ** -23
GRID_THREADS = 132 * 16 * 256
GUARD = 0x7FBADBAD
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "io_side.pt")
# absolute error of an fp32 tap weight against the float64 Keys weight, in units of 2^-23: the rounding of the fractional
# position x to fp32 moves a weight by up to |dw/dx| * 2^-24 (|dw/dx| < 2), and the fp32 polynomials round intermediates
# of magnitude up to 6 three times each; the fourth weight, 1 - the other three, collects all of it.  The worst over the
# axis pairs of this module is 9.3.
C_W = 12.0

# (source h x w, output Ho x Wo); equal sizes take the kernel's no-resize path
FIXTURE_SIZES = [(113, 161), (145, 193), (64, 96), (65, 81)]        # tests/golden/io_side.pt's three configurations
RESIZE_CASES = ([((115, 155), s) for s in FIXTURE_SIZES]
                + [((480, 854), (577, 1041)), ((1080, 1920), (577, 1041)), ((1080, 1920), (753, 1345))]   # > the grid
                + [((1, 155), (17, 33)), ((97, 1), (3, 5)),             # one-row and one-column sources
                   ((115, 155), (1, 1)), ((1, 1), (5, 7)),              # one-pixel output and source
                   ((115, 155), (115, 97)), ((64, 31), (129, 31)),      # an identity axis
                   ((1000, 3), (3, 1000)), ((3, 1000), (1000, 3))])     # 1000 -> 3 and 3 -> 1000
SAME_CASES = [((115, 155), (115, 155)), ((1, 1), (1, 1)), ((1, 7), (1, 7)), ((577, 1041), (577, 1041))]
CASES = RESIZE_CASES + SAME_CASES
CASE_IDS = [f"{h}x{w}-{Ho}x{Wo}" for (h, w), (Ho, Wo) in CASES]
KINDS = ("source", "zeros", "full", "checker")
assert any(Ho * Wo > GRID_THREADS for _, (Ho, Wo) in RESIZE_CASES) and any(Ho * Wo > GRID_THREADS for _, (Ho, Wo) in SAME_CASES)


@functools.lru_cache(maxsize=None)
def _fixture_image():
    return torch.load(FIXTURE)["img"].numpy()


def make_image(kind, h, w):
    """uint8 [h, w, 3]: the fixture frame (at its size) or a seeded random one, all 0, all 255, or a 0 / 255
    checkerboard whose phase differs per channel."""
    if kind == "source":
        if (h, w) == (115, 155):
            return _fixture_image()
        return np.random.default_rng(h * 10007 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "zeros":
        return np.zeros((h, w, 3), np.uint8)
    if kind == "full":
        return np.full((h, w, 3), 255, np.uint8)
    assert kind == "checker"
    y, x, c = np.meshgrid(np.arange(h), np.arange(w), np.arange(3), indexing="ij")
    return (((y + x + c) % 2) * 255).astype(np.uint8)


@functools.lru_cache(maxsize=8)
def _resized(kind, h, w, Ho, Wo):
    img = np.array(make_image(kind, h, w), dtype=np.float32)          # eval_datasets.py: the float copy of the frame
    return img if (Ho, Wo) == (h, w) else IO.resize_cubic(img, Ho, Wo)


def oracle_frame(kind, h, w, Ho, Wo, flip):
    img = _resized(kind, h, w, Ho, Wo)
    return IO.to_tensor(img[:, ::-1].copy() if flip else img)


def _taps(h, w, Ho, Wo):
    """The device tap tables FramePreprocessor uploads: (ix, cx, iy, cy)."""
    from aot_benchmark_b200 import io_side
    iy, cy = io_side._cubic_taps(h, Ho)
    ix, cx = io_side._cubic_taps(w, Wo)
    return [torch.from_numpy(a).to(DEV) for a in (ix, cx, iy, cy)]


def run_kernel(img, Ho, Wo, flip):
    """ops.preprocess_bgr_u8 into the head of a guarded buffer, with the tap tables io_side uploads; checks that nothing
    past the [1, 3, Ho, Wo] output was written and returns it on the host."""
    from aot_benchmark_b200 import ops
    h, w = img.shape[:2]
    n = 3 * Ho * Wo
    buf = torch.full((n + 64,), GUARD, dtype=torch.int32, device=DEV).view(torch.float32)
    out = buf[:n].view(1, 3, Ho, Wo)
    taps = None if (Ho, Wo) == (h, w) else tuple(_taps(h, w, Ho, Wo))
    ops.preprocess_bgr_u8(torch.from_numpy(np.ascontiguousarray(img)).to(DEV), out, taps, flip)
    torch.cuda.synchronize()
    assert (buf[n:].view(torch.int32) == GUARD).all(), "written past the output"
    return out[0].cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_preprocess_bitwise(case, kind, flip):
    (h, w), (Ho, Wo) = case
    got = run_kernel(make_image(kind, h, w), Ho, Wo, flip)
    want = oracle_frame(kind, h, w, Ho, Wo, flip)
    assert got.shape == want.shape
    diff = (got.view(torch.int32) != want.view(torch.int32))
    assert not diff.any(), (f"{diff.sum().item()} of {diff.numel()} values differ, max |d| "
                            f"{(got - want).abs().max().item():.3e}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", [((115, 155), (145, 193)), ((1000, 3), (3, 1000))], ids=["up", "1000to3"])
def test_checkerboard_overshoot_is_not_clamped(case):
    """The reference resizes a float copy of the frame, so cubic overshoot at 0 / 255 edges is kept: values below 0 and
    above 255 before the normalisation."""
    (h, w), (Ho, Wo) = case
    got = run_kernel(make_image("checker", h, w), Ho, Wo, False).double()
    for c in range(3):
        v = (got[c] * IO.STD[c] + IO.MEAN[c]) * 255.0
        assert v.min().item() < -1.0 and v.max().item() > 256.0, (c, v.min().item(), v.max().item())


@pytest.mark.gpu
def test_frame_preprocessor_outputs_are_the_kernel_at_the_large_sizes():
    """FramePreprocessor, as the evaluator runs it on a 1080p frame at scales 1.0 and 1.3 with flip, gives the bits of the
    direct kernel calls above."""
    from aot_benchmark_b200.io_side import FramePreprocessor
    img = make_image("source", 1080, 1920)
    outs = FramePreprocessor(None, 1040, True, [1.0, 1.3])(img)
    assert [tuple(o.shape) for o in outs] == [(1, 3, 577, 1041)] * 2 + [(1, 3, 753, 1345)] * 2
    for o, (size, flip) in zip(outs, [((577, 1041), False), ((577, 1041), True), ((753, 1345), False),
                                       ((753, 1345), True)]):
        assert torch.equal(o[0].cpu().view(torch.int32), oracle_frame("source", 1080, 1920, *size, flip).view(torch.int32))


# --------------------------------------------------------------------------------------------------------- rejections
@pytest.mark.gpu
@pytest.mark.parametrize("bad", ["out_one_channel", "out_three_dims", "ix_transposed", "cx_transposed", "iy_transposed",
                                 "cy_transposed"])
def test_preprocess_rejects(bad):
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import AotbError
    h, w, Ho, Wo = 9, 11, 6, 7
    img = torch.zeros(h, w, 3, dtype=torch.uint8, device=DEV)
    taps = _taps(h, w, Ho, Wo)
    ops.preprocess_bgr_u8(img, torch.empty(1, 3, Ho, Wo, device=DEV), tuple(taps))    # the well-formed call
    out = torch.empty(1, 3, Ho, Wo, device=DEV)
    if bad == "out_one_channel":
        out = torch.empty(1, 1, Ho, Wo, device=DEV)
    elif bad == "out_three_dims":
        out = torch.empty(3, Ho, Wo, device=DEV)
    else:
        i = ["ix", "cx", "iy", "cy"].index(bad[:2])
        taps[i] = taps[i].t().contiguous().t()                   # same shape, column-major
        assert not taps[i].is_contiguous()
    with pytest.raises(AotbError):
        ops.preprocess_bgr_u8(img, out, tuple(taps))


# ---------------------------------------------------------------------------------------------------------- CPU checks
def keys_taps64(src, dst):
    """float64 cv2 INTER_CUBIC taps: sample position (d + 0.5) * src / dst - 0.5, Keys kernel with A = -0.75, each of the
    four weights from its own polynomial."""
    d = np.arange(dst)
    f = (d + 0.5) * (src / dst) - 0.5
    s = np.floor(f)
    x = f - s
    A = -0.75

    def near(t):
        return ((A + 2) * t - (A + 3)) * t * t + 1

    def far(t):
        return ((A * t - 5 * A) * t + 8 * A) * t - 4 * A

    idx = np.clip(s.astype(np.int64)[:, None] + np.arange(-1, 3)[None, :], 0, src - 1)
    return idx, np.stack([far(x + 1), near(x), near(1 - x), far(2 - x)], -1)


AXES = sorted({(h, Ho) for (h, _), (Ho, _) in RESIZE_CASES} | {(w, Wo) for (_, w), (_, Wo) in RESIZE_CASES})


def test_tap_tables_are_the_oracle_taps():
    """The engine's tables equal the oracle's bit for bit; the weights are the float64 Keys weights within C_W ulps; an
    identity axis has the weights (0, 1, 0, 0) exactly."""
    from aot_benchmark_b200 import io_side
    worst = 0.0
    for src, dst in AXES:
        i1, w1 = io_side._cubic_taps(src, dst)
        i2, w2 = IO.cubic_taps(src, dst)
        assert i1.dtype == i2.dtype == np.int32 and w1.dtype == w2.dtype == np.float32
        assert np.array_equal(i1, i2) and np.array_equal(w1.view(np.int32), w2.view(np.int32)), (src, dst)
        i64, w64 = keys_taps64(src, dst)
        assert np.array_equal(i1, i64), (src, dst)
        worst = max(worst, np.abs(w1 - w64).max() / U)
        if src == dst:
            assert np.array_equal(w1, np.tile(np.float32([0, 1, 0, 0]), (dst, 1)))
            assert np.array_equal(i1[:, 1], np.arange(dst))
    assert worst <= C_W, worst


def test_sizes_are_the_frame_preprocessor_sizes():
    """The fixture sizes are the three configurations of tests/golden/io_side.pt, and the large sizes are what
    FramePreprocessor picks for a 480p and a 1080p frame."""
    from aot_benchmark_b200.io_side import FramePreprocessor
    fx = torch.load(FIXTURE)
    sizes = set()
    for c in fx["cases"].values():
        kw = c["kw"]
        fp = FramePreprocessor(kw["max_short_edge"], kw["max_long_edge"], kw["flip"], kw["multi_scale"],
                               kw["align_corners"])
        for s, r in zip(kw["multi_scale"], c["ref"][::2 if kw["flip"] else 1]):
            size = fp.target_size(115, 155, s)
            assert size == tuple(r.shape[1:])
            sizes.add(size)
    assert sizes == set(FIXTURE_SIZES)
    assert FramePreprocessor(None, 800).target_size(480, 854, 1.3) == (577, 1041)
    assert FramePreprocessor(None, 1040).target_size(1080, 1920, 1.0) == (577, 1041)
    assert FramePreprocessor(None, 1040).target_size(1080, 1920, 1.3) == (753, 1345)


def reference64(img, Ho, Wo):
    """float64 resize + normalisation of uint8 img -> (out [3, Ho, Wo], tolerance of the fp32 evaluation)."""
    h, w = img.shape[:2]
    iy, wy = keys_taps64(h, Ho)
    ix, wx = keys_taps64(w, Wo)
    I = img.astype(np.float64)
    rows = I[:, ix, :]                                                  # [h, Wo, 4, 3]
    hs = np.einsum("xk,hxkc->hxc", wx, rows)                            # horizontal pass
    dh = U * (C_W * rows.sum(2) + 2 * np.einsum("xk,hxkc->hxc", np.abs(wx), rows))
    v = np.einsum("yr,yrxc->yxc", wy, hs[iy])
    dv = np.einsum("yr,yrxc->yxc", np.abs(wy), dh[iy]) + U * np.einsum("yr,yrxc->yxc", C_W + 2 * np.abs(wy),
                                                                       np.abs(hs[iy]))
    mean, std = np.array(IO.MEAN), np.array(IO.STD)
    a = v / 255.0
    out = (a - mean) / std
    tol = (dv / 255.0 + U * (np.abs(a) + np.abs(a - mean))) / std + U * np.abs(out)
    return out.transpose(2, 0, 1), tol.transpose(2, 0, 1)


@pytest.mark.parametrize("kind", ["source", "checker"])
@pytest.mark.parametrize("case", RESIZE_CASES, ids=CASE_IDS[:len(RESIZE_CASES)])
def test_oracle_resize_is_the_float64_operation(case, kind):
    """oracle.io_side.resize_cubic + to_tensor, which the kernel must equal bit for bit, is the float64 cubic resize and
    normalisation within the bound of its fp32 roundings: C_W ulps per weight, and one ulp per product and sum."""
    (h, w), (Ho, Wo) = case
    ref, tol = reference64(make_image(kind, h, w), Ho, Wo)
    got = oracle_frame(kind, h, w, Ho, Wo, False).numpy().astype(np.float64)
    ratio = (np.abs(got - ref) / tol).max()
    assert ratio <= 1.0, f"worst err / tol {ratio:.3f}"
