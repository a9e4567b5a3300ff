"""GPU: the Swin-B window attention and patch merging kernels (csrc/window_attn.cu) at the edges of their envelope.

Window attention is compared with a float64 restatement of the reference's own steps (SwinTransformerBlock.forward and
WindowAttention.forward): pad, roll by -shift, partition, q * scale @ k^T + relative bias + mask (-100), softmax, @ v,
reverse, roll back, crop.  It is fed the float32 qkv and qkv bias the kernel reads, with no GEMM in front.  Padding comes
after norm1 and before the qkv Linear, so a padded token has q = k = v = the qkv bias.  The tolerance is derived per
element from the case's own inputs:

  |o - o64| <= 2^-23 (A_FIX + A_ACC sqrt(49)) sum_j p_j |v_j|  +  sum_j p_j (e_j + E) |v_j|,     E = sum_k p_k e_k
  e_j = 2^-23 (A_SCORE sqrt(32) scale sum_c |q_c k_jc| + |s_j| + |s_j - m|)

with p the float64 softmax, s_j the score with bias and mask, and m the row maximum.  A score error ds_j moves p_j by
p_j (ds_j - sum_k p_k ds_k), and e_j bounds ds_j: the FMA dot product and the rounding of q * scale (A_SCORE), the
additions of the bias and the mask (|s_j|), and the subtraction of the row maximum before expf (|s_j - m|).  So the
rounding of the -100 mask costs in proportion to the weight of the masked key only.  The constants are those of
tests/test_gpu_simt_envelope.py: expf, the sequential row sum, 1 / sum and the FMA value sum have the same structure here.

Patch merging only moves data and is compared bit for bit through integer views, so -0.0, infinities and NaN payloads
are checked too.
"""
import math

import pytest
import torch

from oracle import aot_oracle as O
from test_gpu_simt_envelope import A_ACC, A_FIX, A_SCORE

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
U = 2.0 ** -23
WS, D = 7, 32
T = WS * WS
SCALE = D ** -0.5
GUARD = 0x7FBADBAD          # a signalling-NaN bit pattern for guard cells: any write to one changes it
DISTS = ("normal", "sharp", "bias", "mask_sharp")


def _padded(n):
    return -(-n // WS) * WS


# ------------------------------------------------------------------------------------------------ float64 reference
def window_reference(qkv, qkv_bias, relb, H, W, heads, shift, mask=None, roll=1, drop_pad=False):
    """float64 window attention of float32 qkv [H*W, 3C] (the un-padded tokens), qkv_bias [3C] and relb [heads, 49, 49]
    -> (out [H*W, C], tol [H*W, C]).  The keyword arguments exist for the negative controls: `mask` replaces the
    shifted-window mask [nW, 49, 49], roll = -1 shifts the wrong way, drop_pad removes padded keys from the softmax."""
    C = heads * D
    Hp, Wp = _padded(H), _padded(W)
    nwy, nwx = Hp // WS, Wp // WS
    y = qkv_bias.double().expand(Hp, Wp, 3 * C).clone()
    y[:H, :W] = qkv.double().view(H, W, 3 * C)
    pad = torch.ones(Hp, Wp, 1, dtype=torch.bool)
    pad[:H, :W] = False
    if shift:
        y = torch.roll(y, (-roll * shift, -roll * shift), (0, 1))
        pad = torch.roll(pad, (-roll * shift, -roll * shift), (0, 1))

    def partition(t):
        return t.view(nwy, WS, nwx, WS, -1).permute(0, 2, 1, 3, 4).reshape(nwy * nwx, T, -1)

    win = partition(y).view(-1, T, 3, heads, D).permute(2, 0, 3, 1, 4)            # [3, nW, heads, 49, 32]
    q, k, v = win[0] * SCALE, win[1], win[2]
    if mask is None:
        mask = (O.swin_shift_mask(Hp, Wp, WS, shift, torch.float64) if shift
                else torch.zeros(nwy * nwx, T, T, dtype=torch.float64))
    s = q @ k.transpose(-2, -1) + relb.double().unsqueeze(0) + mask.unsqueeze(1)   # [nW, heads, 49, 49]
    if drop_pad:
        s = s.masked_fill(partition(pad)[:, None, None, :, 0], -math.inf)
    p = torch.softmax(s, -1)
    out = p @ v
    m = s.amax(-1, keepdim=True)
    e = U * (A_SCORE * math.sqrt(D) * (q.abs() @ k.abs().transpose(-2, -1)) + s.abs() + (s - m).abs())
    E = (p * e).sum(-1, keepdim=True)
    tol = U * (A_FIX + A_ACC * math.sqrt(T)) * (p @ v.abs()) + (p * (e + E)) @ v.abs()

    def reverse(t):
        t = t.transpose(1, 2).reshape(nwy, nwx, WS, WS, C).permute(0, 2, 1, 3, 4).reshape(Hp, Wp, C)
        if shift:
            t = torch.roll(t, (roll * shift, roll * shift), (0, 1))
        return t[:H, :W].reshape(H * W, C)

    return reverse(out), reverse(tol)


# ------------------------------------------------------------------------------------------------------------- inputs
def relative_bias(table):
    """[(2ws-1)^2, heads] table -> the dense [heads, 49, 49] bias the engine gathers once per block (plan.py)."""
    heads = table.shape[1]
    return table[O.swin_rel_index(WS).reshape(-1)].view(T, T, heads).permute(2, 0, 1).contiguous()


def case_inputs(H, W, heads, shift, dist):
    """float32 (qkv [H*W, 3C], qkv_bias [3C], relb [heads, 49, 49]) of one case.

    normal      unit-normal qkv, qkv bias of scale 0.5, unit-normal bias table
    sharp       q scaled by 30: near one-hot rows, where a wrong bias or mask term moves the output the most
    bias        qkv bias of scale 4 and a bias table of scale 3: padded tokens score high for many real queries
    mask_sharp  the key at the shifted position (Hp-1, Wp-1), which is the real token (shift-1, shift-1), is parallel to
                the q of every real query of that window outside its region, with scale q.k = 99: after the -100 it scores
                within a few units of the row maximum, so the output depends on the mask being -100 and not -inf.  The
                window holds real queries outside that region when Hp - H or Wp - W is less than 7 - shift.
    """
    g = torch.Generator().manual_seed(H * 7919 + W * 131 + heads * 17 + shift * 5 + DISTS.index(dist))
    C = heads * D
    qkv = torch.randn(H * W, 3 * C, generator=g)
    qkv_bias = torch.randn(3 * C, generator=g) * 0.5
    table = torch.randn((2 * WS - 1) ** 2, heads, generator=g)
    if dist == "sharp":
        qkv[:, :C] *= 30.0
    elif dist == "bias":
        qkv_bias *= 8.0
        table *= 3.0
    elif dist == "mask_sharp":
        assert 0 < shift <= min(H, W)
        qkv *= 0.3
        Hp, Wp = _padded(H), _padded(W)
        u = torch.randn(D, generator=g)
        u /= u.norm()
        ys = (torch.arange(H) - shift) % Hp                       # shifted position of every real row / column
        xs = (torch.arange(W) - shift) % Wp
        in_win = (ys >= Hp - WS)[:, None] & (xs >= Wp - WS)[None, :]
        region8 = (ys >= Hp - shift)[:, None] & (xs >= Wp - shift)[None, :]
        queries = (in_win & ~region8).reshape(-1)
        key = (shift - 1) * W + (shift - 1)
        assert region8.reshape(-1)[key] and queries.any()
        for h in range(heads):
            qkv[key, C + h * D:C + (h + 1) * D] = 30.0 * u
            qkv[queries, h * D:(h + 1) * D] = (99.0 / (30.0 * SCALE)) * u
    else:
        assert dist == "normal", dist
    return qkv, qkv_bias, relative_bias(table)


# (H, W, heads): every map of the engine's Swin-B stages, maps smaller than the window and the shift, and maps that give
# H mod 7 and W mod 7 every value 0..6 between them; heads 1 and 32 are the ends of what the ABI accepts (C = 32 heads)
GEOMS = [(148, 260, 4), (74, 130, 8), (37, 65, 16),                 # BASELINE config 4 at 592 x 1040
         (36, 52, 4), (18, 26, 8), (9, 13, 16),                     # the small Swin golden
         (1, 1, 4), (1, 13, 8), (5, 3, 4), (2, 9, 16),              # smaller than the window or the shift
         (14, 21, 4), (10, 20, 8), (20, 14, 1), (13, 6, 32), (37, 65, 8)]
assert {h % WS for h, _, _ in GEOMS} == set(range(WS)) and {w % WS for _, w, _ in GEOMS} == set(range(WS))

CASES = ([(H, W, h, s, "normal") for H, W, h in GEOMS for s in (0, 3)]
         + [(H, W, h, s, "sharp") for H, W, h in [(37, 65, 16), (9, 13, 16), (5, 3, 4), (2, 9, 16), (14, 21, 4),
                                                   (1, 13, 8)] for s in (0, 3)]
         + [(H, W, h, s, "bias") for H, W, h in [(74, 130, 8), (18, 26, 8), (1, 1, 4), (10, 20, 8), (13, 6, 32)]
            for s in (0, 3)]
         + [(H, W, h, 3, "mask_sharp") for H, W, h in [(14, 21, 4), (9, 13, 16), (5, 3, 4), (18, 26, 8)]]
         # every shift the ABI accepts, at two geometries
         + [(14, 20, 8, s, "mask_sharp") for s in range(1, WS)]
         + [(2, 9, 16, s, "sharp") for s in (1, 2, 4, 5, 6)])
CASE_IDS = [f"{H}x{W}-h{h}-s{s}-{dist}" for H, W, h, s, dist in CASES]


# ------------------------------------------------------------------------------------------------------------- runs
def _guarded(rows, cols):
    return torch.full((rows, cols), GUARD, dtype=torch.int32, device=DEV).view(torch.float32)


def run_window(qkv, qkv_bias, relb, H, W, heads, shift):
    """Window attention with qkv a column slice of a wider NaN-guarded buffer (ld = 3C + 8) and out a row-and-column window
    of a guarded buffer (ldo = C + 8); checks that no guard cell was written and returns the output on the host."""
    from aot_benchmark_b200 import ops
    C, N = heads * D, H * W
    qb = _guarded(N, 3 * C + 8)
    qb[:, 4:4 + 3 * C] = qkv.to(DEV)
    ob = _guarded(N + 2, C + 8)
    ops.window_attention(qb[:, 4:4 + 3 * C], qkv_bias.to(DEV), relb.to(DEV), ob[1:N + 1, 4:4 + C], H, W, heads, shift)
    torch.cuda.synchronize()
    bits = ob.view(torch.int32).cpu()
    inside = torch.zeros_like(bits, dtype=torch.bool)
    inside[1:N + 1, 4:4 + C] = True
    assert (bits[~inside] == GUARD).all(), "a guard row or column was written"
    out = ob[1:N + 1, 4:4 + C].cpu()
    assert not (bits[inside] == GUARD).any(), "a real token was not written"
    return out


def _assert_within(out, ref, tol, what):
    assert torch.isfinite(out).all(), what
    ratio = ((out.double() - ref).abs() / tol).max().item()
    print(f"window attention {what}: worst err / tol {ratio:.3f}")
    assert ratio <= 1.0, f"{what}: worst err / tol {ratio:.3f}"


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_window_attention(case):
    qkv, qkv_bias, relb = case_inputs(*case)
    H, W, heads, shift, _ = case
    ref, tol = window_reference(qkv, qkv_bias, relb, H, W, heads, shift)
    out = run_window(qkv, qkv_bias, relb, H, W, heads, shift)
    _assert_within(out, ref, tol, "-".join(map(str, case)))


@pytest.mark.parametrize("case", [(18, 26, 8, 3, "normal"), (5, 3, 4, 3, "mask_sharp"), (13, 6, 32, 0, "bias")],
                         ids=lambda c: "-".join(map(str, c)))
def test_window_attention_repeatable(case):
    """Dense operands, a repeated launch and two replays of a captured graph give the bits of the strided eager launch."""
    from aot_benchmark_b200 import ops
    H, W, heads, shift, _ = case
    qkv, qkv_bias, relb = case_inputs(*case)
    strided = run_window(qkv, qkv_bias, relb, H, W, heads, shift).to(DEV)
    q, b, r = qkv.to(DEV), qkv_bias.to(DEV), relb.to(DEV)
    out = _guarded(H * W, heads * D)
    for _ in range(2):
        out.fill_(math.nan)
        ops.window_attention(q, b, r, out, H, W, heads, shift)
        torch.cuda.synchronize()
        assert torch.equal(out, strided)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.window_attention(q, b, r, out, H, W, heads, shift)
    for _ in range(2):
        out.fill_(math.nan)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, strided)


# ------------------------------------------------------------------------------------------------------- patch merging
def merge_reference(x, H, W):
    """int32 bit patterns [H*W, C] -> PatchMerging's gather [ceil(H/2) * ceil(W/2), 4C] in the order (0,0), (1,0),
    (0,1), (1,1), padded with +0.0 (all-zero bits)."""
    C = x.shape[1]
    y = torch.zeros(H + H % 2, W + W % 2, C, dtype=torch.int32)
    y[:H, :W] = x.view(H, W, C)
    return torch.cat([y[0::2, 0::2], y[1::2, 0::2], y[0::2, 1::2], y[1::2, 1::2]], -1).reshape(-1, 4 * C)


def merge_steps(H, W, C):
    """Steps of the grid-stride loop: one float4 per thread, at most 132 * 16 blocks of 256 threads."""
    items = ((H + 1) // 2) * ((W + 1) // 2) * C
    threads = min(-(-items // 256), 132 * 16) * 256
    return -(-items // threads)


# odd and even H and W, single rows and columns, C 4 to 512, and config 4's two merges (148 x 260 at C 128, 74 x 130 at
# C 256), whose grid-stride loops take three and two steps
MERGE_CASES = [(8, 12, 128), (9, 13, 256), (1, 5, 128), (37, 65, 256), (1, 1, 4), (1, 7, 4), (7, 1, 4), (2, 2, 4),
               (3, 5, 4), (19, 33, 512), (6, 10, 512), (148, 260, 128), (74, 130, 256)]
assert [merge_steps(*c) for c in MERGE_CASES[-2:]] == [3, 2]


@pytest.mark.parametrize("H,W,C", MERGE_CASES)
def test_patch_merge(H, W, C):
    """Random bit patterns (every float class) plus -0.0, +-inf and a NaN payload, read from a column slice of a guarded
    buffer (ldx = C + 8) and written into a column slice of another (ldo = 4C + 12): bit-exact, guards untouched."""
    from aot_benchmark_b200 import ops
    g = torch.Generator().manual_seed(H * 1000 + W + C)
    x = torch.randint(-2 ** 31, 2 ** 31, (H * W, C), generator=g, dtype=torch.int32)
    x[0, :4] = torch.tensor([-0.0, math.inf, -math.inf, 0.0]).view(torch.int32)
    x[-1, -1] = 0x7FC0FFEE
    want = merge_reference(x, H, W)
    xb = _guarded(H * W, C + 8)
    xb.view(torch.int32)[:, 4:4 + C] = x.to(DEV)
    ob = _guarded(want.shape[0], 4 * C + 12)
    ops.patch_merge(xb[:, 4:4 + C], ob[:, 8:8 + 4 * C], H, W)
    torch.cuda.synchronize()
    bits = ob.view(torch.int32).cpu()
    assert torch.equal(bits[:, 8:8 + 4 * C], want)
    assert (bits[:, :8] == GUARD).all() and (bits[:, 8 + 4 * C:] == GUARD).all()


# --------------------------------------------------------------------------------------------------------- rejections
def _win_call(C=64, heads=2, shift=3, qkv_off=0, out_off=0, bias_off=0, bias_len=None, relb_heads=None):
    from aot_benchmark_b200 import ops
    H, W = 7, 9
    N = H * W
    qb = torch.zeros(N, 3 * C + 4, device=DEV)
    ob = torch.zeros(N, C + 4, device=DEV)
    bb = torch.zeros(3 * C + 4, device=DEV)
    rb = torch.zeros(heads if relb_heads is None else relb_heads, T, T, device=DEV)
    n = 3 * C if bias_len is None else bias_len
    ops.window_attention(qb[:, qkv_off:qkv_off + 3 * C], bb[bias_off:bias_off + n], rb, ob[:, out_off:out_off + C],
                         H, W, heads, shift)


WINDOW_REJECTS = {
    "head_dim_48": dict(C=96, heads=2),
    "shift_7": dict(shift=7),
    "misaligned_qkv": dict(qkv_off=1),
    "misaligned_out": dict(out_off=1),
    "misaligned_qkv_bias": dict(bias_off=1),
    "rel_bias_one_head_short": dict(relb_heads=1),
    "rel_bias_one_head_over": dict(relb_heads=3),
    "short_qkv_bias": dict(bias_len=3 * 64 - 4),
}


def test_window_attention_accepts_the_well_formed_call():
    _win_call()
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", list(WINDOW_REJECTS))
def test_window_attention_rejects(name):
    from aot_benchmark_b200._lib import AotbError
    with pytest.raises(AotbError):
        _win_call(**WINDOW_REJECTS[name])


def test_patch_merge_rejects_channels_not_a_multiple_of_4():
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import AotbError
    with pytest.raises(AotbError):
        ops.patch_merge(torch.zeros(4, 6, device=DEV), torch.zeros(1, 24, device=DEV), 2, 2)
