"""GPU: the tensor-core short-term local attention (local_attn_mma_kernel, AOT head shape: 8 heads x 32, 15 x 15 window,
relative_emb_k and relative_emb_v) against the float64 oracle, at the engine's maps and where the window is wider than the map.

Every product runs in split fp16x2 (DESIGN 3.1): an element of q, q / T, k, relative_emb_k, p, v or relative_emb_v carries a
relative error of 2^-22 and an absolute floor of 2^-25.  Per (query, head), with S_j = sum_c |q_c / T||k_c| + |q_c||w_c| + |b|
the magnitude of tap j's score, and F_j = sum_c |q_c| / T + |k_c| + |q_c| + |w_c| the operands the floor applies to:

  score       ds = max_j  2^-21 S_j + 2^-25 F_j + 2^-23 (8 + 4 sqrt(32)) S_j
  output      |o - o64| <= (2 ds + 2^-21 + 2^-23 (8 + 2 sqrt(225))) sum_j p_j |u_j|  +  2^-25 sum_j |u_j|

with u_j = v_j + relv_j (v zero outside the frame): a score error ds moves p by 2 ds relative; the P and V splits cost 2^-21
relative and the P floor 2^-25 per tap; the fp32 sums over taps and channels add the 2^-23 terms."""
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
H, D, P = 8, 32, 225
# the two engine maps (31 x 54: R50, MobileNetV3, ResNeSt; 37 x 65: SwinB), maps narrower than the window, and widths that
# are no multiple of the 16-query tile (and heights no multiple of its 8 rows)
SHAPES = [(31, 54), (37, 65), (8, 8), (5, 40), (13, 22), (9, 17), (3, 1)]


def _dev():
    return torch.device("cuda:0")


def _inputs(h, w, qscale, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(1, H * D, h, w, generator=g) * qscale
    k = torch.randn(1, H * D, h, w, generator=g)
    v = torch.randn(1, H * D, h, w, generator=g)
    rkw = torch.randn(H * P, D, 1, 1, generator=g) * 0.2
    rkb = torch.randn(H * P, generator=g) * 0.1
    rv = torch.randn(H, D, P, generator=g) * 0.3
    return q, k, v, rkw, rkb, rv


def _reference(q, k, v, rkw, rkb, rv):
    """float64 oracle output [hw, H*D] and the bound above, both computed on the GPU."""
    from test_gpu_local_attn_tc_range import local_law
    return local_law(q, k, v, rkw, rkb, rv, _dev())


def _tok(t):
    return t[0].permute(1, 2, 0).reshape(t.shape[2] * t.shape[3], -1).contiguous()


def _engine_slices(q, k, v):
    """q, k, v as column slices of one wider [hw, ...] buffer, the way the engine passes them."""
    tq, tk, tv = _tok(q), _tok(k), _tok(v)
    C = H * D
    buf = torch.zeros(tq.shape[0], 3 * C + 24, device=_dev())
    buf[:, 4:4 + C] = tq.to(_dev())
    buf[:, 12 + C:12 + 2 * C] = tk.to(_dev())
    buf[:, 20 + 2 * C:20 + 3 * C] = tv.to(_dev())
    return buf[:, 4:4 + C], buf[:, 12 + C:12 + 2 * C], buf[:, 20 + 2 * C:20 + 3 * C]


def _weights(rkw, rkb, rv):
    d = _dev()
    return rkw.view(H * P, D).contiguous().to(d), rkb.to(d), rv.permute(0, 2, 1).contiguous().to(d)


def _run(qs, ks, vs, w2, b2, rvt, h, w, c0=36):
    from aot_benchmark_b200 import ops
    ob = torch.full((h * w, H * D + 40), float("nan"), device=_dev())
    ops.local_attention_tc(qs, ks, vs, w2, b2, rvt, ob[:, c0:c0 + H * D], h, w, H)
    torch.cuda.synchronize()
    assert torch.isnan(ob[:, :c0]).all() and torch.isnan(ob[:, c0 + H * D:]).all(), "wrote outside its columns"
    return ob[:, c0:c0 + H * D]


@pytest.mark.parametrize("qscale", [1.0, 30.0])
@pytest.mark.parametrize("h,w", SHAPES)
def test_local_attention_tc_vs_float64(h, w, qscale):
    q, k, v, rkw, rkb, rv = _inputs(h, w, qscale, seed=h * 1000 + w + int(qscale))
    ref, tol = _reference(q, k, v, rkw, rkb, rv)
    out = _run(*_engine_slices(q, k, v), *_weights(rkw, rkb, rv), h, w)
    assert torch.isfinite(out).all()
    err = (out.double() - ref).abs()
    ratio = (err / tol).max().item()
    assert ratio <= 1.0, f"max |err| {err.max().item():.3e}, worst err / bound {ratio:.3f}"


@pytest.mark.parametrize("h,w", [(31, 54), (13, 22)])
def test_local_attention_tc_value_scale_equivariant(h, w):
    """V and relative_emb_v scaled by 2^c: with their fp16 halves normal before and after (exact hi + lo pairs, c = -2 .. 14)
    every split and every product scales exactly, so the output is bitwise 2^c times."""
    from test_gpu_tc_operand_range import exact_pairs
    q, k, _, rkw, rkb, _ = _inputs(h, w, 1.0, seed=7)
    v = exact_pairs((1, H * D, h, w), 8)
    rv = exact_pairs((H, D, P), 9)
    qs, ks, vs = _engine_slices(q, k, v)
    w2, b2, rvt = _weights(rkw, rkb, rv)
    base = _run(qs, ks, vs, w2, b2, rvt, h, w).clone()
    for c in (-2, 5, 14):
        scaled = _run(qs, ks, vs * 2.0 ** c, w2, b2, rvt * 2.0 ** c, h, w)
        assert torch.equal(scaled, base * 2.0 ** c), c


def test_local_attention_tc_graph_replay_matches_eager():
    from aot_benchmark_b200 import ops
    h, w = 31, 54
    q, k, v, rkw, rkb, rv = _inputs(h, w, 1.0, seed=11)
    qs, ks, vs = _engine_slices(q, k, v)
    w2, b2, rvt = _weights(rkw, rkb, rv)
    eager = _run(qs, ks, vs, w2, b2, rvt, h, w).clone()
    out = torch.full((h * w, H * D), float("nan"), device=_dev())
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        ops.local_attention_tc(qs, ks, vs, w2, b2, rvt, out, h, w, H)     # module load before the capture
        st.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=st):
            ops.local_attention_tc(qs, ks, vs, w2, b2, rvt, out, h, w, H)
    out.fill_(float("nan"))
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
