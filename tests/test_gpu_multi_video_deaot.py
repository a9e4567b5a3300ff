"""GPU: the entry points that run DeAOT's gated propagation for several independent videos per launch against the one-video
launches on each video's operands (bit for bit), and DeAOTMultiVideoInferEngine against separate bounded DeAOTInferEngines
and the float64 bounded oracle, in fp32 and fp16, and graphs against eager."""
import pytest
import torch

import test_gpu_engine_protocol as P
import test_gpu_multi_video as MV
from oracle import weights as OW

pytestmark = pytest.mark.gpu
dev = "cuda"


def _packed(rows, chunks, g, scale=1.0):
    from aot_benchmark_b200 import ops
    x = torch.randn(rows, chunks * 32, device=dev, generator=g) * scale
    p = torch.zeros(chunks, rows, 64, dtype=torch.float16, device=dev)
    ops.tc_pack_rows(x, p, 0)
    return p


def _one_video(Qp, Kp, Vp, N, Tk, Tk_dev, splits, exact):
    """gp_attention_tc on one video's operands, Q padded to 128 rows as the one-video engine keeps it."""
    from aot_benchmark_b200 import ops
    q = torch.zeros(4, ((N + 127) // 128) * 128, 64, dtype=torch.float16, device=dev)
    q[:, :N] = Qp
    dv = Vp.shape[0] * 32
    out = torch.empty(N, dv, device=dev)
    part = tuple(torch.empty(s, device=dev) for s in ((splits, N, dv), (splits, 1, N), (splits, 1, N)))
    ops.gp_attention_tc(q, Kp.contiguous(), Vp.contiguous(), N, Tk, O=out, Tk_dev=Tk_dev, splits=splits, exact=exact,
                        part=part)
    return out


@pytest.mark.parametrize("n", [1, 2, 3, 5])
@pytest.mark.parametrize("exact", [True, False])
def test_gp_attention_batched_equals_one_video_launches(n, exact):
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200.engine import gp_splits
    g = torch.Generator(device=dev).manual_seed(n)
    N, Mf, dv = 300, 4, 1024
    kvs = Mf * N
    Qp = _packed(n * N, 4, g, scale=3.0)
    Kp, Vp = _packed(n * kvs, 4, g), _packed(n * kvs, dv // 32, g)
    live = [N * (1 + (b * 3) % Mf) for b in range(n)]
    live[0] = N                                  # one memory frame next to fuller banks
    if n > 1:
        live[-1] = kvs
    tk = torch.tensor(live, dtype=torch.int32, device=dev)
    for splits in sorted({1, 3, gp_splits(n * N, 256, max(live))}):
        part = tuple(torch.empty(s, device=dev) for s in ((splits, n * N, dv), (splits, 1, n * N), (splits, 1, n * N)))
        O = torch.empty(n * N, dv, device=dev)
        ops.gp_attention_tc_batched(Qp, N, Kp, Vp, kvs, n, N, Tk_dev=tk, O=O, splits=splits, exact=exact, part=part)
        for b in range(n):
            kv = slice(b * kvs, (b + 1) * kvs)
            want = _one_video(Qp[:, b * N:(b + 1) * N], Kp[:, kv], Vp[:, kv], N, 0, tk[b:b + 1], splits, exact)
            assert torch.equal(O[b * N:(b + 1) * N], want), (b, splits)
    # the self-attention form: every video's own N keys, no live counts
    Ks, Vs = _packed(n * N, 4, g), _packed(n * N, dv // 32, g)
    for splits in (1, 2):
        part = tuple(torch.empty(s, device=dev) for s in ((splits, n * N, dv), (splits, 1, n * N), (splits, 1, n * N)))
        O = torch.empty(n * N, dv, device=dev)
        ops.gp_attention_tc_batched(Qp, N, Ks, Vs, N, n, N, Tk=N, O=O, splits=splits, exact=exact, part=part)
        for b in range(n):
            r = slice(b * N, (b + 1) * N)
            want = _one_video(Qp[:, r], Ks[:, r], Vs[:, r], N, N, None, splits, exact)
            assert torch.equal(O[r], want), ("self", b, splits)


@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_local_gated_tile_batched_equals_one_video_launches(n):
    from aot_benchmark_b200 import ops
    g = torch.Generator(device=dev).manual_seed(20 + n)
    r = lambda *s: torch.randn(*s, device=dev, generator=g)
    relk_w, relk_b = r(225, 128) * 0.1, r(225)
    for h, w in ((31, 54), (13, 22), (9, 17)):               # partial 8 x 6 tiles in both directions
        m = h * w
        q, k, v = r(n * m, 128), r(n * m, 128), r(n * m, 1024)
        out = torch.empty(n * m, 1024, device=dev)
        ops.local_gated_tile_batched(q, k, v, relk_w, relk_b, out, h, w, n)
        for b in range(n):
            s = slice(b * m, (b + 1) * m)
            want = torch.empty(m, 1024, device=dev)
            ops.local_gated_tile(q[s].contiguous(), k[s].contiguous(), v[s].contiguous(), relk_w, relk_b, want, h, w)
            assert torch.equal(out[s], want), (h, w, b)


def _run(model, precision, graphs, monkeypatch, oracle_sd=None):
    """test_gpu_multi_video._run (three videos that open at different steps, gain an object mid-clip and close from the
    middle slot) with DeAOTMultiVideoInferEngine and one bounded DeAOTInferEngine per video in place of the AOT classes."""
    from aot_benchmark_b200 import engine, multi_video
    with monkeypatch.context() as m:
        m.setattr(multi_video, "MultiVideoInferEngine", multi_video.DeAOTMultiVideoInferEngine)
        m.setattr(engine, "AOTInferEngine", engine.DeAOTInferEngine)
        return MV._run(model, precision, graphs, m, oracle_sd=oracle_sd)


@pytest.mark.parametrize("precision,tol", [("fp32", 2e-3), ("fp16", 5e-2)])
def test_engine_matches_separate_bounded_engines(monkeypatch, precision, tol):
    model = MV._model("r50_deaotl", OW.build_state_dict("r50_deaotl", seed=0))
    dmax, frac, _, _ = _run(model, precision, True, monkeypatch)
    print(f"R50-DeAOTL {precision}: max |dlogit| vs separate engines {dmax:.3e}, label mismatch {frac:.2e}")
    assert dmax < tol, dmax
    assert frac < 1e-3, frac


def test_engine_matches_the_float64_bounded_oracle_per_video(monkeypatch):
    sd = OW.build_state_dict("r50_deaotl", seed=0)
    _, _, _, omax = _run(MV._model("r50_deaotl", sd), "fp32", True, monkeypatch, oracle_sd=sd)
    print(f"R50-DeAOTL: max |dlogit| vs the float64 bounded oracle {omax:.3e}")
    assert 0 < omax < P.TOL, f"max |dlogit| vs the float64 bounded oracle = {omax:.3e}"


def test_graphs_equal_eager(monkeypatch):
    model = MV._model("deaott", OW.build_state_dict("deaott", seed=1))
    _, _, eager, _ = _run(model, "fp32", False, monkeypatch)
    _, _, graph, _ = _run(model, "fp32", True, monkeypatch)
    assert len(eager) == len(graph)
    for a, b in zip(eager, graph):
        assert a.keys() == b.keys()
        for i in a:
            assert torch.equal(a[i], b[i]), i
