"""GPU: the entry points that run several independent videos per launch against the one-video launches on each video's
operands (bit for bit), and MultiVideoInferEngine against separate bounded AOTInferEngines, graphs against eager, fp16 and
slot compaction."""
import pytest
import torch

import bounded_bank_support as S
import test_gpu_engine_protocol as P
from oracle import aot_oracle as O
from oracle import weights as OW

pytestmark = pytest.mark.gpu
dev = "cuda"


def _packed(rows, H=8, scale=1.0, g=None):
    from aot_benchmark_b200 import ops
    x = torch.randn(rows, H * 32, device=dev, generator=g) * scale
    p = torch.zeros(H, rows, 64, dtype=torch.float16, device=dev)
    ops.tc_pack_rows(x, p, 0)
    return p


@pytest.mark.parametrize("n", [1, 2, 3, 5])
@pytest.mark.parametrize("exact", [True, False])
def test_lt_attention_batched_equals_one_video_launches(n, exact):
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200.engine import lt_splits
    g = torch.Generator(device=dev).manual_seed(n)
    N, Mf, H = 300, 4, 8
    kvs = Mf * N
    Qp = _packed(n * N, g=g, scale=3.0)
    Kp, Vp = _packed(n * kvs, g=g), _packed(n * kvs, g=g)
    live = [N * (1 + (b * 3) % Mf) for b in range(n)]
    live[0] = N                                  # one memory frame next to fuller banks
    if n > 1:
        live[-1] = kvs
    tk = torch.tensor(live, dtype=torch.int32, device=dev)
    for splits in sorted({1, 3, lt_splits(n * N, H, max(live))}):
        part = tuple(torch.empty(s, device=dev) for s in ((splits, n * N, 256), (splits, H, n * N), (splits, H, n * N)))
        O = torch.empty(n * N, 256, device=dev)
        ops.lt_attention_tc_batched(Qp, N, Kp, Vp, kvs, n, N, Tk_dev=tk, O=O, splits=splits, exact=exact, part=part)
        for b in range(n):
            q = torch.zeros(H, 512, 64, dtype=torch.float16, device=dev)
            q[:, :N] = Qp[:, b * N:(b + 1) * N]
            k, v = Kp[:, b * kvs:(b + 1) * kvs].contiguous(), Vp[:, b * kvs:(b + 1) * kvs].contiguous()
            want = torch.empty(N, 256, device=dev)
            pb = tuple(torch.empty(s, device=dev) for s in ((splits, N, 256), (splits, H, N), (splits, H, N)))
            ops.lt_attention_tc(q, k, v, N, 0, O=want, Tk_dev=tk[b:b + 1], splits=splits, exact=exact, part=pb,
                                variant="tile")
            assert torch.equal(O[b * N:(b + 1) * N], want), (b, splits)


@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_local_id_ring_batched_equal_one_video_launches(n):
    from aot_benchmark_b200 import ops
    g = torch.Generator(device=dev).manual_seed(10 + n)
    h, w, Hh = 19, 37, 8
    m = h * w
    r = lambda *s: torch.randn(*s, device=dev, generator=g)
    q, k, v = r(n * m, 256), r(n * m, 256), r(n * m, 256)
    relk_w, relk_b, relv_t = r(Hh * 225, 32), r(Hh * 225), r(Hh, 225, 32)
    out = torch.empty(n * m, 256, device=dev)
    ops.local_attention_tc_batched(q, k, v, relk_w, relk_b, relv_t, out, h, w, Hh, n)
    for b in range(n):
        s = slice(b * m, (b + 1) * m)
        want = torch.empty(m, 256, device=dev)
        ops.local_attention_tc(q[s].contiguous(), k[s].contiguous(), v[s].contiguous(), relk_w, relk_b, relv_t, want, h, w, Hh)
        assert torch.equal(out[s], want), b
    # ID embedding of n label maps
    K, st, pad, nid = 17, 16, 8, 11
    Hm, Wm = 97, 161
    masks = torch.randint(0, nid, (n, Hm, Wm), device=dev, generator=g).float()
    wp = r(K, K + 1, nid, 256)
    bias = r(256)
    ho, wo = (Hm + 2 * pad - K) // st + 1, (Wm + 2 * pad - K) // st + 1
    emb = torch.empty(n * ho * wo, 256, device=dev)
    ops.id_embed_runs_batched(masks, wp, bias, emb, 256, nid, K, st, pad)
    for b in range(n):
        want = torch.empty(ho * wo, 256, device=dev)
        ops.id_embed_runs(masks[b].contiguous(), wp, bias, want, 256, nid, K, st, pad)
        assert torch.equal(emb[b * ho * wo:(b + 1) * ho * wo], want), b
    # ring store + advance with per-video counters and store flags
    rows, Mf = 40, 3
    cap = Mf * rows
    ks, vs = r(n * rows, 256), r(n * rows, 256)
    kb, vb = torch.zeros(n * cap, 256, device=dev), torch.zeros(n * cap, 256, device=dev)
    kp, vp = (torch.zeros(8, n * cap, 64, dtype=torch.float16, device=dev) for _ in range(2))
    # the last bank is full with its write offset at its last slot: its advance wraps to the first unpinned slot
    live = torch.tensor([cap if b == n - 1 else (b % Mf) * rows for b in range(n)], dtype=torch.int32, device=dev)
    wr = torch.tensor([cap - rows if b == n - 1 else (b % Mf) * rows for b in range(n)], dtype=torch.int32, device=dev)
    flags = torch.tensor([0 if b == 1 and b != n - 1 else 1 for b in range(n)], dtype=torch.int32, device=dev)
    live0, wr0 = live.clone(), wr.clone()
    ops.bank_ring_store_batched(ks, vs, kb, vb, kp, vp, wr, flags, n, cap)
    ops.ring_advance_batched(live, wr, flags, n, rows, cap, rows)
    for b in range(n):
        c = slice(b * cap, (b + 1) * cap)
        kb1, vb1 = torch.zeros(cap, 256, device=dev), torch.zeros(cap, 256, device=dev)
        kp1, vp1 = (torch.zeros(8, cap, 64, dtype=torch.float16, device=dev) for _ in range(2))
        l1, w1 = live0[b:b + 1].clone(), wr0[b:b + 1].clone()
        if int(flags[b]):
            ops.bank_ring_store(ks[b * rows:(b + 1) * rows], vs[b * rows:(b + 1) * rows], kb1, vb1, kp1, vp1, w1)
            ops.ring_advance(l1, w1, rows, cap, rows)
        assert torch.equal(kb[c], kb1) and torch.equal(vb[c], vb1)
        assert torch.equal(kp[:, c], kp1) and torch.equal(vp[:, c], vp1)
        assert int(live[b]) == int(l1) and int(wr[b]) == int(w1)
    assert int(wr[n - 1]) == rows and int(live[n - 1]) == cap        # the wrap happened


def _model(name, sd):
    from aot_benchmark_b200 import EngineConfig, build_vos_model
    cfg = EngineConfig("t", name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd)
    return model.cuda().eval()


def _run(model, precision, graphs, monkeypatch, Hh=129, Ww=193, M=3, oracle_sd=None):
    """Three videos (lengths 7, 4, 6; one opens at step 1; video 0 gains an object at frame 3; video 1 closes from the
    middle slot) through MultiVideoInferEngine and through one AOTInferEngine each.  With oracle_sd, each video also runs
    through the float64 bounded oracle, whose argmax is fed back to every engine.  -> (max |dlogit| vs AOTInferEngine,
    label mismatch fraction, multi-video logits per step, max |dlogit| vs the oracle)."""
    from aot_benchmark_b200 import engine
    from aot_benchmark_b200.engine import AOTInferEngine
    from aot_benchmark_b200.multi_video import MultiVideoInferEngine
    monkeypatch.setattr(engine, "USE_GRAPHS", graphs)
    eng = MultiVideoInferEngine(model, max_videos=3, long_term_mem_max=M, long_term_mem_gap=2, precision=precision)
    lens, objs, t0, gaps = [7, 4, 6], [3, 2, 5], [0, 0, 1], [2, 1, 3]
    clips = [O.synthetic_video(n, Hh, Ww, o, seed=20 + i) for i, (n, o) in enumerate(zip(lens, objs))]
    refs, vids, local = {}, {}, {}
    dmax, mism, tot, trace, omax = 0.0, 0, 0, [], 0.0
    oracles = {}

    def new_oracle(gap):
        return S.BoundedOracleEngine(oracle_sd, O.OracleConfig(model.cfg.MODEL_NAME), long_term_mem_gap=gap,
                                     dtype=torch.float64, device="cuda", long_term_mem_max=M)
    with torch.no_grad():
        for step in range(8):
            for i in range(3):
                if step == t0[i]:
                    f, m = clips[i]
                    vids[i] = eng.open_video(f[0].cuda(), m.cuda(), objs[i], long_term_mem_gap=gaps[i])
                    refs[i] = AOTInferEngine(model, long_term_mem_gap=gaps[i], long_term_mem_max=M, precision=precision)
                    refs[i].add_reference_frame(f[0].cuda(), m.cuda(), obj_nums=[objs[i]], frame_step=0)
                    if oracle_sd is not None:
                        oracles[i] = new_oracle(gaps[i])
                        oracles[i].add_reference_frame(f[0].cuda(), m.cuda(), obj_nums=[objs[i]], frame_step=0)
                    local[i] = 0
            live = [i for i in vids if local[i] + 1 < lens[i]]
            for i in [i for i in vids if i not in live]:
                eng.close_video(vids.pop(i))
            if not live:
                break
            for i in live:
                local[i] += 1
            eng.propagate({vids[i]: clips[i][0][local[i]].cuda() for i in live})
            got = eng.decode_current_logits((Hh, Ww))
            trace.append({i: got[vids[i]].clone() for i in live})
            labs = eng.decode_labels((Hh, Ww))
            labels = {}
            for i in live:
                refs[i].match_propogate_one_frame(clips[i][0][local[i]].cuda())
                want = refs[i].decode_current_logits((Hh, Ww))
                k = objs[i] + 1
                dmax = max(dmax, (got[vids[i]][:, :k] - want[:, :k]).abs().max().item())
                lw = torch.argmax(want[:, :k], dim=1)
                mism += int((labs[vids[i]] != lw).sum())
                tot += lw.numel()
                labels[i] = lw.unsqueeze(1).float()
                if oracle_sd is not None:
                    oracles[i].match_propogate_one_frame(clips[i][0][local[i]].cuda().double())
                    ow = oracles[i].decode_current_logits((Hh, Ww))
                    omax = max(omax, (got[vids[i]][:, :k].double() - ow[:, :k]).abs().max().item())
                    labels[i] = torch.argmax(ow[:, :k], dim=1, keepdim=True).float()
            if 0 in live and local[0] == 3:
                objs[0] += 1
                m = labels[0].clone()
                m[..., 10:30, 10:40] = objs[0]
                eng.add_reference_frame(vids[0], clips[0][0][3].cuda(), m, objs[0])
                refs[0].add_reference_frame(clips[0][0][3].cuda(), m, obj_nums=[objs[0]], frame_step=3)
                got0 = eng.decode_current_logits((Hh, Ww))[vids[0]]
                refs[0].decode_current_logits((Hh, Ww))
                if oracle_sd is not None:
                    oracles[0].add_reference_frame(clips[0][0][3].cuda().double(), m.double(), obj_nums=[objs[0]],
                                                   frame_step=3)
                    ow = oracles[0].decode_current_logits((Hh, Ww))
                    omax = max(omax, (got0[:, :objs[0] + 1].double() - ow[:, :objs[0] + 1]).abs().max().item())
            eng.update_memory({vids[i]: labels[i] for i in live})
            for i in live:
                refs[i].update_memory(labels[i])
                if oracle_sd is not None:
                    oracles[i].update_memory(labels[i].double())
    torch.cuda.synchronize()
    return dmax, mism / max(tot, 1), trace, omax


@pytest.mark.parametrize("precision,tol", [("fp32", 2e-3), ("fp16", 5e-2)])
def test_engine_matches_separate_bounded_engines(monkeypatch, precision, tol):
    model = _model("r50_aotl", OW.build_state_dict("r50_aotl", seed=0))
    dmax, frac, _, _ = _run(model, precision, True, monkeypatch)
    assert dmax < tol, dmax
    assert frac < 1e-3, frac


def test_engine_matches_the_float64_bounded_oracle_per_video(monkeypatch):
    """Each video against its own float64 bounded oracle (the oracle's labels fed back to both), within the fp32 tolerance
    of tests/test_gpu_bounded_bank.py."""
    sd = OW.build_state_dict("r50_aotl", seed=0)
    _, _, _, omax = _run(_model("r50_aotl", sd), "fp32", True, monkeypatch, oracle_sd=sd)
    assert 0 < omax < P.TOL, f"max |dlogit| vs the float64 bounded oracle = {omax:.3e}"


def test_graphs_equal_eager(monkeypatch):
    model = _model("aott", OW.build_state_dict("aott", seed=1))
    _, _, eager, _ = _run(model, "fp32", False, monkeypatch)
    _, _, graph, _ = _run(model, "fp32", True, monkeypatch)
    assert len(eager) == len(graph)
    for a, b in zip(eager, graph):
        assert a.keys() == b.keys()
        for i in a:
            assert torch.equal(a[i], b[i]), i
