"""CPU: the usage eviction policy of the bounded long-term bank (long_term_mem_policy="usage"), driven through the emulated
entry points (tests/usage_bank_support.py): the selection rule, the product engines against the usage oracle over clips that
evict, what the captured graphs may assume, the refusals and how the policy reaches the engines."""
import ctypes
import math
import os

import pytest
import torch

import test_cpu_graph_static as GS
import usage_bank_support as S
from oracle import aot_oracle as O
from oracle import weights as OW


def _engine(model_name, sd, gap, M=None, policy=None, cfg_policy=None, phase="eval", **kw):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", model_name)
    if cfg_policy is not None:
        cfg.TEST_LONG_TERM_MEM_POLICY = cfg_policy
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    model.load_state_dict(sd, strict=True)
    if M is not None:
        kw["long_term_mem_max"] = M
    if policy is not None:
        kw["long_term_mem_policy"] = policy
    eng = build_engine(cfg.MODEL_ENGINE, phase=phase, aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                       short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP, **kw)
    eng.eval()
    return eng


# ------------------------------------------------------------------------------------------------------------------
# the selection rule and the emulated entry points
# ------------------------------------------------------------------------------------------------------------------
def _select(U, A, live, rows=5, M=4):
    live_t, write = torch.tensor([live], dtype=torch.int32), torch.tensor([-7], dtype=torch.int32)
    U, A = torch.tensor(U, dtype=torch.float32), torch.tensor(A, dtype=torch.int32)
    S.ring_select_usage(live_t, write, U, A, rows, rows * M, rows)
    return int(write) // rows, U, A


def test_selection_rule():
    # not full: the next free slot, whatever the scores
    for live in range(4):
        s, U, A = _select([0.9, 0.1, 0.0, 0.0], [3, 2, 0, 0], live * 5)
        assert s == live and U[s] == 0 and A[s] == 0
    # full: the lowest U / A among slots 1..3; slot 0 never, however low
    s, U, A = _select([0.0, 0.6, 0.3, 0.5], [9, 3, 1, 5], 20)
    assert s == 3 and U[3] == 0 and U[1] > 0 and U[2] > 0 and A.tolist() == [9, 3, 1, 0]
    # A = 0 is +inf: never chosen while another slot has been read
    assert _select([0.5, 0.0, 0.9, 0.9], [1, 0, 1, 1], 20)[0] == 2
    # ties go to the lowest slot, +inf ties included
    assert _select([0.0, 0.4, 0.2, 0.2], [1, 2, 1, 1], 20)[0] == 1
    assert _select([0.0, 0.0, 0.0, 0.0], [1, 0, 0, 0], 20)[0] == 1
    # a live count beyond the bank still selects a slot inside it
    assert _select([0.0, 0.4, 0.1, 0.2], [1, 2, 2, 2], 10 ** 6)[0] == 2


def test_emulation_argument_checks():
    from aot_benchmark_b200.ops import AotbError
    live, write = torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32)
    U, A = torch.zeros(4), torch.zeros(4, dtype=torch.int32)
    for rows, cap, pinned in ((0, 20, 0), (5, 20, 3), (5, 22, 5), (5, 20, 20), (5, 15, 5)):
        with pytest.raises(AotbError):
            S.ring_select_usage(live, write, U, A, rows, cap, pinned)
    Op, Mp, Lp = torch.zeros(33, 4, 32), torch.zeros(33, 1, 4), torch.ones(33, 1, 4)
    with pytest.raises(AotbError):
        S.attn_merge_usage(Op, Mp, Lp, torch.zeros(4, 32), 1, 32, torch.zeros(33), None, live, 4, 1, None)
    q = torch.zeros(1, 256, 64, dtype=torch.float16)
    with pytest.raises(AotbError):
        S.lt_attention_tc_slots(q, q, q, 10, torch.tensor([5], dtype=torch.int32), 1, 5, (Op, Mp, Lp))


def test_slot_split_and_merge_emulations_give_slot_masses():
    """Splits of HW rows over a bank of M slots, HW no multiple of 64, not full: each split is one slot, the masses the merge
    counts equal the float64 slot masses, and O equals the unsplit attention."""
    import emu_ops
    torch.manual_seed(0)
    H, N, HW, M, live = 8, 40, 77, 4, 3
    Q, K, V = torch.randn(N, H * 32), torch.randn(M * HW, H * 32), torch.randn(M * HW, H * 32)
    pk = lambda x, cap: emu_ops.tc_pack_rows(x, torch.zeros(H, cap, 64, dtype=torch.float16))
    Qp, Kp, Vp = pk(Q / math.sqrt(32), 256), pk(K, M * HW), pk(V, M * HW)
    tk = torch.tensor([live * HW], dtype=torch.int32)
    part = (torch.zeros(M, N, H * 32), torch.zeros(M, H, N), torch.zeros(M, H, N))
    S.lt_attention_tc_slots(Qp, Kp, Vp, N, tk, M, HW, part)
    assert torch.isinf(part[1][live:]).all() and (part[2][live:] == 0).all()
    O1, O2 = torch.zeros(N, H * 32), torch.zeros(N, H * 32)
    U, A = torch.zeros(M), torch.zeros(M, dtype=torch.int32)
    S.attn_merge_usage(*part, O1, H, 32, U, A, tk, HW, 2, None)
    emu_ops.lt_attention_tc(Qp, Kp, Vp, N, 0, O=O2, Tk_dev=tk)
    assert (O1 - O2).abs().max() < 1e-5
    want = S.slot_masses(Q.unsqueeze(1), K[:live * HW].unsqueeze(1), H, M, HW) / 2
    assert (U.double() - want).abs().max() < 1e-6 and abs(U.sum().item() - 0.5) < 1e-6
    assert A.tolist() == [1, 1, 1, 0]


# ------------------------------------------------------------------------------------------------------------------
# the engines against the usage oracle
# ------------------------------------------------------------------------------------------------------------------
def _compare_with_oracle(eng, oe, c_lo, o_lo, counts, deaot):
    for f, (sa, sb) in enumerate(zip(c_lo, o_lo)):
        for j, (a, b, c) in enumerate(zip(sa, sb, counts)):
            d = (a[:, :c + 1] - b[:, :c + 1]).abs().max().item()
            assert d < 2e-4, f"frame {f + 1}, sub-engine {j}: max |dlogit| vs the usage oracle = {d}"
    subs = getattr(eng, "aot_engines", None) or [eng]
    osubs = getattr(oe, "aot_engines", None) or [oe]
    for e, o in zip(subs, osubs):
        for c_layer, o_layer in zip(e.long_term_memories, o.long_term_memories):
            for a, b in zip(c_layer, o_layer):
                assert (a is None) == (b is None)
                if a is not None:
                    assert a.shape == b.shape and (a - b).abs().max().item() < 2e-4 * max(1.0, b.abs().max().item())
        U, A = e.long_term_memory_usage
        assert A.tolist() == o.A
        assert (U.double() - torch.tensor(o.U, dtype=torch.float64)).abs().max().item() < 2e-5
        # the engine chose the oracle's own argmin wherever that is not a near tie
        assert len(o.evictions) >= 3
        for own, gap, took in o.evictions:
            assert own == took or gap <= 1e-4, o.evictions


@pytest.mark.parametrize("name", ["r50_aotl_small", "r50_deaotl_small"])
def test_usage_engine_vs_usage_oracle_on_a_golden_clip(monkeypatch, golden_dir, name):
    """Weights and frames of a committed golden clip, gap 1, M = 3 over 8 frames: five evictions by usage."""
    S.install_engine(monkeypatch)
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    T, M = 8, 3
    sd = OW.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    frames, mask = O.synthetic_video(T, g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    oe = S.oracle(g["model"], sd, M, g["objs"])
    eng = _engine(g["model"], sd, 1, M, "usage")
    c_lo, o_lo, _ = S.run_lockstep(eng, oe, frames, mask, g["objs"], tuple(g["out_size"]))
    _compare_with_oracle(eng, oe, c_lo, o_lo, [g["objs"]], "deaot" in g["model"])
    assert len(oe.evictions) == T - M


@pytest.mark.parametrize("model_name", ["aott", "deaott"])
def test_usage_two_sub_engines_vs_usage_oracle(monkeypatch, model_name):
    S.install_engine(monkeypatch)
    H, W, objs, T, M = 65, 81, 13, 7, 3
    sd = OW.build_state_dict(model_name, seed=6)
    frames, mask = O.synthetic_video(T, H, W, objs, seed=9)
    oe = S.oracle(model_name, sd, M, objs)
    eng = _engine(model_name, sd, 1, M, "usage")
    c_lo, o_lo, _ = S.run_lockstep(eng, oe, frames, mask, objs, (H, W))
    assert len(eng.aot_engines) == len(oe.aot_engines) == 2
    _compare_with_oracle(eng, oe, c_lo, o_lo, [10, 3], model_name == "deaott")
    assert all(u is not None for u in eng.long_term_memory_usage)


def behaviour_clip(H, W, seed=21):
    """Frames f0, X, Y, X', X'': X is a synthetic frame, Y noise, X' and X'' X with small noise.  With gap 1 and M = 3 the
    first eviction (at X''s store) chooses between slot 1 (X) and slot 2 (Y)."""
    g = torch.Generator().manual_seed(seed)
    frames, mask = O.synthetic_video(4, H, W, 2, seed=seed)
    X = frames[2]
    Y = torch.randn(1, 3, H, W, generator=g) * 1.5
    rep = [X + 0.03 * torch.randn(1, 3, H, W, generator=g) for _ in range(2)]
    return [frames[0], X, Y] + rep, mask


@pytest.mark.parametrize("model_name", ["r50_aotl", "r50_deaotl"])
def test_behaviour_clip_margin_on_the_oracle(model_name):
    """The GPU behaviour test's clip: X's mean mass clearly beats Y's, so usage keeps X where FIFO evicts it."""
    H, W = 97, 129
    frames, mask = behaviour_clip(H, W)
    sd = OW.build_state_dict(model_name, seed=3)
    oe = S.oracle(model_name, sd, 3, 2)
    with torch.no_grad():
        O.run_video(oe, frames, mask, 2, (H, W))
    own, gap, took = oe.evictions[0]
    assert own == took == 2 and gap > 0.2, oe.evictions


# ------------------------------------------------------------------------------------------------------------------
# graphs, refusals, plumbing
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_name,objs", [("aott", 3), ("deaott", 3), ("aott", 12)])
def test_usage_bodies_are_static_across_frames_evictions_and_videos(monkeypatch, model_name, objs):
    """The graph tracer of test_cpu_graph_static over usage-mode clips: every replay issues the captured launches over the
    captured memory, the LSTT body has one key from the first propagated frame on (one split per slot whatever the live
    count), and the second video captures nothing new."""
    from aot_benchmark_b200 import ops
    GS._install(monkeypatch)
    import bounded_bank_support as B
    for name in B.EMULATED:
        monkeypatch.setattr(ops, name, GS._traced(name, getattr(B, name)))
    for name in S.EMULATED:
        monkeypatch.setattr(ops, name, GS._traced(name, getattr(S, name)))
    M, T, H, W = 3, 10, 97, 129
    sd = OW.build_state_dict(model_name, seed=4)
    eng = _engine(model_name, sd, 1, M, "usage")
    captured = lambda: sum(1 for e in eng.aot_engines for s in e.graphs.slots.values() if s[1] is not None)
    log, outs = [], []
    for video in range(2):
        frames, mask = O.synthetic_video(T, H, W, objs, seed=31 + video)
        with torch.no_grad():
            lo, _ = O.run_video(eng, frames, mask, objs, (H, W),
                                on_frame=lambda t, *_: log.append((video, t, captured(), GS.TracingGraphCache.replays)))
        outs.append(lo)
    subs = len(eng.aot_engines)
    assert subs == (objs + 9) // 10
    for e in eng.aot_engines:
        assert len({k for k in e.graphs.slots if k[0] == "lstt"}) == 1
    settled = [r for r in log if r[0] == 0 and r[1] >= 3]
    assert len({r[2] for r in settled}) == 1, f"bodies captured after frame 2: {settled}"
    assert {r[2] for r in log if r[0] == 1} == {settled[-1][2]}
    per_frame = [b[3] - a[3] for a, b in zip(settled, settled[1:])]
    assert all(n == 1 + 3 * subs for n in per_frame), per_frame
    assert T - M >= 3


def test_refusals_and_errors(monkeypatch):
    from aot_benchmark_b200 import engine, ops
    S.install_engine(monkeypatch)
    sd = OW.build_state_dict("aott", seed=4)
    with pytest.raises(ValueError, match="long_term_mem_policy"):
        _engine("aott", sd, 1, 3, "lru")
    with pytest.raises(ValueError, match="long_term_mem_max"):
        _engine("aott", sd, 1, None, "usage")
    with pytest.raises(ValueError, match="long_term_mem_max"):
        _engine("aott", sd, 1, None, cfg_policy="usage", phase="train")
    with pytest.raises(NotImplementedError, match="32"):
        _engine("aott", sd, 1, 33, "usage")
    monkeypatch.setattr(engine, "LT_IMPL", "simt")
    with pytest.raises(NotImplementedError, match="AOTB_LT_IMPL=simt"):
        _engine("aott", sd, 1, 3, "usage")
    _engine("aott", sd, 1, 3, "fifo")                                        # FIFO keeps every path
    monkeypatch.setattr(engine, "LT_IMPL", "tc_exact")
    monkeypatch.setattr(ops, "LT_VARIANT", "groups")
    with pytest.raises(NotImplementedError, match="AOTB_LT_VARIANT=groups"):
        _engine("aott", sd, 1, 3, "usage", phase="train")
    monkeypatch.setattr(ops, "LT_VARIANT", "tile")
    dsd = OW.build_state_dict("deaott", seed=4)
    for impl in ("simt", "gemm"):
        monkeypatch.setattr(engine, "DEAOT_LT", impl)
        with pytest.raises(NotImplementedError, match=f"AOTB_DEAOT_LT={impl}"):
            _engine("deaott", dsd, 1, 3, "usage")
    monkeypatch.setattr(engine, "DEAOT_LT", "tc")
    eng = _engine("aott", sd, 1, 3, "usage")
    with pytest.raises(NotImplementedError, match="shard"):
        eng.enable_kv_sharding(0, 2)
    from aot_benchmark_b200 import TTAInferEngine, EngineConfig, build_vos_model
    cfg = EngineConfig("t", "aott")
    with pytest.raises(ValueError, match="long_term_mem_max"):
        TTAInferEngine(build_vos_model(cfg.MODEL_VOS, cfg), long_term_mem_policy="usage")


@pytest.mark.parametrize("model_name", ["aott", "deaott"])
def test_policy_from_config_keyword_and_sub_engines(monkeypatch, model_name):
    S.install_engine(monkeypatch)
    sd = OW.build_state_dict(model_name, seed=4)
    assert _engine(model_name, sd, 1, 3).long_term_mem_policy == "fifo"
    assert _engine(model_name, sd, 1, 3, cfg_policy="usage").long_term_mem_policy == "usage"
    assert _engine(model_name, sd, 1, 3, "fifo", cfg_policy="usage").long_term_mem_policy == "fifo"
    eng = _engine(model_name, sd, 1, 3, cfg_policy="usage")
    frames, mask = O.synthetic_video(5, 65, 81, 12, seed=3)
    with torch.no_grad():
        O.run_video(eng, frames, mask, 12, (65, 81))
    assert len(eng.aot_engines) == 2
    for e in eng.aot_engines:
        assert e.long_term_mem_policy == "usage"
        U, A = e.long_term_memory_usage
        # 4 propagated frames; the last store (an eviction) restarted one unpinned slot
        assert A[0] == 4 and sorted(A[1:].tolist())[0] == 0 and 0 < U.sum().item() < 4
    assert torch.equal(eng.long_term_memory_usage[0][1], eng.aot_engines[0].long_term_memory_usage[1])
    eng.restart_engine()
    fifo = _engine(model_name, sd, 1, 3)
    with torch.no_grad():
        O.run_video(fifo, frames[:3], mask, 2, (65, 81))
    assert fifo.aot_engines[0].long_term_memory_usage is None
    # restart zeroes the counters; a pooled sub-engine follows the facade's policy
    e0 = eng.aot_engines[0] if eng.aot_engines else eng._pool[0]
    e0.restart_engine()
    U, A = e0.long_term_memory_usage
    assert not U.any() and not A.any()
    from aot_benchmark_b200 import TTAInferEngine, EngineConfig, build_vos_model
    cfg = EngineConfig("t", model_name)
    tta = TTAInferEngine(build_vos_model(cfg.MODEL_VOS, cfg), flip=True, long_term_mem_max=3, long_term_mem_policy="usage")
    assert all(e.long_term_mem_policy == "usage" for e in tta.aug_engines)


def test_new_entry_points_are_declared_and_exported():
    from aot_benchmark_b200 import _lib
    decl = _lib.parse_header()
    assert os.path.exists(_lib.LIB_PATH), "build the library first"
    h = ctypes.CDLL(_lib.LIB_PATH)
    for name, nargs, ret in (("aotb_lt_attn_tc_slots_f16x2", 16, "int"), ("aotb_gp_attn_tc_slots_f16x2", 16, "int"),
                             ("aotb_attn_merge_usage_f32", 16, "int"), ("aotb_attn_merge_usage_workspace_bytes", 1, "size_t"),
                             ("aotb_ring_select_usage", 8, "int")):
        assert name in decl and len(decl[name][1]) == nargs and decl[name][0] == ret, (name, decl.get(name))
        assert hasattr(h, name)
