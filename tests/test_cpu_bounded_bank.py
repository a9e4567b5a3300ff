"""CPU: the bounded long-term bank (long_term_mem_max = M) of the product engines, driven through the emulated entry points
(tests/emu_ops.py, tests/bounded_bank_support.py): which frame each slot holds, the two device counters, the oracle with the
same policy, the unbounded engine while nothing has been evicted, what the captured graphs may assume, the refused
combinations and how the bound reaches the engines."""
import ctypes
import os

import pytest
import torch

import bounded_bank_support as S
import test_cpu_graph_static as GS
from oracle import aot_oracle as O
from oracle import weights as OW


def _engine(model_name, sd, gap, M=None, cfg_M=None, **kw):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", model_name)
    if cfg_M is not None:
        cfg.TEST_LONG_TERM_MEM_MAX = cfg_M
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    model.load_state_dict(sd, strict=True)
    if M is not None:
        kw["long_term_mem_max"] = M
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                       short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP, **kw)
    eng.eval()
    return eng


def _policy(M, stored):
    """Frame index held by each slot after `stored` frames: slot 0 pinned, slots 1 .. M - 1 a FIFO ring."""
    slots, nxt = [], 1
    for f in range(stored):
        if len(slots) < M:
            slots.append(f)
        else:
            slots[nxt] = f
            nxt = nxt + 1 if nxt + 1 < M else 1
    return slots


def test_policy_model_keeps_the_first_and_the_newest_frames():
    for M in (2, 3, 5, 8):
        for stored in range(1, 40):
            s = _policy(M, stored)
            assert s[0] == 0 and set(s) == {0} | set(range(max(1, stored - (M - 1)), stored))


@pytest.mark.parametrize("model_name,lt_impl", [("aott", "tc_exact"), ("aott", "simt"), ("deaott", "tc_exact")])
@pytest.mark.parametrize("M", [2, 3, 5])
def test_slot_bookkeeping(monkeypatch, model_name, lt_impl, M):
    """12 stored frames, each tagged with its index: every slot of every copy of the bank holds the frame the policy says."""
    from aot_benchmark_b200 import engine
    S.install_engine(monkeypatch)
    monkeypatch.setattr(engine, "LT_IMPL", lt_impl)
    stored = [0]
    latest = engine.AOTEngine._latest_kv

    def tagged(self):
        K, V = latest(self)
        i = float(stored[0])
        stored[0] += 1
        return [torch.full_like(k, i) for k in K], [torch.full_like(v, i) for v in V]
    monkeypatch.setattr(engine.AOTEngine, "_latest_kv", tagged)
    sd = OW.build_state_dict(model_name, seed=4)
    eng = _engine(model_name, sd, 1, M)
    frames, mask = O.synthetic_video(12, 65, 81, 2, seed=3)

    def check(t, *_):
        e = eng.aot_engines[0]
        N, want = e.enc_hw, _policy(M, t + 1)
        assert stored[0] == t + 1
        assert e.bank_cap == M * N and e.bank_len == len(want) * N == int(e.tk_dev.item())
        assert N <= int(e.wr_dev.item()) <= M * N - N and int(e.wr_dev.item()) % N == 0
        packed = (e.bank_Kp, e.bank_Vp) if e._tc else (e.bank_gpK, e.bank_gpV) if e._gp_tc else None
        assert (packed is not None) == (lt_impl != "simt")
        for li in range(len(e.bank_K)):
            for s, f in enumerate(want):
                for bank in (e.bank_K[li], e.bank_V[li]):
                    assert (bank[s * N:(s + 1) * N] == f).all(), f"frame {t}, layer {li}: slot {s} should hold frame {f}"
                for p in packed or ():
                    assert p[li].shape[1] == M * N
                    assert (p[li][:, s * N:(s + 1) * N, :32] == f).all() and (p[li][:, s * N:(s + 1) * N, 32:] == 0).all()
            mem = e.long_term_memories[li]
            assert mem[0].shape[0] == len(want) * N and (mem[0].view(len(want), N, -1)[:, 0, 0] == torch.tensor(want)).all()
    with torch.no_grad():
        O.run_video(eng, frames, mask, 2, (65, 81), on_frame=check)
    assert stored[0] == 12


def test_ring_advance_emulation_vs_model_and_rejected_arguments():
    from aot_benchmark_b200.ops import AotbError
    for rows, M in ((1, 2), (7, 3), (63, 5), (1674, 8)):
        cap = rows * M
        live, write = torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32)
        hl, hw = 0, 0
        for step in range(300):
            assert 0 <= hw and hw + rows <= cap                  # a store at the current offset fits
            S.ring_advance(live, write, rows, cap, rows)
            hl = min(hl + rows, cap)
            hw = hw + rows
            if hw + rows > cap:
                hw = rows
            assert (int(live), int(write)) == (hl, hw), (rows, M, step)
    live, write = torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32)
    for bad in ((0, 8, 0), (-4, 8, 4), (4, 8, -4), (4, 4, 4), (4, 10, 4), (3, 8, 4)):
        with pytest.raises(AotbError):
            S.ring_advance(live, write, *bad)
    assert int(live) == 0 and int(write) == 0


def test_ring_store_emulation_drops_a_store_that_does_not_fit():
    k, v = torch.ones(4, 32), torch.ones(4, 64)
    kb, vb = torch.zeros(8, 32), torch.zeros(8, 64)
    kp, vp = torch.zeros(1, 8, 64, dtype=torch.float16), torch.zeros(2, 8, 64, dtype=torch.float16)
    S.bank_ring_store(k, v, kb, vb, kp, vp, torch.tensor([6], dtype=torch.int32))
    assert not kb.any() and not vb.any() and not kp.any() and not vp.any()
    S.bank_ring_store(k, v, kb, vb, kp, None, torch.tensor([4], dtype=torch.int32))
    assert (kb[4:] == 1).all() and (vb[4:] == 1).all() and (kp[:, 4:, :32] == 1).all() and not kb[:4].any() and not vp.any()


@pytest.mark.parametrize("name", ["aott_raw_257", "deaott_small", "r50_aotl_small"])
def test_bounded_engine_vs_bounded_oracle_on_a_golden_clip(monkeypatch, golden_dir, name):
    """Weights and frames of a committed golden clip, gap 1, M = 3 over 8 frames: five evictions.  The oracle keeps its bounded
    memory in slot order, so the banks compare row for row."""
    S.install_engine(monkeypatch)
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    T, M = 8, 3
    sd = OW.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    frames, mask = O.synthetic_video(T, g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    out = tuple(g["out_size"])
    oe = S.BoundedOracleEngine(sd, O.OracleConfig(g["model"]), long_term_mem_gap=1, long_term_mem_max=M)
    eng = _engine(g["model"], sd, 1, M)
    with torch.no_grad():
        o_lo, o_labels = O.run_video(oe, frames, mask, g["objs"], out)
        c_lo, _ = O.run_video(eng, frames, mask, g["objs"], out, forced_masks=o_labels)
    n = g["objs"] + 1
    dmax = max((a[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(c_lo, o_lo))
    assert dmax < 2e-4, f"max |dlogit| vs the bounded oracle = {dmax}"
    e0 = eng.aot_engines[0]
    assert e0.bank_len == M * e0.enc_hw and T - M >= 3
    for c_layer, o_layer in zip(e0.long_term_memories, oe.long_term_memories):
        for a, b in zip(c_layer, o_layer):
            assert (a is None) == (b is None)
            if a is not None:
                assert a.shape == b.shape and (a - b).abs().max().item() < 2e-4 * max(1.0, b.abs().max().item())
    # the unbounded oracle sees other keys by now
    ou = O.OracleEngine(sd, O.OracleConfig(g["model"]), long_term_mem_gap=1)
    with torch.no_grad():
        u_lo, _ = O.run_video(ou, frames, mask, g["objs"], out, forced_masks=o_labels)
    assert torch.equal(u_lo[M - 1], o_lo[M - 1]) or (u_lo[M - 1] - o_lo[M - 1]).abs().max().item() < 1e-5   # nothing evicted yet
    assert (u_lo[-1][:, :n] - o_lo[-1][:, :n]).abs().max().item() > 1e-4


@pytest.mark.parametrize("model_name,objs", [("aott", 3), ("deaott", 3), ("aott", 14)])
def test_bound_never_reached_is_the_unbounded_engine(monkeypatch, model_name, objs):
    S.install_engine(monkeypatch)
    sd = OW.build_state_dict(model_name, seed=5)
    frames, mask = O.synthetic_video(6, 97, 129, objs, seed=17)
    runs = []
    for M in (None, 6, 9):                                       # 6 stored frames: M = 6 fills the bank exactly
        eng = _engine(model_name, sd, 1, M)
        with torch.no_grad():
            runs.append(O.run_video(eng, frames, mask, objs, (97, 129)))
        assert all(e.bank_len == 6 * e.enc_hw for e in eng.aot_engines)
    for lo, labels in runs[1:]:
        for a, b in zip(lo, runs[0][0]):
            assert torch.equal(a, b)
        for a, b in zip(labels, runs[0][1]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("model_name,lt_impl,deaot_lt,objs", [("aott", "tc_exact", "tc", 3), ("aott", "simt", "tc", 3),
                                                              ("deaott", "tc_exact", "tc", 3), ("deaott", "tc_exact", "simt", 12)])
def test_captured_bodies_are_static_once_the_ring_is_full(monkeypatch, model_name, lt_impl, deaot_lt, objs):
    """The graph tracer of test_cpu_graph_static over bounded clips: every replay issues the captured launches over the captured
    memory (the tracer asserts it), and from the second frame after the ring filled no body is captured again -- the live
    row count and the write offset are device counters, and the KV-split count no longer changes."""
    from aot_benchmark_b200 import engine, ops
    GS._install(monkeypatch)
    for name in S.EMULATED:                                      # the two entry points of the bounded bank, traced like the rest
        monkeypatch.setattr(ops, name, GS._traced(name, getattr(S, name)))
    monkeypatch.setattr(engine, "LT_IMPL", lt_impl)
    monkeypatch.setattr(engine, "DEAOT_LT", deaot_lt)
    M, T, H, W = 3, 14, 97, 129
    sd = OW.build_state_dict(model_name, seed=4)
    eng = _engine(model_name, sd, 1, M)
    captured = lambda: sum(1 for e in eng.aot_engines for s in e.graphs.slots.values() if s[1] is not None)
    log = []
    outs = []
    for video in range(2):                                       # the second video replays the first one's graphs
        frames, mask = O.synthetic_video(T, H, W, objs, seed=31)
        with torch.no_grad():
            lo, _ = O.run_video(eng, frames, mask, objs, (H, W),
                                on_frame=lambda t, *_: log.append((video, t, captured(), GS.TracingGraphCache.replays)))
        outs.append(lo)
    subs = len(eng.aot_engines)
    assert subs == (objs + 9) // 10
    # video 0: the ring is full after frame M - 1; frame M runs the full-bank bodies eagerly, frame M + 1 captures them
    settled = [r for r in log if r[0] == 0 and r[1] >= M + 1]
    assert len({r[2] for r in settled}) == 1, f"bodies captured after the ring filled: {settled}"
    per_frame = [b[3] - a[3] for a, b in zip(settled, settled[1:])]
    # the shared encoder, then LSTT, decoder and memory update of every sub-engine: all replayed
    assert all(n == 1 + 3 * subs for n in per_frame), per_frame
    # video 1: same engine, same geometry -> nothing new is captured at all
    assert {r[2] for r in log if r[0] == 1} == {settled[-1][2]}
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    for e in eng.aot_engines:
        assert e.bank_len == M * e.enc_hw


def test_refused_combinations(monkeypatch):
    from aot_benchmark_b200 import engine
    S.install_engine(monkeypatch)
    sd = OW.build_state_dict("aott", seed=4)
    for bad in (1, 0, -3, 2.5):
        with pytest.raises(ValueError, match="long_term_mem_max"):
            _engine("aott", sd, 1, bad)
    with pytest.raises(ValueError, match="long_term_mem_max"):
        _engine("aott", sd, 1, cfg_M=1)
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", "aott")
    model = build_vos_model(cfg.MODEL_VOS, cfg).eval()
    with pytest.raises(ValueError, match="long_term_mem_max"):
        build_engine(cfg.MODEL_ENGINE, phase="train", aot_model=model, long_term_mem_max=1)
    # sharding: on the facade before any sub-engine exists, and on a single engine
    eng = _engine("aott", sd, 1, 4)
    with pytest.raises(NotImplementedError, match="shard"):
        eng.enable_kv_sharding(0, 2)
    single = build_engine(cfg.MODEL_ENGINE, phase="train", aot_model=model, long_term_mem_max=4)
    with pytest.raises(NotImplementedError, match="shard"):
        single.enable_kv_sharding(0, 2)
    # the GEMM formulation of DeAOT's long-term attention
    monkeypatch.setattr(engine, "DEAOT_LT", "gemm")
    dsd = OW.build_state_dict("deaott", seed=4)
    frames, mask = O.synthetic_video(2, 65, 81, 2, seed=3)
    deng = _engine("deaott", dsd, 1, 4)
    with pytest.raises(NotImplementedError, match="gemm"):
        deng.add_reference_frame(frames[0], mask, obj_nums=[2], frame_step=0)
    _engine("deaott", dsd, 1).add_reference_frame(frames[0], mask, obj_nums=[2], frame_step=0)      # unbounded: still runs


@pytest.mark.parametrize("model_name", ["aott", "deaott"])
def test_bound_from_the_config_reaches_every_sub_engine(monkeypatch, model_name):
    """build_engine with the reference's keyword set only: the bound comes from cfg.TEST_LONG_TERM_MEM_MAX.  Video 1 has 3
    objects (one sub-engine), video 2 has 14 (the pooled engine and a new one): both are bounded, and changing the bound on
    the facade re-allocates the pooled engine's bank."""
    S.install_engine(monkeypatch)
    sd = OW.build_state_dict(model_name, seed=4)
    eng = _engine(model_name, sd, 1, cfg_M=3)
    assert eng.long_term_mem_max == 3
    frames, mask = O.synthetic_video(6, 65, 81, 3, seed=3)
    with torch.no_grad():
        O.run_video(eng, frames, mask, 3, (65, 81))
    first = eng.aot_engines[0]
    assert len(eng.aot_engines) == 1 and first.long_term_mem_max == 3 and first.bank_len == first.bank_cap == 3 * first.enc_hw
    frames, mask = O.synthetic_video(6, 65, 81, 14, seed=3)
    eng.long_term_mem_max = 4
    with torch.no_grad():
        O.run_video(eng, frames, mask, 14, (65, 81))
    assert len(eng.aot_engines) == 2 and eng.aot_engines[0] is first
    for e in eng.aot_engines:
        assert e.long_term_mem_max == 4 and e.bank_len == e.bank_cap == 4 * e.enc_hw
    # the keyword wins over the config; no bound anywhere leaves the engine unbounded
    assert _engine(model_name, sd, 1, M=5, cfg_M=3).long_term_mem_max == 5
    assert _engine(model_name, sd, 1).long_term_mem_max is None


def test_new_entry_points_are_declared_and_exported():
    from aot_benchmark_b200 import _lib
    decl = _lib.parse_header()
    assert os.path.exists(_lib.LIB_PATH), "build the library first"
    h = ctypes.CDLL(_lib.LIB_PATH)
    for name, nargs in (("aotb_bank_ring_store", 16), ("aotb_ring_advance", 6)):
        assert name in decl and len(decl[name][1]) == nargs and decl[name][0] == "int"
        assert hasattr(h, name)
