"""GPU: the bounded long-term bank (long_term_mem_max = M: the first memory frame pinned in slot 0, the newest M - 1 in a
ring) -- the two entry points that maintain it, through the C ABI, and the engines that use it against the float64 oracle
with the same policy, against the unbounded engines while nothing has been evicted, and with graphs on against graphs off."""
import pytest
import torch

import bounded_bank_support as S
import test_gpu_engine_protocol as P
from oracle import aot_oracle as O
from oracle import weights as OW

pytestmark = pytest.mark.gpu

GUARD = 7.25        # fp32 guard value; as fp16 it is exact too


def _build(model_name, sd, gap, M):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", model_name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                       short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP, long_term_mem_max=M)
    eng.eval()
    return eng


def _oracle(model_name, sd, gap, M, objs=1):
    cfg = O.OracleConfig(model_name)
    cls = S.BoundedOracleInferEngine if objs > cfg.MODEL_MAX_OBJ_NUM else S.BoundedOracleEngine
    return cls(sd, cfg, long_term_mem_gap=gap, dtype=torch.float64, device="cuda", long_term_mem_max=M)


# ------------------------------------------------------------------------------------------------------------------
# the entry points
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kc,vc,rows,pad,slots", [
    (256, 256, 150, 0, 3),          # AOT: 8 heads x 32, a row count that is no multiple of 64
    (128, 1024, 77, 0, 4),          # DeAOT-L: keys 128, values [V | ID_V] 1024
    (128, 1024, 130, 64, 2),        # the same from a wider buffer (row stride > width): a column slice
    (256, 256, 64, 32, 5)])
@pytest.mark.parametrize("where", ["first", "mid", "last"])
def test_ring_store_equals_append_plus_pack(kc, vc, rows, pad, slots, where):
    from aot_benchmark_b200 import ops
    d = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(kc + rows)
    cap = slots * rows
    slot = {"first": 0, "mid": slots // 2, "last": slots - 1}[where]
    off = slot * rows
    k_src = (torch.randn(rows, kc + pad, device=d, generator=g) * 3)[:, :kc]
    v_src = (torch.randn(rows, vc + pad, device=d, generator=g) * 3)[:, pad:]
    assert k_src.stride(0) == kc + pad and v_src.stride(0) == vc + pad
    G = 2 * rows                     # guard rows before and after every fp32 destination, 64-half rows around the packed ones

    def dest():
        kb = torch.full((G + cap + G, kc), GUARD, device=d)
        vb = torch.full((G + cap + G, vc + 4), GUARD, device=d)          # bank rows wider than the source
        kp = torch.full((G + (kc // 32) * cap + G, 64), GUARD, dtype=torch.float16, device=d)
        vp = torch.full((G + (vc // 32) * cap + G, 64), GUARD, dtype=torch.float16, device=d)
        return kb, vb, kp, vp
    view = lambda p, c: p[G:-G].view(c // 32, cap, 64)
    # reference: the separate launches of the unbounded path
    kb0, vb0, kp0, vp0 = dest()
    ops.bank_append(k_src, kb0[G:G + cap], off)
    ops.bank_append(v_src, vb0[G:G + cap], off)
    ops.tc_pack_rows(k_src, view(kp0, kc), off)
    ops.tc_pack_rows(v_src, view(vp0, vc), off)
    # one launch, offset read from the device counter
    kb1, vb1, kp1, vp1 = dest()
    write = torch.tensor([off], dtype=torch.int32, device=d)
    ops.bank_ring_store(k_src, v_src, kb1[G:G + cap], vb1[G:G + cap], view(kp1, kc), view(vp1, vc), write)
    torch.cuda.synchronize()
    for a, b, name in ((kb0, kb1, "fp32 keys"), (vb0, vb1, "fp32 values"), (kp0, kp1, "packed keys"), (vp0, vp1, "packed values")):
        assert torch.equal(a, b), f"{name}: ring store differs from append + pack"
    assert torch.equal(kb1[G + off:G + off + rows], k_src) and torch.equal(vb1[G + off:G + off + rows, :vc], v_src)
    for t in (kb1, vb1, kp1, vp1):                                       # guards (and every other slot) untouched
        assert (t[:G] == GUARD).all() and (t[-G:] == GUARD).all()
    assert (vb1[:, vc:] == GUARD).all()
    assert int(write.item()) == off                                      # the store does not move the counter
    # null destinations are skipped: only the fp32 copies (SIMT attention), then only the packed ones
    kb2, vb2, kp2, vp2 = dest()
    ops.bank_ring_store(k_src, v_src, kb2[G:G + cap], vb2[G:G + cap], None, None, write)
    assert torch.equal(kb2, kb0) and torch.equal(vb2, vb0) and (kp2 == GUARD).all() and (vp2 == GUARD).all()
    kb3, vb3, kp3, vp3 = dest()
    ops.bank_ring_store(k_src, v_src, None, None, view(kp3, kc), view(vp3, vc), write)
    assert torch.equal(kp3, kp0) and torch.equal(vp3, vp0) and (kb3 == GUARD).all() and (vb3 == GUARD).all()


def test_ring_store_argument_checks():
    from aot_benchmark_b200 import ops
    d = torch.device("cuda")
    k, v = torch.zeros(8, 64, device=d), torch.zeros(8, 64, device=d)
    kb, vb = torch.zeros(32, 64, device=d), torch.zeros(32, 64, device=d)
    kp = torch.zeros(2, 32, 64, dtype=torch.float16, device=d)
    w = torch.zeros(1, dtype=torch.int32, device=d)
    with pytest.raises(ops.AotbError):
        ops.bank_ring_store(k, v, kb, vb[:16], None, None, w)             # two capacities
    with pytest.raises(ops.AotbError):
        ops.bank_ring_store(k, v, kb, vb, kp[:1], None, w)                # packed copy of another width
    with pytest.raises(ops.AotbError):
        ops.bank_ring_store(k, v, kb[:4], vb[:4], None, None, w)          # a frame larger than the bank
    with pytest.raises(ops.AotbError):
        ops.bank_ring_store(k, v, kb, vb, None, None, w.long())           # counter type
    with pytest.raises(ops.AotbError):
        ops.bank_ring_store(k, v, None, None, None, None, w)              # nothing to write
    with pytest.raises(ops.AotbError):
        ops.bank_ring_store(k.t().contiguous().t(), v, kb, vb, None, None, w)


def _ring_model(live, write, rows, cap, pinned):
    live = min(live + rows, cap)
    write += rows
    if write + rows > cap:
        write = pinned
    return live, write


@pytest.mark.parametrize("rows,frames", [(5, 2), (63, 3), (1620, 8)])
def test_ring_advance_full_wrap_vs_host_model(rows, frames):
    from aot_benchmark_b200 import ops
    d = torch.device("cuda")
    cap = rows * frames
    live = torch.zeros(1, dtype=torch.int32, device=d)
    write = torch.zeros(1, dtype=torch.int32, device=d)
    hl, hw = 0, 0
    for step in range(3 * frames + 2):                                    # fills the bank and wraps the ring twice
        assert 0 <= hw <= cap - rows
        ops.ring_advance(live, write, rows, cap, rows)
        hl, hw = _ring_model(hl, hw, rows, cap, rows)
        assert (int(live.item()), int(write.item())) == (hl, hw), f"step {step}"
        assert step == 0 or rows <= hw <= cap - rows
    for bad in ((0, cap, rows), (rows, rows, rows), (rows, cap + 1, rows), (rows, cap, -1)):
        with pytest.raises(ops.AotbError):
            ops.ring_advance(live, write, *bad)


# ------------------------------------------------------------------------------------------------------------------
# the engines
# ------------------------------------------------------------------------------------------------------------------
def _bank_equals_oracle(e0, oe, deaot):
    """Slot for slot: the engine's live rows against the oracle's memory, which is kept in slot order when bounded."""
    o_mem, c_mem = oe.long_term_memories, e0.long_term_memories
    assert c_mem[0][0].shape[0] == o_mem[0][0].shape[0] == e0.bank_len
    for li in range(len(o_mem)):
        for part in (0, 1, 3) if deaot else (0, 1):
            a, b = c_mem[li][part].double(), o_mem[li][part]
            assert (a - b).abs().max().item() < 1e-3 * max(1.0, b.abs().max().item()), f"layer {li}, part {part}"


@pytest.mark.parametrize("model_name,lt_impl,deaot_lt", [("r50_aotl", "tc_exact", "tc"), ("r50_deaotl", "tc_exact", "tc"),
                                                         ("aott", "simt", "tc"), ("deaott", "tc_exact", "simt")])
def test_bounded_engine_vs_bounded_oracle(monkeypatch, model_name, lt_impl, deaot_lt):
    from aot_benchmark_b200 import engine
    monkeypatch.setattr(engine, "LT_IMPL", lt_impl)
    monkeypatch.setattr(engine, "DEAOT_LT", deaot_lt)
    H, W, objs, T, M, gap = 161, 241, 6, 33, 3, 2
    sd = OW.build_state_dict(model_name, seed=8)
    frames, mask = P._clip(T, H, W, objs, seed=61)
    oe = _oracle(model_name, sd, gap, M)
    ref = P._drive(oe, frames, mask, objs, (H, W))
    eng = _build(model_name, sd, gap, M)
    lens = []

    def on_frame(t):
        e = eng.aot_engines[0]
        lens.append(e.bank_len)
        assert e.bank_cap == M * e.enc_hw and e.bank_len == min(1 + t // gap, M) * e.enc_hw
        assert int(e.tk_dev.item()) == e.bank_len
        P._packed_copies_match(e)
    run = P._drive(eng, frames, mask, objs, (H, W), forced=ref[2], on_frame=on_frame)
    e0 = eng.aot_engines[0]
    assert (T - 1) // gap - (M - 1) >= 3, "the clip must evict at least three frames"
    assert e0._tc == (model_name == "r50_aotl") and e0._gp_tc == (model_name == "r50_deaotl")
    P._check_vs_oracle(run, ref, [objs])
    _bank_equals_oracle(e0, oe, "deaot" in model_name)
    # the engine's own labels: equal to the oracle's outside its tie band
    from test_gpu_engine import _tie_band_ok
    own = [lg.argmax(1, keepdim=True) for lg in run[0]]
    assert _tie_band_ok([s[0] for s in run[1]], [s[0].float().cpu() for s in ref[1]], own, ref[2], (H, W), objs + 1,
                        align=O.OracleConfig(model_name).MODEL_ALIGN_CORNERS) == 0


@pytest.mark.parametrize("model_name", ["r50_aotl", "r50_deaotl"])
def test_bound_above_the_clip_length_is_the_unbounded_engine(model_name):
    from aot_benchmark_b200 import engine
    assert engine.USE_GRAPHS
    H, W, objs, T = 161, 241, 4, 9
    sd = OW.build_state_dict(model_name, seed=8)
    frames, mask = P._clip(T, H, W, objs, seed=62)
    free = P._drive(_build(model_name, sd, 1, None), frames, mask, objs, (H, W))
    eng = _build(model_name, sd, 1, T + 3)
    run = P._drive(eng, frames, mask, objs, (H, W))
    P._assert_bitwise(run, free, "bound never reached vs unbounded")
    for a, b in zip(run[2], free[2]):
        assert torch.equal(a, b)
    assert eng.aot_engines[0].bank_len == T * eng.aot_engines[0].enc_hw < eng.aot_engines[0].bank_cap


@pytest.mark.parametrize("model_name", ["r50_aotl", "r50_deaotl"])
def test_bounded_graphs_vs_eager_over_two_videos(monkeypatch, model_name):
    from aot_benchmark_b200 import engine
    assert engine.USE_GRAPHS
    H, W, objs, M = 161, 241, 5, 3
    sd = OW.build_state_dict(model_name, seed=8)
    clips = [P._clip(12, H, W, objs, seed=63), P._clip(10, H, W, objs, seed=64)]
    eng = _build(model_name, sd, 1, M)
    runs, slot0 = [], []
    for frames, mask in clips:
        runs.append(P._drive(eng, frames, mask, objs, (H, W)))
        e0 = eng.aot_engines[0]
        assert e0.bank_len == M * e0.enc_hw and e0.enc_hw <= int(e0.wr_dev.item()) <= (M - 1) * e0.enc_hw
        slot0.append(e0.bank_K[0][:e0.enc_hw].clone())
    assert not torch.equal(slot0[0], slot0[1])
    monkeypatch.setattr(engine, "USE_GRAPHS", False)
    eager = _build(model_name, sd, 1, M)
    for i, (frames, mask) in enumerate(clips):
        ref = P._drive(eager, frames, mask, objs, (H, W))
        P._assert_bitwise(runs[i], ref, f"video {i + 1}: graphs vs eager")
        # slot 0 is the video's own first frame: the rows a fresh engine stores for its reference frame
        assert torch.equal(slot0[i], eager.aot_engines[0].bank_K[0][:eager.aot_engines[0].enc_hw]), f"video {i + 1}: slot 0"
    eng.restart_engine()
    eng.add_reference_frame(clips[0][0][0], clips[0][1], obj_nums=[objs], frame_step=0)
    e0 = eng.aot_engines[0]
    assert (int(e0.tk_dev.item()), int(e0.wr_dev.item())) == (e0.enc_hw, e0.enc_hw)      # restart reset both counters


@pytest.mark.parametrize("model_name", ["aott", "deaott"])
def test_bounded_two_sub_engines_vs_oracle(model_name):
    H, W, objs, T, M = 129, 161, 14, 10, 3
    sd = OW.build_state_dict(model_name, seed=2)
    frames, mask = P._clip(T, H, W, objs, seed=5)
    oe = _oracle(model_name, sd, 1, M, objs)
    ref = P._drive(oe, frames, mask, objs, (H, W))
    eng = _build(model_name, sd, 1, M)
    run = P._drive(eng, frames, mask, objs, (H, W), forced=ref[2])
    assert len(eng.aot_engines) == len(oe.aot_engines) == 2
    P._check_vs_oracle(run, ref, [10, 4])
    for e, o in zip(eng.aot_engines, oe.aot_engines):
        assert e.long_term_mem_max == M and e.bank_len == M * e.enc_hw
        _bank_equals_oracle(e, o, model_name.startswith("deaot"))
