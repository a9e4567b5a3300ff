"""GPU: the usage eviction policy of the bounded long-term bank (long_term_mem_policy="usage") -- the slot-split attention
launches against the default launch and float64, the fused merge + usage counters, the selection kernel, and the engines
against the float64 usage oracle, on a clip where the policy matters, and with the default policy passed explicitly."""
import math

import pytest
import torch

import test_gpu_bounded_bank as BB
import test_gpu_engine_protocol as P
import usage_bank_support as S
from oracle import aot_oracle as O
from oracle import weights as OW
from test_cpu_usage_bank import behaviour_clip

pytestmark = pytest.mark.gpu

MASS_TOL = {True: 1e-5, False: 2e-3}        # |U - float64 mass| per frame: exact (fp32) mode, fast (fp16) mode


def _build(model_name, sd, gap, M, policy, precision=None):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", model_name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    kw = {} if policy is None else {"long_term_mem_policy": policy}
    if precision is not None:
        kw["precision"] = precision
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                       short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP, long_term_mem_max=M, **kw)
    eng.eval()
    return eng


# ------------------------------------------------------------------------------------------------------------------
# slot-split attention
# ------------------------------------------------------------------------------------------------------------------
def _bank(kind, N, M, HW, seed):
    """Random Q / K / V for the AOT head shape (8 x 32) or DeAOT's (1 x 128 / 1024), packed; -> (fp32 tensors, packed)."""
    from aot_benchmark_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    dq, dv, H = (256, 256, 8) if kind == "aot" else (128, 1024, 1)
    Q = torch.randn(N, dq, device="cuda", generator=g) * 2
    K = torch.randn(M * HW, dq, device="cuda", generator=g)
    V = torch.randn(M * HW, dv, device="cuda", generator=g)
    hz = lambda c, r: torch.zeros(c // 32, r, 64, dtype=torch.float16, device="cuda")
    Qp = ops.tc_pack_rows(Q, hz(dq, ((N + 255) // 256) * 256), 0, div=math.sqrt(dq // H))
    Kp, Vp = ops.tc_pack_rows(K, hz(dq, M * HW), 0), ops.tc_pack_rows(V, hz(dv, M * HW), 0)
    return (Q, K, V, H, dq // H, dv), (Qp, Kp, Vp)


def _slot_launch(kind, packed, N, live, M, HW, exact):
    from aot_benchmark_b200 import ops
    Qp, Kp, Vp = packed
    dv = Vp.shape[0] * 32
    H = 8 if kind == "aot" else 1
    part = (torch.full((M, N, dv), float("nan"), device="cuda"), torch.full((M, H, N), float("nan"), device="cuda"),
            torch.full((M, H, N), float("nan"), device="cuda"))
    tk = torch.tensor([live], dtype=torch.int32, device="cuda")
    fn = ops.lt_attention_tc_slots if kind == "aot" else ops.gp_attention_tc_slots
    fn(Qp, Kp, Vp, N, tk, M, HW, part, exact=exact)
    return part, tk


def _default_launch(kind, packed, N, live, exact):
    from aot_benchmark_b200 import ops
    Qp, Kp, Vp = packed
    O = torch.empty(N, Vp.shape[0] * 32, device="cuda")
    fn = ops.lt_attention_tc if kind == "aot" else ops.gp_attention_tc
    fn(Qp, Kp, Vp, N, live, O=O, splits=1, exact=exact)
    return O


def _mass64(packed, N, H, live, M, HW, exact):
    """float64 per-(head, query) slot masses over the operands the kernel multiplies (hi + lo exact, hi fast) -> [M, H, N]."""
    Qp, Kp, _ = packed
    un = lambda P_, rows: (P_[:, :rows, :32].double() + (P_[:, :rows, 32:].double() if exact else 0))
    q, k = un(Qp, N), un(Kp, live)                                            # [C / 32, rows, 32]
    C = q.shape[0]
    q = q.permute(1, 0, 2).reshape(N, H, -1).permute(1, 0, 2)
    k = k.permute(1, 0, 2).reshape(live, H, -1).permute(1, 2, 0)
    p = torch.softmax(q @ k, -1)
    out = torch.zeros(M, H, N, dtype=torch.float64, device="cuda")
    for s in range(live // HW):
        out[s] = p[:, :, s * HW:(s + 1) * HW].sum(-1)
    return out


def _masses(part):
    Op, Mp, Lp = part
    m = Mp.max(0).values
    w = torch.where(torch.isfinite(Mp), torch.exp((Mp - m).double()), torch.zeros_like(Mp, dtype=torch.float64))
    return w * Lp.double() / (w * Lp.double()).sum(0)


@pytest.mark.parametrize("kind", ["aot", "deaot"])
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
@pytest.mark.parametrize("M", [2, 3, 8])
@pytest.mark.parametrize("HW", [128, 77, 1674])
def test_slot_split_attention_vs_default_launch(kind, exact, M, HW):
    """Every split is one slot, starting at a key that is no multiple of the 64-key tile when HW is not: the merged slots
    equal the default launch (DESIGN §3.1 bound: fp32 reordering; fast mode: P rounded against another running max), each
    slot's mass equals float64's, and slots beyond the live keys (bank not yet full) are empty."""
    from aot_benchmark_b200 import ops
    N = 300
    (Q, K, V, H, _, dv), packed = _bank(kind, N, M, HW, seed=M * 7 + HW)
    for fill in sorted({1, M - 1, M}):
        live = fill * HW
        part, tk = _slot_launch(kind, packed, N, live, M, HW, exact)
        assert torch.isinf(part[1][fill:]).all() and (part[1][fill:] < 0).all() and (part[2][fill:] == 0).all()
        assert torch.isfinite(part[1][:fill]).all() and (part[2][:fill] > 0).all()
        O = torch.empty(N, dv, device="cuda")
        ops.attn_merge(*part, O, H, dv // H)
        ref = _default_launch(kind, packed, N, live, exact)
        d = (O - ref).abs().max().item() / V.abs().max().item()
        assert d < (2e-5 if exact else 2e-3), f"fill {fill}: merged slots vs default launch {d:.3e}"
        dm = (_masses(part) - _mass64(packed, N, H, live, M, HW, exact)).abs().max().item()
        assert dm < 1e-5, f"fill {fill}: slot masses vs float64 over the multiplied operands {dm:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# fused merge + usage
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,exact", [("aot", True), ("aot", False), ("deaot", True), ("deaot", False)])
def test_fused_merge_usage(kind, exact):
    """O bitwise equal to aotb_attn_merge_f32 on the same partials; U within MASS_TOL of the float64 mass of the fp32
    attention; A ticks the live slots; U bitwise reproducible, and graph replay bitwise equal to eager."""
    from aot_benchmark_b200 import ops
    N, M, HW, fill, layers = 1674, 8, 1674, 6, 3
    (Q, K, V, H, d, dv), packed = _bank(kind, N, M, HW, seed=11)
    part, tk = _slot_launch(kind, packed, N, fill * HW, M, HW, exact)
    O0 = torch.empty(N, dv, device="cuda")
    ops.attn_merge(*part, O0, H, dv // H)
    ws = ops.attn_merge_usage_workspace(M, "cuda")

    def run():
        U, A = torch.zeros(M, device="cuda"), torch.zeros(M, dtype=torch.int32, device="cuda")
        O = torch.empty(N, dv, device="cuda")
        for li in range(layers):                                   # one frame: `layers` launches, the first ticks A
            ops.attn_merge_usage(*part, O, H, dv // H, U, A if li == 0 else None, tk, HW, layers, ws)
        return O, U, A
    O1, U1, A1 = run()
    O2, U2, A2 = run()
    torch.cuda.synchronize()
    assert torch.equal(O1, O0), "fused merge O differs from aotb_attn_merge_f32"
    assert torch.equal(U1, U2) and torch.equal(A1, A2), "usage not bitwise reproducible"
    assert A1.tolist() == [1] * fill + [0] * (M - fill)
    assert (U1[fill:] == 0).all() and abs(U1.sum().item() - 1.0) < 1e-5
    q = (Q.double() / math.sqrt(d)).view(N, H, d).permute(1, 0, 2)
    k = K[:fill * HW].double().view(fill * HW, H, d).permute(1, 2, 0)
    p = torch.softmax(q @ k, -1)
    want = torch.stack([p[:, :, s * HW:(s + 1) * HW].sum(-1).mean() for s in range(fill)])
    err = (U1[:fill].double() - want).abs().max().item()
    print(f"fused merge usage, {kind} {'exact' if exact else 'fast'}: max |U - float64 mass| = {err:.3e}")
    assert err < MASS_TOL[exact]
    # graph capture of the same frame: replays from a zero launch counter give the eager bits
    U, A = torch.zeros(M, device="cuda"), torch.zeros(M, dtype=torch.int32, device="cuda")
    O = torch.empty(N, dv, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for li in range(layers):
                ops.attn_merge_usage(*part, O, H, dv // H, U, A if li == 0 else None, tk, HW, layers, ws)
    torch.cuda.current_stream().wait_stream(s)
    for rep in range(2):
        U.zero_()
        A.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(O, O1) and torch.equal(U, U1) and torch.equal(A, A1), f"graph replay {rep}"


def test_fused_merge_argument_checks():
    from aot_benchmark_b200 import ops
    Op, Mp, Lp = torch.zeros(33, 64, 32, device="cuda"), torch.zeros(33, 1, 64, device="cuda"), torch.ones(33, 1, 64, device="cuda")
    tk = torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(ops.AotbError):
        ops.attn_merge_usage(Op, Mp, Lp, torch.zeros(64, 32, device="cuda"), 1, 32, torch.zeros(33, device="cuda"), None, tk, 64,
                             1, ops.attn_merge_usage_workspace(33, "cuda"))
    with pytest.raises(ops.AotbError):
        ops.attn_merge_usage(Op[:4], Mp[:4], Lp[:4], torch.zeros(64, 32, device="cuda"), 1, 32, torch.zeros(4, device="cuda"),
                             None, tk, 64, 0, ops.attn_merge_usage_workspace(4, "cuda"))


# ------------------------------------------------------------------------------------------------------------------
# selection
# ------------------------------------------------------------------------------------------------------------------
def _select_gpu(U, A, live, rows=1674, M=4):
    from aot_benchmark_b200 import ops
    lv = torch.tensor([live], dtype=torch.int32, device="cuda")
    w = torch.tensor([-7], dtype=torch.int32, device="cuda")
    U = torch.tensor(U, dtype=torch.float32, device="cuda")
    A = torch.tensor(A, dtype=torch.int32, device="cuda")
    ops.ring_select_usage(lv, w, U, A, rows, rows * M, rows)
    return int(w.item()), U.cpu(), A.cpu()


def test_selection_kernel():
    rows = 1674
    for fill in range(4):                                                    # not full: the next free slot
        w, U, A = _select_gpu([0.9, 0.1, 0.0, 0.0], [3, 2, 0, 0], fill * rows)
        assert w == fill * rows and U[fill] == 0 and A[fill] == 0
    w, U, A = _select_gpu([0.0, 0.6, 0.3, 0.5], [9, 3, 1, 5], 4 * rows)       # argmin of U / A; slot 0 never
    assert w == 3 * rows and U[3] == 0 and A.tolist() == [9, 3, 1, 0] and U[1] > 0 and U[2] > 0
    assert _select_gpu([0.5, 0.0, 0.9, 0.9], [1, 0, 1, 1], 4 * rows)[0] == 2 * rows     # A = 0 is +inf
    assert _select_gpu([0.0, 0.4, 0.2, 0.2], [1, 2, 1, 1], 4 * rows)[0] == rows          # ties: the lowest slot
    assert _select_gpu([0.0, 0.0, 0.0, 0.0], [1, 0, 0, 0], 4 * rows)[0] == rows
    for live in (10 ** 8, -rows):                                            # a corrupt live count: still a slot of the bank
        w = _select_gpu([0.0, 0.4, 0.1, 0.2], [1, 2, 2, 2], live)[0]
        assert 0 <= w <= 3 * rows and w % rows == 0
    g = torch.Generator().manual_seed(3)
    for _ in range(50):                                                      # the emulated contract, bit for bit
        M = int(torch.randint(2, 33, (1,), generator=g))
        U = (torch.rand(M, generator=g) * 3).tolist()
        A = torch.randint(0, 4, (M,), generator=g).tolist()
        w, Ug, Ag = _select_gpu(U, A, M * 7, rows=7, M=M)
        we, Ue, Ae = torch.zeros(1, dtype=torch.int32), torch.tensor(U), torch.tensor(A, dtype=torch.int32)
        S.ring_select_usage(torch.tensor([M * 7], dtype=torch.int32), we, Ue, Ae, 7, 7 * M, 7)
        assert w == int(we) and torch.equal(Ug, Ue) and torch.equal(Ag, Ae)
    from aot_benchmark_b200 import ops
    z = lambda dt: torch.zeros(4, dtype=dt, device="cuda")
    c = lambda: torch.zeros(1, dtype=torch.int32, device="cuda")
    for rows, cap, pinned in ((5, 20, 3), (5, 20, 20)):                    # the entry point's geometry checks
        with pytest.raises(ops.AotbError):
            ops.ring_select_usage(c(), c(), z(torch.float32), z(torch.int32), rows, cap, pinned)


# ------------------------------------------------------------------------------------------------------------------
# the engines
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_name,precision", [("r50_aotl", "fp32"), ("r50_deaotl", "fp32"), ("r50_aotl", "fp16")])
def test_usage_engine_vs_usage_oracle(model_name, precision):
    """Gap 1, M = 3, 12 frames (nine evictions), the float64 oracle in lockstep: it overwrites the slot the engine chose,
    which must be its own argmin unless its two best scores are within 1e-4 relative.  fp32: logits and bank rows within the
    bounded-bank tolerances, U within 1e-5 per frame; fp16: U within 2e-3 per frame."""
    from aot_benchmark_b200 import engine
    assert engine.USE_GRAPHS
    H, W, objs, T, M = 161, 241, 5, 12, 3
    sd = OW.build_state_dict(model_name, seed=8)
    frames, mask = P._clip(T, H, W, objs, seed=71)
    oe = S.oracle(model_name, sd, M, objs, dtype=torch.float64, device="cuda")
    eng = _build(model_name, sd, 1, M, "usage", precision)
    c_lo, o_lo, _ = S.run_lockstep(eng, oe, frames, mask, objs, (H, W))
    e0 = eng.aot_engines[0]
    U, A = e0.long_term_memory_usage
    assert A.tolist() == oe.A
    du = (U.double().cpu() - torch.tensor(oe.U)).abs().max().item()
    frames_per_slot = max(oe.A)
    print(f"{model_name} {precision}: max |U - oracle U| = {du:.3e} over up to {frames_per_slot} frames; "
          f"evictions (own, gap, taken) = {oe.evictions}")
    assert du < (1e-5 if precision == "fp32" else 2e-3) * frames_per_slot
    assert len(oe.evictions) == T - M
    for own, gap, took in oe.evictions:
        assert own == took or gap <= 1e-4, oe.evictions
    if precision == "fp32":
        for f, (a, b) in enumerate(zip(c_lo, o_lo)):
            d = P._dmax(a[0], b[0], objs + 1)
            assert d < P.TOL, f"frame {f + 1}: max |dlogit| = {d:.3e}"
        BB._bank_equals_oracle(e0, oe, "deaot" in model_name)
        P._packed_copies_match(e0)


@pytest.mark.parametrize("model_name", ["r50_aotl", "r50_deaotl"])
def test_usage_keeps_the_frame_the_clip_returns_to(model_name):
    """f0, X, Y (noise), X' (X again): at X''s store the full bank evicts Y under usage and X under FIFO (the margin is
    checked on the CPU oracle by test_cpu_usage_bank)."""
    H, W = 97, 129
    frames, mask = behaviour_clip(H, W)
    frames, mask = [f.cuda() for f in frames[:4]], mask.cuda()
    sd = OW.build_state_dict(model_name, seed=3)
    kept = {}
    for policy in ("usage", "fifo"):
        eng = _build(model_name, sd, 1, 3, policy)
        x_rows = []

        def on_frame(t):
            e = eng.aot_engines[0]
            if t == 1:
                x_rows.append(e.bank_K[0][e.enc_hw:2 * e.enc_hw].clone())
        P._drive(eng, frames, mask, 2, (H, W), on_frame=on_frame)
        e = eng.aot_engines[0]
        N = e.enc_hw
        kept[policy] = any(torch.equal(e.bank_K[0][s * N:(s + 1) * N], x_rows[0]) for s in range(3))
        if policy == "usage":
            assert torch.equal(e.bank_K[0][N:2 * N], x_rows[0])
    assert kept == {"usage": True, "fifo": False}


@pytest.mark.parametrize("model_name", ["r50_aotl", "r50_deaotl"])
def test_fifo_passed_explicitly_is_the_default_engine(model_name):
    H, W, objs, T, M = 161, 241, 4, 8, 3
    sd = OW.build_state_dict(model_name, seed=8)
    frames, mask = P._clip(T, H, W, objs, seed=72)
    a = P._drive(_build(model_name, sd, 1, M, None), frames, mask, objs, (H, W))
    eng = _build(model_name, sd, 1, M, "fifo")
    b = P._drive(eng, frames, mask, objs, (H, W))
    P._assert_bitwise(b, a, "explicit fifo vs default")
    assert eng.aot_engines[0].long_term_memory_usage is None


@pytest.mark.parametrize("model_name", ["r50_aotl", "r50_deaotl"])
def test_usage_graphs_vs_eager(monkeypatch, model_name):
    """Usage mode with captured graphs over two videos equals it eagerly, logits and counters bit for bit."""
    from aot_benchmark_b200 import engine
    H, W, objs, M = 161, 241, 3, 3
    sd = OW.build_state_dict(model_name, seed=8)
    clips = [P._clip(9, H, W, objs, seed=73), P._clip(8, H, W, objs, seed=74)]
    eng = _build(model_name, sd, 1, M, "usage")
    runs = []
    for frames, mask in clips:
        runs.append((P._drive(eng, frames, mask, objs, (H, W)), eng.aot_engines[0].long_term_memory_usage))
    monkeypatch.setattr(engine, "USE_GRAPHS", False)
    eager = _build(model_name, sd, 1, M, "usage")
    for i, (frames, mask) in enumerate(clips):
        ref = P._drive(eager, frames, mask, objs, (H, W))
        P._assert_bitwise(runs[i][0], ref, f"video {i + 1}: usage graphs vs eager")
        U, A = eager.aot_engines[0].long_term_memory_usage
        assert torch.equal(runs[i][1][0], U) and torch.equal(runs[i][1][1], A)
