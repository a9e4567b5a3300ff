"""GPU: the engine's host-side state machine on the real kernels -- long-term bank re-allocation and an exactly full bank,
sub-engines reused across videos of different geometry and object count, the protocol paths the evaluator rarely takes
(skip_long_term_update, probability-form masks), the multi-layer MobileNetV2 models and encoder maps at tile edges.
The reference is the float64 oracle on the same device, teacher-forced with its own labels."""
import pytest
import torch
import torch.nn.functional as F

from oracle import aot_oracle as O
from oracle import weights as OW

pytestmark = pytest.mark.gpu

TOL = 1e-3          # max |dlogit| against the float64 oracle (fp32 logits)


def _build(model_name, sd, gap):
    from aot_benchmark_b200 import EngineConfig, build_engine, build_vos_model
    cfg = EngineConfig("t", model_name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    eng = build_engine(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                       short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP)
    eng.eval()
    return eng


def _oracle(model_name, sd, gap, objs=1):
    cfg = O.OracleConfig(model_name)
    if objs > cfg.MODEL_MAX_OBJ_NUM:
        return O.OracleInferEngine(sd, cfg, long_term_mem_gap=gap, dtype=torch.float64, device="cuda")
    return O.OracleEngine(sd, cfg, long_term_mem_gap=gap, dtype=torch.float64, device="cuda")


def _clip(n, h, w, objs, seed):
    frames, mask = O.synthetic_video(n, h, w, objs, seed=seed)
    return [f.cuda() for f in frames], mask.cuda()


def _drive(eng, frames, first, objs, out_size, forced=None, skip=(), as_probs=None, on_frame=None):
    """The evaluator's per-frame loop.  Returns, per propagated frame, the merged logits decode_current_logits returned,
    every sub-engine's pred_id_logits, and the label map fed back (the engine's argmax, or `forced`).  `skip`: frames whose
    update_memory skips the long-term update; `as_probs`: turns each label map into a probability-form mask."""
    subs_of = lambda: getattr(eng, "aot_engines", None) or [eng]
    eng.restart_engine()
    eng.add_reference_frame(frames[0], first if as_probs is None else as_probs(first), obj_nums=[objs], frame_step=0)
    merged, subs, labels = [], [], []
    with torch.no_grad():
        for t in range(1, len(frames)):
            eng.match_propogate_one_frame(frames[t])
            lg = eng.decode_current_logits(out_size)
            merged.append(lg.clone())
            subs.append([e.pred_id_logits.clone() for e in subs_of()])
            lab = lg.argmax(1, keepdim=True).to(lg.dtype) if forced is None else forced[t - 1].to(lg.device, lg.dtype)
            labels.append(lab.clone())
            fb = F.interpolate(lab, size=tuple(eng.input_size_2d), mode="nearest")
            eng.update_memory(fb if as_probs is None else as_probs(fb), skip_long_term_update=t in skip)
            if on_frame is not None:
                on_frame(t)
    return merged, subs, labels


def _dmax(a, b, n=None):
    a, b = a.double(), b.to(a.device).double()
    if n is not None:
        a, b = a[:, :n], b[:, :n]
    return (a - b).abs().max().item()


def _check_vs_oracle(run, ref, counts, what=""):
    """Every sub-engine's live logit channels and the merged logits of every frame within TOL of the oracle's."""
    for f, (sa, sb) in enumerate(zip(run[1], ref[1])):
        assert len(sa) == len(sb) == len(counts)
        for j, (a, b, c) in enumerate(zip(sa, sb, counts)):
            d = _dmax(a, b, c + 1)
            assert d < TOL, f"{what} frame {f + 1}, sub-engine {j}: max |dlogit| = {d:.3e}"
    for f, (a, b) in enumerate(zip(run[0], ref[0])):
        d = _dmax(a, b, 1 + sum(counts) if len(counts) == 1 else None)
        assert d < TOL, f"{what} frame {f + 1}, merged: max |dlogit| = {d:.3e}"


def _assert_bitwise(run, ref, what):
    assert len(run[0]) == len(ref[0])
    for f, (a, b) in enumerate(zip(run[0], ref[0])):
        assert torch.equal(a, b), f"{what}: merged logits of frame {f + 1} differ, max {_dmax(a, b):.3e}"
    for f, (sa, sb) in enumerate(zip(run[1], ref[1])):
        assert len(sa) == len(sb)
        for j, (a, b) in enumerate(zip(sa, sb)):
            assert torch.equal(a, b), f"{what}: sub-engine {j} logits of frame {f + 1} differ, max {_dmax(a, b):.3e}"


def _enc_side(n):
    """Side of the 16x encoder map for an input side n: four stride-2 stages (stem conv, then max-pool or strided blocks);
    ResNet's 7x7 / pad 3 stem and the 3x3 / pad 1 convs and pools all give ceil(n / 2)."""
    from aot_benchmark_b200.engine import _Encoder
    for _ in range(4):
        n = _Encoder._osz(n, 3, 2, 1)
    return n


# ------------------------------------------------------------------------------------------------------------------
# A. bank re-allocation: 2 -> 4 -> 8 frames (1 frame per step on the GEMM path), exactly full at memory frame 2
# ------------------------------------------------------------------------------------------------------------------
def _packed_copies_match(e):
    """The packed operand copies the attention kernels read hold exactly the fp32 bank's live rows, and zeros beyond."""
    from aot_benchmark_b200 import ops
    n = e.bank_len
    for li in range(len(e.bank_K)):
        pairs = []
        if e._tc:
            pairs = [(e.bank_K[li], e.bank_Kp[li], "bank_Kp"), (e.bank_V[li], e.bank_Vp[li], "bank_Vp")]
        if e._gp_tc:
            pairs = [(e.bank_K[li], e.bank_gpK[li], "bank_gpK"), (e.bank_V[li], e.bank_gpV[li], "bank_gpV")]
        for src, packed, name in pairs:
            assert packed.shape[1] == e.bank_cap
            want = torch.zeros_like(packed)
            ops.tc_pack_rows(src[:n], want, 0)
            assert torch.equal(packed, want), f"layer {li}: {name} is not the packed fp32 bank ({n} live rows)"
        if e._gemm_lt:
            kh, kl = torch.zeros_like(e.bank_Kh[li]), torch.zeros_like(e.bank_Kl[li])
            ops.split_rows(e.bank_K[li][:n], kh, kl)
            vh, vl = torch.zeros_like(e.bank_VhT[li]), torch.zeros_like(e.bank_VlT[li])
            ops.split_cols(e.bank_V[li][:n], vh, vl)
            assert kh.shape[0] == vh.shape[1] == e._capw >= e.bank_cap
            for got, want, name in ((e.bank_Kh[li], kh, "bank_Kh"), (e.bank_Kl[li], kl, "bank_Kl"),
                                    (e.bank_VhT[li], vh, "bank_VhT"), (e.bank_VlT[li], vl, "bank_VlT")):
                assert torch.equal(got, want), f"layer {li}: {name} is not the split fp32 bank ({n} live rows)"


@pytest.mark.parametrize("model_name,lt_impl,deaot_lt", [
    ("r50_aotl", "tc_exact", "tc"), ("aott", "simt", "tc"),
    ("deaott", "tc_exact", "tc"), ("deaott", "tc_exact", "gemm"), ("deaott", "tc_exact", "simt")])
def test_bank_reallocation_vs_oracle(monkeypatch, model_name, lt_impl, deaot_lt):
    from aot_benchmark_b200 import engine
    monkeypatch.setattr(engine, "LT_IMPL", lt_impl)
    monkeypatch.setattr(engine, "DEAOT_LT", deaot_lt)
    monkeypatch.setattr(engine, "BANK_INIT_FRAMES", 2)
    monkeypatch.setattr(engine, "GEMM_GROW_FRAMES", 1)
    H, W, objs, T = 161, 241, 6, 7
    sd = OW.build_state_dict(model_name, seed=8)
    frames, mask = _clip(T, H, W, objs, seed=61)
    oe = _oracle(model_name, sd, 1)
    ref = _drive(oe, frames, mask, objs, (H, W))
    gemm = model_name.startswith("deaot") and deaot_lt == "gemm"
    eng = _build(model_name, sd, 1)
    full_before = []

    def on_frame(t):
        e = eng.aot_engines[0]
        N = e.enc_hw
        cap, n = (1 if gemm else 2) * N, N                       # after the reference frame
        for _ in range(t):                                       # gap 1: one memory frame per propagated frame
            if n + N > cap:                                      # _bank_reserve's growth rule
                cap = max(cap + N, n + N) if gemm else max(2 * cap, n + N)
            n += N
        assert (e.bank_len, e.bank_cap) == (n, cap), f"frame {t}: bank {e.bank_len} / {e.bank_cap}, expected {n} / {cap}"
        _packed_copies_match(e)
        full_before.append(n == cap)
    run = _drive(eng, frames, mask, objs, (H, W), forced=ref[2], on_frame=on_frame)
    e0 = eng.aot_engines[0]
    assert e0._tc == (model_name == "r50_aotl") and e0._gp_tc == (model_name == "deaott" and deaot_lt == "tc")
    assert e0._gemm_lt == gemm
    assert any(full_before[:-1]), "no frame ran its long-term attention over an exactly full bank"
    assert e0.bank_cap > (1 if gemm else 2) * e0.enc_hw
    _check_vs_oracle(run, ref, [objs])
    # bank rows: the oracle prepends memory frames, the bank appends them
    o_mem, c_mem, N = oe.long_term_memories, e0.long_term_memories, e0.enc_hw
    nfr = T
    assert c_mem[0][0].shape[0] == o_mem[0][0].shape[0] == nfr * N
    for li in range(len(o_mem)):
        for slot in (0, 1, 3) if model_name.startswith("deaot") else (0, 1):
            a = c_mem[li][slot].double().view(nfr, N, -1)
            b = o_mem[li][slot].view(nfr, N, -1).flip(0)
            assert (a - b).abs().max().item() < 1e-3 * max(1.0, b.abs().max().item()), f"layer {li}, slot {slot}"
    # the same video again on the grown engine (capacity kept, bank_len reset) and on a fresh engine without graphs
    again = _drive(eng, frames, mask, objs, (H, W), forced=ref[2])
    assert eng.aot_engines[0].bank_cap == e0.bank_cap and eng.aot_engines[0].bank_len == T * N
    if gemm:
        # the GEMM formulation reduces over the whole capacity (zeros past the live keys): a larger capacity reorders
        # its fp32 sums, so only the first video's bank sizes reproduce it bit for bit
        d = max(_dmax(a, b) for a, b in zip(again[0], run[0]))
        assert d < 1e-5, f"second video on the grown bank vs the first: max |dlogit| = {d:.3e}"
    else:
        _assert_bitwise(again, run, "second video on the grown bank vs the first")
    monkeypatch.setattr(engine, "USE_GRAPHS", False)
    eager = _drive(_build(model_name, sd, 1), frames, mask, objs, (H, W), forced=ref[2])
    _assert_bitwise(run, eager, "graphs vs eager")


# ------------------------------------------------------------------------------------------------------------------
# B. one infer engine over videos of changing geometry and object count
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_name", ["aott", "deaott"])
def test_video_sequence_with_sub_engine_reuse(model_name):
    """restart_engine() pools the sub-engines and the next video pops them in order: in the third video the first
    video's follower owns the encoder (a fresh one) while keeping the workspace and graphs of the first video, with 10
    objects in both roles.  Every video must equal a fresh engine running it alone, bit for bit, on every sub-engine."""
    from aot_benchmark_b200 import engine
    assert engine.USE_GRAPHS and engine.USE_PDL
    sd = OW.build_state_dict(model_name, seed=6)
    A, B = (97, 129), (129, 177)
    seq = [(A, 20), (B, 3), (A, 20), (A, 3), (B, 14)]
    eng = _build(model_name, sd, 2)
    follower = None
    for i, ((h, w), objs) in enumerate(seq):
        frames, mask = _clip(5, h, w, objs, seed=70 + i)
        ref = None
        if i in (2, 4):
            ref = _drive(_oracle(model_name, sd, 2, objs), frames, mask, objs, (h, w))
        forced = None if ref is None else ref[2]
        run = _drive(eng, frames, mask, objs, (h, w), forced=forced)
        counts = [10] * (objs // 10) + ([objs % 10] if objs % 10 else [])
        assert [int(e.obj_nums[0]) for e in eng.aot_engines] == counts
        if i == 0:
            follower = eng.aot_engines[1]
        if i == 2:
            assert eng.aot_engines[0] is follower, "the pooled follower did not become the encoder owner"
        alone = _drive(_build(model_name, sd, 2), frames, mask, objs, (h, w), forced=forced)
        _assert_bitwise(run, alone, f"video {i + 1} ({h}x{w}, {objs} objects) vs a fresh engine")
        if ref is not None:
            _check_vs_oracle(run, ref, counts, f"video {i + 1}")


# ------------------------------------------------------------------------------------------------------------------
# C. skip_long_term_update and probability-form masks
# ------------------------------------------------------------------------------------------------------------------
def _one_hot(lab, nid=11):
    return F.one_hot(lab[:, 0].long(), nid).permute(0, 3, 1, 2).float().contiguous()


def _soft(seed, nid=11):
    """Label map -> a soft mask: 0.6 on the label's channel plus 0.4 spread by seeded noise over all channels."""
    g = torch.Generator().manual_seed(seed)

    def f(lab):
        noise = torch.rand((1, nid) + tuple(lab.shape[-2:]), generator=g).to(lab.device)
        return 0.6 * _one_hot(lab, nid) + 0.4 * noise / noise.sum(1, keepdim=True)
    return f


@pytest.mark.parametrize("model_name", ["aott", "deaott", "r50_aotl"])
def test_protocol_paths_vs_oracle(monkeypatch, model_name):
    H, W, objs, T = 113, 145, 4, 6
    sd = OW.build_state_dict(model_name, seed=9)
    frames, mask = _clip(T, H, W, objs, seed=81)
    # skip_long_term_update: gap 1, frames 2 and 3 keep the bank as it is
    skip = {2, 3}
    oe = _oracle(model_name, sd, 1)
    ref = _drive(oe, frames, mask, objs, (H, W), skip=skip)
    eng = _build(model_name, sd, 1)
    lens = []
    run = _drive(eng, frames, mask, objs, (H, W), forced=ref[2], skip=skip,
                 on_frame=lambda t: lens.append(eng.aot_engines[0].bank_len))
    N = eng.enc_hw
    assert lens == [N * (1 + sum(1 for s in range(1, t + 1) if s not in skip)) for t in range(1, T)]
    assert oe.long_term_memories[0][0].shape[0] == lens[-1]
    _check_vs_oracle(run, ref, [objs], "skip_long_term_update:")
    # probability-form masks [1, 11, H, W] (reference frame and memory updates): the engine's dense ID-bank conv; the
    # oracle runs its ID-bank conv on the same mask instead of a one-hot of a label map
    one_hot = O.one_hot_mask
    monkeypatch.setattr(O, "one_hot_mask", lambda m, k: m if m.dim() == 4 and m.shape[1] > 1 else one_hot(m, k))
    for name, as_probs in (("one-hot", lambda: _one_hot), ("soft", lambda: _soft(5))):
        ref = _drive(_oracle(model_name, sd, 1), frames, mask, objs, (H, W), as_probs=as_probs())
        run = _drive(eng, frames, mask, objs, (H, W), forced=ref[2], as_probs=as_probs())
        _check_vs_oracle(run, ref, [objs], f"{name} mask:")
        if name == "one-hot":
            by_label = _drive(eng, frames, mask, objs, (H, W), forced=ref[2])
            d = max(_dmax(a[0], b[0], objs + 1) for a, b in zip(run[1], by_label[1]))
            assert d < 1e-5, f"one-hot mask vs the same labels as a label map: max |dlogit| = {d:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# D. the multi-layer MobileNetV2 models
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_name", ["aots", "aotb", "aotl", "deaots", "deaotb", "deaotl"])
def test_mobilenetv2_models_vs_oracle(model_name):
    H, W, objs = 113, 145, 4
    sd = OW.build_state_dict(model_name, seed=10)
    frames, mask = _clip(5, H, W, objs, seed=91)
    ref = _drive(_oracle(model_name, sd, 2), frames, mask, objs, (H, W))
    eng = _build(model_name, sd, 2)
    run = _drive(eng, frames, mask, objs, (H, W), forced=ref[2])
    assert eng.aot_engines[0].bank_len == eng.enc_hw * 3
    _check_vs_oracle(run, ref, [objs])


# ------------------------------------------------------------------------------------------------------------------
# E. encoder maps of one pixel, one row, and N around the 64 / 128 / 256 tiles
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_name,H,W,enc", [
    ("aott", 16, 16, (1, 1)), ("aott", 16, 144, (1, 9)), ("aott", 97, 129, (7, 9)), ("aott", 113, 113, (8, 8)),
    ("aott", 65, 193, (5, 13)), ("aott", 113, 241, (8, 16)), ("aott", 33, 673, (3, 43)), ("aott", 241, 241, (16, 16)),
    ("aott", 16, 4097, (1, 257)), ("r50_aotl", 16, 16, (1, 1)), ("r50_aotl", 33, 673, (3, 43))])
def test_small_and_tile_edge_maps_vs_oracle(model_name, H, W, enc):
    assert (_enc_side(H), _enc_side(W)) == enc
    objs = 3
    sd = OW.build_state_dict(model_name, seed=12)
    frames, mask = _clip(4, H, W, objs, seed=101)
    ref = _drive(_oracle(model_name, sd, 1), frames, mask, objs, (H, W))
    eng = _build(model_name, sd, 1)
    run = _drive(eng, frames, mask, objs, (H, W), forced=ref[2])
    assert eng.enc_size_2d == enc and eng.aot_engines[0].bank_len == 4 * enc[0] * enc[1]
    _check_vs_oracle(run, ref, [objs])
