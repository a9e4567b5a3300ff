"""TEST INFRASTRUCTURE ONLY for the usage eviction policy of the bounded long-term bank (long_term_mem_policy="usage"): the
oracle with the same policy, a lockstep driver, and torch-CPU emulations of the contracts of aotb_lt_attn_tc_slots_f16x2,
aotb_gp_attn_tc_slots_f16x2, aotb_attn_merge_usage_f32 and aotb_ring_select_usage (include/aotb200.h) that extend
tests/emu_ops.py and tests/bounded_bank_support.py.  Nothing under aot_benchmark_b200/ imports this module."""
import math

import torch
import torch.nn.functional as F

import bounded_bank_support as B
import emu_ops
from oracle import aot_oracle as O


# ------------------------------------------------------------------------------------------------------------------
# oracle: masses in float64 from the oracle's own long-term attention, the policy applied to them
# ------------------------------------------------------------------------------------------------------------------
def slot_masses(Q, K, heads, slots, rows):
    """Mean over (head, query) of the softmax((Q / sqrt(d)) K^T) mass on each slot's keys (slot s = key rows
    [s rows, (s + 1) rows)), in float64.  Q [N, 1, heads * d], K [Tk, 1, heads * d]."""
    N, Tk = Q.shape[0], K.shape[0]
    d = Q.shape[-1] // heads
    q = (Q.double().reshape(N, heads, d) / math.sqrt(d)).permute(1, 0, 2)
    k = K.double().reshape(Tk, heads, d).permute(1, 2, 0)
    p = torch.softmax(q @ k, dim=-1)                                      # [heads, N, Tk]
    u = torch.zeros(slots, dtype=torch.float64, device=Q.device)
    for s in range(Tk // rows):
        u[s] = p[:, :, s * rows:(s + 1) * rows].sum(-1).mean()
    return u


def scores(U, A):
    return [U[s] / A[s] if A[s] > 0 else math.inf for s in range(len(U))]


class UsageOracleEngine(B.BoundedOracleEngine):
    """BoundedOracleEngine whose full bank overwrites the unpinned slot with the lowest U / A.  Not in the reference.
    `follow` (optional) is called when the bank is full and returns the slot to overwrite instead of the oracle's own
    choice, so the oracle can stay in lockstep with an engine whose choice differs at a near tie; every eviction is logged
    in `evictions` as (own choice, relative gap between the two best scores, slot overwritten)."""

    def __init__(self, weights, cfg, *args, long_term_mem_max, **kwargs):
        kwargs["keep_taps"] = True
        super().__init__(weights, cfg, *args, long_term_mem_max=long_term_mem_max, **kwargs)
        self.follow = None

    def restart_engine(self):
        super().restart_engine()
        M = self.long_term_mem_max
        self.U = [0.0] * M
        self.A = [0] * M
        self.frame_masses = []
        self.evictions = []

    def match_propogate_one_frame(self, img):
        super().match_propogate_one_frame(img)
        M, hw = self.long_term_mem_max, self.enc_hw
        L = self.cfg.MODEL_LSTT_NUM
        heads = 1 if self.deaot else self.cfg.MODEL_ATT_HEADS
        u = sum(slot_masses(self.taps[f"LSTT.layers.{li}.lt_in"][0], self.taps[f"LSTT.layers.{li}.lt_in"][1], heads, M, hw)
                for li in range(L)) / L
        live = self.long_term_memories[0][0].shape[0] // hw
        for s in range(live):
            self.U[s] += float(u[s])
            self.A[s] += 1
        self.frame_masses.append(u.cpu())

    def update_long_term_memory(self, new_mems):
        M, hw = self.long_term_mem_max, self.enc_hw
        if self.long_term_memories[0][0].shape[0] >= M * hw:
            sc = scores(self.U, self.A)[1:]
            own = 1 + min(range(M - 1), key=lambda i: (sc[i], i))
            best = sorted(sc)[:2]
            gap = math.inf if math.isinf(best[1]) else (best[1] - best[0]) / max(abs(best[1]), 1e-300)
            s = own if self.follow is None else self.follow()
            self.evictions.append((own, gap, s))
            self._ring_slot = s
            self.U[s], self.A[s] = 0.0, 0
        else:
            s = self.long_term_memories[0][0].shape[0] // hw
            self.U[s], self.A[s] = 0.0, 0
        super().update_long_term_memory(new_mems)


class UsageOracleInferEngine(O.OracleInferEngine):
    """aot_oracle.OracleInferEngine whose sub-engines are UsageOracleEngines with the same bound."""

    def __init__(self, weights, cfg, *args, long_term_mem_max, **kwargs):
        super().__init__(weights, cfg, *args, **kwargs)
        self.long_term_mem_max = long_term_mem_max

    def add_reference_frame(self, img, mask, obj_nums, frame_step=-1):
        n = obj_nums[0] if isinstance(obj_nums, list) else obj_nums
        need = max(math.ceil(n / self.max_aot_obj_num), 1)
        while need > len(self.aot_engines):
            self.aot_engines.append(UsageOracleEngine(self.weights, self.cfg, self.long_term_mem_gap, self.short_term_mem_skip,
                                                      self.dtype, device=self.device, long_term_mem_max=self.long_term_mem_max))
        return super().add_reference_frame(img, mask, obj_nums, frame_step)


def oracle(model_name, sd, M, objs, dtype=torch.float32, device="cpu", gap=1):
    cfg = O.OracleConfig(model_name)
    cls = UsageOracleInferEngine if objs > cfg.MODEL_MAX_OBJ_NUM else UsageOracleEngine
    return cls(sd, cfg, long_term_mem_gap=gap, dtype=dtype, device=device, long_term_mem_max=M)


def chosen_slot(e):
    """The slot an engine's last store went to, with gap 1 and a full bank: the only unpinned slot whose age A is 0 (every
    other live slot has been read by at least the frame just propagated)."""
    A = e.long_term_memory_usage[1].cpu()
    z = [s for s in range(1, len(A)) if int(A[s]) == 0]
    assert len(z) == 1, f"expected exactly one freshly stored slot, ages {A.tolist()}"
    return z[0]


def run_lockstep(eng, oe, frames, mask, objs, out_size, on_frame=None):
    """The evaluator's loop over the engine and the oracle side by side, gap 1.  The oracle's labels are fed back to both,
    and each oracle sub-engine overwrites the slot its engine counterpart chose.  Returns (engine pred_id_logits per frame
    and sub-engine, oracle's, labels)."""
    subs = lambda x: getattr(x, "aot_engines", None) or [x]
    eng.restart_engine()
    oe.restart_engine()
    oe.add_reference_frame(frames[0].to(oe_device(oe)), mask.to(oe_device(oe)), obj_nums=[objs], frame_step=0)
    eng.add_reference_frame(frames[0], mask, obj_nums=[objs], frame_step=0)
    for j, o in enumerate(subs(oe)):
        o.follow = (lambda j=j: chosen_slot(subs(eng)[j]))
    c_lo, o_lo, labels = [], [], []
    with torch.no_grad():
        for t in range(1, len(frames)):
            oe.match_propogate_one_frame(frames[t].to(oe_device(oe)))
            olg = oe.decode_current_logits(out_size)
            eng.match_propogate_one_frame(frames[t])
            eng.decode_current_logits(out_size)
            lab = olg.argmax(1, keepdim=True).to(torch.float32)
            c_lo.append([e.pred_id_logits.clone() for e in subs(eng)])
            o_lo.append([o.pred_id_logits.clone() for o in subs(oe)])
            labels.append(lab)
            fb = F.interpolate(lab, size=tuple(eng.input_size_2d), mode="nearest")
            eng.update_memory(fb.to(mask.device))
            oe.update_memory(fb.to(oe_device(oe), oe.dtype if hasattr(oe, "dtype") else torch.float32))
            if on_frame is not None:
                on_frame(t)
    return c_lo, o_lo, labels


def oe_device(oe):
    return torch.device(getattr(oe, "device", "cpu"))


# ------------------------------------------------------------------------------------------------------------------
# contract emulations
# ------------------------------------------------------------------------------------------------------------------
def _err(msg):
    from aot_benchmark_b200._lib import AotbError
    raise AotbError(msg)


def _slot_partials(q, k, v, tk, splits, split_rows):
    """Split-KV partials with the kernel's split arithmetic (attn_tc.cuh): units of split_rows keys, `per` units a split.
    q [H, N, d], k [H, tk, d], v [H, tk, dv] -> [(O [H, N, dv], m [H, N], l [H, N])] per split."""
    units = (tk + split_rows - 1) // split_rows
    per = (units + splits - 1) // splits
    Hh, N, dv = q.shape[0], q.shape[1], v.shape[2]
    parts = []
    for z in range(splits):
        k0, k1 = min(z * per * split_rows, tk), min((z + 1) * per * split_rows, tk)
        if k1 > k0:
            s = q @ k[:, k0:k1].transpose(1, 2)
            m = s.max(-1).values
            p = torch.exp(s - m.unsqueeze(-1))
            parts.append((p @ v[:, k0:k1], m, p.sum(-1)))
        else:
            parts.append((torch.zeros(Hh, N, dv), torch.full((Hh, N), float("-inf")), torch.zeros(Hh, N)))
    return parts


def _slot_args(name, N, Tk_dev, slots, slot_rows, cap):
    if not (N > 0 and slots >= 2 and slot_rows > 0):
        _err(f"{name}: bad args")
    tk = int(Tk_dev.item())
    if tk > cap:
        _err(f"{name}: live keys beyond the bank")
    return tk


def lt_attention_tc_slots(Qp, Kp, Vp, N, Tk_dev, slots, slot_rows, part, exact=True, stream=None):
    """Contract of aotb_lt_attn_tc_slots_f16x2."""
    tk = _slot_args("aotb_lt_attn_tc_slots_f16x2", N, Tk_dev, slots, slot_rows, Kp.shape[1])
    unpack = lambda P, rows, lo: P[:, :rows, :32].float() + (P[:, :rows, 32:].float() if lo else 0)
    q, k, v = unpack(Qp, N, exact), unpack(Kp, tk, exact), unpack(Vp, tk, True)
    Op, Mp, Lp = part
    for z, (o, m, l) in enumerate(_slot_partials(q, k, v, tk, slots, slot_rows)):
        Op[z].copy_(o.permute(1, 0, 2).reshape(N, -1))
        Mp[z].copy_(m)
        Lp[z].copy_(l)


def gp_attention_tc_slots(Qp, Kp, Vp, N, Tk_dev, slots, slot_rows, part, exact=True, stream=None):
    """Contract of aotb_gp_attn_tc_slots_f16x2: one head, 32-channel chunks."""
    tk = _slot_args("aotb_gp_attn_tc_slots_f16x2", N, Tk_dev, slots, slot_rows, Kp.shape[1])
    unpack = lambda P, rows, lo: (P[:, :rows, :32].float() + (P[:, :rows, 32:].float() if lo else 0)).permute(1, 0, 2) \
        .reshape(rows, -1).unsqueeze(0)
    q, k, v = unpack(Qp, N, exact), unpack(Kp, tk, exact), unpack(Vp, tk, True)
    Op, Mp, Lp = part
    for z, (o, m, l) in enumerate(_slot_partials(q, k, v, tk, slots, slot_rows)):
        Op[z].copy_(o[0])
        Mp[z].copy_(m)
        Lp[z].copy_(l)


def attn_merge_usage_workspace(R, device):
    return torch.zeros(1, dtype=torch.float64, device=device)


def attn_merge_usage(Opart, Mpart, Lpart, O, H, d_v, U, A, live_dev, rows, layers, workspace, stream=None):
    """Contract of aotb_attn_merge_usage_f32: O as attn_merge; U += the slot masses summed over (query, head) / (layers H N);
    A ticks every live slot."""
    R, N = Opart.shape[0], Opart.shape[1]
    if R > 32 or layers <= 0 or (A is not None and rows <= 0) or U.numel() != R:
        _err("aotb_attn_merge_usage_f32: bad args")
    emu_ops.attn_merge(Opart, Mpart, Lpart, O, H, d_v)
    m = Mpart.max(dim=0).values
    w = torch.where(torch.isfinite(Mpart), torch.exp(Mpart - m.unsqueeze(0)), torch.zeros_like(Mpart))
    den = (w * Lpart).sum(0)
    mass = (w * Lpart / den.unsqueeze(0)).double().sum(dim=(1, 2))             # [R]
    U += (mass / (layers * H * N)).to(U.dtype)
    if A is not None:
        A[:min(int(live_dev.item()) // rows, R)] += 1
    return O


def ring_select_usage(live_dev, write_dev, U, A, rows, cap_rows, pinned_rows, stream=None):
    """Contract of aotb_ring_select_usage, with the entry point's argument checks."""
    rows, cap_rows, pinned_rows = int(rows), int(cap_rows), int(pinned_rows)
    if not (rows > 0 and pinned_rows >= 0 and pinned_rows % rows == 0 and cap_rows % rows == 0 and
            pinned_rows + rows <= cap_rows) or U.numel() * rows != cap_rows or A.numel() * rows != cap_rows:
        _err(f"aotb_ring_select_usage: bad geometry (rows {rows}, cap_rows {cap_rows}, pinned_rows {pinned_rows})")
    slots, used = cap_rows // rows, max(int(live_dev.item()), 0) // rows
    s = used
    if used >= slots:
        sc = [float(U[c]) / int(A[c]) if int(A[c]) > 0 else math.inf for c in range(slots)]
        s = min(range(pinned_rows // rows, slots), key=lambda c: (sc[c], c))
    write_dev.fill_(s * rows)
    U[s] = 0
    A[s] = 0


EMULATED = ("lt_attention_tc_slots", "gp_attention_tc_slots", "attn_merge_usage_workspace", "attn_merge_usage",
            "ring_select_usage")


def install_engine(monkeypatch, wrap=None):
    """bounded_bank_support.install_engine plus the entry points of the usage policy; `wrap(name, fn)` decorates them."""
    from aot_benchmark_b200 import ops
    B.install_engine(monkeypatch, wrap)
    for name in EMULATED:
        fn = globals()[name]
        monkeypatch.setattr(ops, name, fn if wrap is None else wrap(name, fn))
