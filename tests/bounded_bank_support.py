"""TEST INFRASTRUCTURE ONLY for the bounded long-term bank (long_term_mem_max = M): the oracle with the same policy, and
torch-CPU emulations of the contracts of aotb_bank_ring_store / aotb_ring_advance (include/aotb200.h) that extend
tests/emu_ops.py, so the host tests can drive the bounded product engines without a GPU.  Nothing under aot_benchmark_b200/
imports this module."""
import math

import torch

import emu_ops
from oracle import aot_oracle as O


# ------------------------------------------------------------------------------------------------------------------
# oracle: the first stored frame pinned in slot 0, the other M - 1 slots a FIFO ring
# ------------------------------------------------------------------------------------------------------------------
class BoundedOracleEngine(O.OracleEngine):
    """aot_oracle.OracleEngine with at most `long_term_mem_max` memory frames.  Not in the reference.  The memory is kept in
    SLOT order (slot s = rows [s hw, (s + 1) hw)), not prepended, so it compares row for row with the product engines' bank."""

    def __init__(self, weights, cfg, *args, long_term_mem_max, **kwargs):
        if long_term_mem_max < 2:
            raise ValueError(f"long_term_mem_max must be >= 2, got {long_term_mem_max}")
        self.long_term_mem_max = long_term_mem_max
        super().__init__(weights, cfg, *args, **kwargs)

    def restart_engine(self):
        super().restart_engine()
        self._ring_slot = 1          # slot the next frame overwrites once all slots are taken

    def update_long_term_memory(self, new_mems):
        M, hw = self.long_term_mem_max, self.enc_hw
        full = next(t for t in self.long_term_memories[0] if t is not None).shape[0] >= M * hw
        s = self._ring_slot
        upd = []
        for new_m, last_m in zip(new_mems, self.long_term_memories):
            row = []
            for a, b in zip(new_m, last_m):
                if a is None or b is None:
                    row.append(None)
                elif full:                   # overwrite the oldest unpinned frame in place
                    row.append(torch.cat([b[:s * hw], a, b[(s + 1) * hw:]], dim=0))
                else:                        # free slots are taken in order
                    row.append(torch.cat([b, a], dim=0))
            upd.append(row)
        if full:
            self._ring_slot = s + 1 if s + 1 < M else 1
        self.long_term_memories = upd


class BoundedOracleInferEngine(O.OracleInferEngine):
    """aot_oracle.OracleInferEngine whose sub-engines are BoundedOracleEngines with the same bound."""

    def __init__(self, weights, cfg, *args, long_term_mem_max, **kwargs):
        super().__init__(weights, cfg, *args, **kwargs)
        self.long_term_mem_max = long_term_mem_max

    def add_reference_frame(self, img, mask, obj_nums, frame_step=-1):
        n = obj_nums[0] if isinstance(obj_nums, list) else obj_nums
        need = max(math.ceil(n / self.max_aot_obj_num), 1)
        while need > len(self.aot_engines):          # the base class then finds its sub-engines in place
            self.aot_engines.append(BoundedOracleEngine(self.weights, self.cfg, self.long_term_mem_gap, self.short_term_mem_skip,
                                                        self.dtype, device=self.device,
                                                        long_term_mem_max=self.long_term_mem_max))
        return super().add_reference_frame(img, mask, obj_nums, frame_step)


# ------------------------------------------------------------------------------------------------------------------
# contract emulations
# ------------------------------------------------------------------------------------------------------------------
def bank_ring_store(k_src, v_src, k_bank, v_bank, k_packed, v_packed, write_dev, stream=None):
    """Contract of aotb_bank_ring_store: every copy that is given receives the rows at *write_dev; a store that does not
    fit writes nothing."""
    off, rows = int(write_dev.item()), k_src.shape[0]
    for src, bank, packed in ((k_src, k_bank, k_packed), (v_src, v_bank, v_packed)):
        cap = bank.shape[0] if bank is not None else packed.shape[1] if packed is not None else None
        if cap is None or off < 0 or off + rows > cap:
            continue
        if bank is not None:
            bank[off:off + rows, :src.shape[1]] = src
        if packed is not None:
            emu_ops.tc_pack_rows(src, packed, off)


def ring_advance(live_dev, write_dev, rows, cap_rows, pinned_rows, stream=None):
    """Contract of aotb_ring_advance, with the entry point's argument checks."""
    rows, cap_rows, pinned_rows = int(rows), int(cap_rows), int(pinned_rows)
    if not (rows > 0 and pinned_rows >= 0 and pinned_rows + rows <= cap_rows and (cap_rows - pinned_rows) % rows == 0):
        from aot_benchmark_b200._lib import AotbError
        raise AotbError(f"aotb_ring_advance: bad geometry (rows {rows}, cap_rows {cap_rows}, pinned_rows {pinned_rows})")
    live_dev.fill_(min(int(live_dev.item()) + rows, cap_rows))
    w = int(write_dev.item()) + rows
    write_dev.fill_(pinned_rows if w + rows > cap_rows else w)


EMULATED = ("bank_ring_store", "ring_advance")


def install_engine(monkeypatch, wrap=None):
    """emu_ops.install_engine plus the two entry points of the bounded bank; `wrap(name, fn)` decorates them (a tracer)."""
    from aot_benchmark_b200 import ops
    emu_ops.install_engine(monkeypatch)
    for name in EMULATED:
        fn = globals()[name]
        monkeypatch.setattr(ops, name, fn if wrap is None else wrap(name, fn))
