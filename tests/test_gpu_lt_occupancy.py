"""The default ("tile") layout of the tensor-core long-term attention runs two CTAs per SM: its kernel fits 96 registers
without spilling in both modes, and the carveout leaves shared memory for two 83 KB CTAs (aotb_lt_attn_tc_occupancy).  The
KV-split policy sizes its waves from that count (engine.LT_TILE_CTAS_PER_SM)."""
import pytest
import torch

from aot_benchmark_b200 import engine, ops


@pytest.mark.gpu
@pytest.mark.parametrize("exact", [True, False])
def test_tile_kernel_two_ctas_per_sm(exact):
    torch.cuda.set_device(0)
    ctas, regs, local = ops.lt_attn_tc_occupancy(exact)
    assert ctas == 2 == engine.LT_TILE_CTAS_PER_SM, (ctas, regs, local)
    assert 0 < regs <= 96, regs
    assert local == 0, local
