"""CPU: the persistent tensor-core conv without a GPU.

- The discrete-event model of its stage ring (scripts/conv_tc_protocol_sim.py): tiles crossing the ring with the chunk
  counter and the barrier phases carried over, CTAs with no tile, one tile and several, early constant-weight loads, and
  the split-K form whose finish stages its tile in the operand stages: no deadlock, no stage overwritten while read.
- The constant-weights opt-in: ops.conv2d / ops.linear over packed model weights set AOTB_CONV_CONST_WEIGHTS in the act
  argument; ops.linear_tc (memory-bank operand copies, refreshed by kernels of the same stream) never does."""
import importlib.util
import os

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sim():
    spec = importlib.util.spec_from_file_location("conv_tc_protocol_sim", os.path.join(REPO, "scripts",
                                                                                      "conv_tc_protocol_sim.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("stages", [2, 3, 4, 6, 8])
def test_persistent_ring_protocol_model(stages):
    m = _sim()
    for tiles in range(0, 6):
        for chunks in (1, 2, 3, 4, 7):
            for seed in range(12):
                for early in (False, True):
                    m.Sim(tiles, chunks, seed * 7919 + tiles * 31 + chunks, stages, early).run()


@pytest.mark.parametrize("stages", [2, 3, 4, 8])
def test_split_k_ring_protocol_model(stages):
    m = _sim()
    for tiles in (0, 1):
        for chunks in (0, 1, 2, 5, 9):
            for seed in range(12):
                m.Sim(tiles, chunks, seed * 104729 + chunks, stages, early=seed % 2 == 0, splitk=True).run()


def test_protocol_model_catches_an_unreleased_last_stage():
    """Without the release of each tile's last stage the ring runs dry after STAGES tiles: the model must report it."""
    m = _sim()
    m.Sim(2, 1, 0, stages=2, release_last=False).run()
    with pytest.raises(AssertionError, match="deadlock"):
        m.Sim(3, 1, 0, stages=2, release_last=False).run()


class _FakeLib:
    def __init__(self):
        self.acts = []

    def aotb_conv2d_nhwc_tc(self, *args):
        self.acts.append(args[19])
        return 0


def test_constant_weight_flag_only_for_packed_weights(monkeypatch):
    from aot_benchmark_b200 import ops
    fake = _FakeLib()
    monkeypatch.setattr(ops, "lib", lambda: fake)
    monkeypatch.setattr(ops, "_chk", lambda *ts: None)
    monkeypatch.setattr(ops, "_tc_workspace", lambda dev: torch.zeros(1, dtype=torch.uint8))
    monkeypatch.setattr(ops, "CONV_IMPL", "tc")
    monkeypatch.setattr(ops, "_st", lambda stream: None)
    F = ops.CONV_CONST_WEIGHTS
    w = torch.randn(64, 128)
    wh, wl, ws = ops.split_fp16_scaled(w)
    ops.register_tc_weights(w, wh, wl, ws)
    try:
        x, out = torch.randn(10, 64), torch.empty(10, 128)
        ops.linear(x, w, None, out, act=ops.ACT_RELU)
        ops.conv2d(x.view(1, 10, 1, 64), w, None, out.view(1, 10, 1, 128), act=ops.ACT_RELU)
        ops.linear_tc(x, wh[:, :64].contiguous(), wl[:, :64].contiguous(), None, out, act=ops.ACT_RELU)
        ops.conv2d_tc(x.view(1, 10, 1, 64), wh, wl, None, out.view(1, 10, 1, 128), act=ops.ACT_RELU)
    finally:
        ops._TC_WEIGHTS.pop(w.data_ptr(), None)
    assert fake.acts == [ops.ACT_RELU | F, ops.ACT_RELU | F, ops.ACT_RELU, ops.ACT_RELU]
