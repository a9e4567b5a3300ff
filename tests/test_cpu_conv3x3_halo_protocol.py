"""CPU: the discrete-event model of the halo kernel's two rings (scripts/conv_tc_protocol_sim.py, HaloSim).

The weight stage ring (2 to 8 stages, early constant-weight loads or not) beside two halo buffers; CTAs with no tile, one
tile and several, 1 to 4 slices per tile (producers staging the next tile's halos while the consumers finish this one),
each k-step group size of the kernel (KG 1, 2, 4) and the halo released after the slice's last ldmatrix: no halo restaged
while read, every read of the slice and chunk it expects, no bias / scale buffer rewritten under a finish, no deadlock.
A halo released after the slice's first tap instead must be caught."""
import importlib.util
import os

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sim():
    spec = importlib.util.spec_from_file_location("conv_tc_protocol_sim", os.path.join(REPO, "scripts",
                                                                                      "conv_tc_protocol_sim.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("kg", [1, 2, 4])
@pytest.mark.parametrize("stages", [2, 3, 4, 6, 8])
def test_halo_ring_protocol_model(stages, kg):
    m = _sim()
    for tiles in range(0, 5):
        for slices in (1, 2, 3, 4):
            for seed in range(6):
                m.HaloSim(tiles, slices, seed * 7919 + tiles * 31 + slices, stages, kg, early=seed % 2 == 1).run()


@pytest.mark.parametrize("kg", [1, 4])
def test_halo_model_catches_an_early_halo_release(kg):
    m = _sim()
    with pytest.raises(AssertionError, match="reads slice|restaged"):
        for seed in range(50):
            m.HaloSim(2, 2, seed, stages=2, kg=kg, hfree_early=True).run()
