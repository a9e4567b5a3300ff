"""The long-term attention's KV-split policy (engine.lt_splits) sizes its waves from the resident CTAs per SM of the default
("tile") layout, engine.LT_TILE_CTAS_PER_SM; the other layouts keep their own residency."""
import pytest

from aot_benchmark_b200 import engine

N, H = 1674, 8                      # the benchmark's 481x849 input: 1674 queries, 8 heads of 32


@pytest.mark.parametrize("ctas", [1, 2])
def test_benchmark_shapes_take_seven_splits(monkeypatch, ctas):
    # the 99-frame clip: the self-attention (Tk = N) and banks of 1 .. 20 memory frames; 112 CTAs x 7 splits fill 132 and
    # 264 slots to 99 %
    monkeypatch.setattr(engine, "LT_TILE_CTAS_PER_SM", ctas)
    for m in range(1, 21):
        assert engine.lt_splits(N, H, N * m, variant="tile") == 7, m


@pytest.mark.parametrize("n, one, two", [(2048, 1, 2), (1024, 2, 4)])
def test_slots_follow_residency(monkeypatch, n, one, two):
    # 128 CTAs (n = 2048) fill one wave of 132 slots, but half of one of 264; 64 CTAs (n = 1024) need 2 and 4 splits
    for ctas, want in ((1, one), (2, two)):
        monkeypatch.setattr(engine, "LT_TILE_CTAS_PER_SM", ctas)
        assert engine.lt_splits(n, H, 10 * N, variant="tile") == want


@pytest.mark.parametrize("variant, n, want", [("groups", 2048, 1), ("ahead", 1024, 2), ("pair", 1024, 2)])
def test_other_layouts_keep_their_residency(monkeypatch, variant, n, want):
    # groups / ahead stay bounded for one 128-query CTA per SM and pair for two 64-query CTAs, whatever the tile layout's
    # residency
    monkeypatch.setattr(engine, "LT_TILE_CTAS_PER_SM", 7)
    assert engine.lt_splits(n, H, 10 * N, variant=variant) == want
