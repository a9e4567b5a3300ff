"""CPU: the LSTT of the AOT models with the 8 x 32 head shape runs the tensor-core short-term attention by default, inside its
captured graph bodies, and those bodies stay static across frames.  The engine issues it through local_attention_tile inside
ops.local_kernel("tc"), which forwards to local_attention_tc.  Uses the emulated C-ABI and the tracing graph cache of
test_cpu_graph_static: a replay that issues other launches than its capture fails."""
import collections

import pytest
import torch

import test_cpu_graph_static as G
from oracle import aot_oracle as O
from oracle import weights as OW


@pytest.mark.parametrize("model_name,H,W", [("r50_aotl", 97, 129), ("swinb_aotl", 96, 128)])
def test_lstt_calls_the_tensor_core_local_attention(monkeypatch, model_name, H, W):
    from aot_benchmark_b200 import ops
    G._install(monkeypatch)
    calls = collections.Counter()

    def counted(name, fn):
        def wrapper(*args, **kwargs):
            calls[(name, ops._LOCAL_KERNEL, G.TRACE is not None)] += 1
            return fn(*args, **kwargs)
        return wrapper

    for name in ("local_attention_tile", "local_attention"):
        monkeypatch.setattr(ops, name, counted(name, getattr(ops, name)))
    eng = G._engine(model_name, OW.build_state_dict(model_name, seed=4), 2)
    frames, mask = O.synthetic_video(5, H, W, 2, seed=31)
    with torch.no_grad():
        O.run_video(eng, frames, mask, 2, (H, W))
    assert G.TracingGraphCache.replays > 0
    assert calls[("local_attention_tile", "tc", True)] > 0, calls        # inside captured (and replayed) bodies
    assert set(calls) <= {("local_attention_tile", "tc", True), ("local_attention_tile", "tc", False)}, calls
    assert ops._LOCAL_KERNEL == "tile"


def test_local_kernel_selects_the_entry_point(monkeypatch):
    """local_attention_tile forwards every argument to local_attention_tc inside local_kernel("tc") only."""
    from aot_benchmark_b200 import ops
    seen = []
    monkeypatch.setattr(ops, "local_attention_tc", lambda *a, **k: seen.append((a, k)) or "tc")
    args = tuple(range(10))
    with ops.local_kernel("tc"):
        assert ops.local_attention_tile(*args, stream=7) == "tc"
    assert seen == [(args, {"stream": 7})]
    with pytest.raises(ValueError):
        with ops.local_kernel("warp"):
            pass
    assert ops._LOCAL_KERNEL == "tile"
