"""CPU: GPU-free models of the tensor-core attention kernel (csrc/attn_tc.cuh) and the conv K loop (csrc/conv_tc.cu):
  * a discrete-event model of the TMA / mbarrier K-V stage ring (parity waits, asynchronous wgmma reads) in the default and
    the "ahead" issue order and with the DeAOT kernel's parameters: no deadlock, no overwrite of a stage being read;
  * an address-level model of the data path (128B-swizzled tiles, wgmma descriptor offsets, accumulator and register
    fragment layouts, the conv producer's store slots) under which the kernels' addressing reproduces the reference."""
import importlib.util
import os

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REPO, "scripts", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_ahead_layout_protocol_model():
    m = _load("attn_tc_protocol_sim")
    for T in range(0, 9):
        for seed in range(25):
            m.Sim(T, seed * 7919 + T, stages=4, nwg=2, ahead=True).run()      # "ahead"
            m.Sim(T, seed * 7919 + T, stages=4, nwg=2, ahead=False).run()     # "tile"
            m.Sim(T, seed * 7919 + T, stages=4, nwg=1, ahead=False).run()     # "pair"
            m.Sim(T, seed * 7919 + T, stages=2, nwg=2, ahead=False).run()     # "groups"


def test_fused_deaot_kernel_protocol_model():
    m = _load("attn_tc_protocol_sim")
    for T in range(0, 11):
        for seed in range(25):
            m.Sim(T, seed * 104729 + T, stages=2, nwg=2, ahead=False).run()


def test_tensor_core_layout_model():
    m = _load("tc_layout_model")
    rng = np.random.default_rng(1)
    Q = (rng.standard_normal((64, 32)) * 3).astype(np.float32)
    K = rng.standard_normal((150, 32)).astype(np.float32)
    V = rng.standard_normal((150, 32)).astype(np.float32)
    ref = m.reference(Q.astype(np.float64), K.astype(np.float64), V.astype(np.float64), np.sqrt(32.0))
    for bk in (64, 128):                                                      # "tile" / "groups" score tiles
        assert np.abs(m.model_attention(Q, K, V, np.sqrt(32.0), qc=1, bk=bk) - ref).max() < 1e-4
    Q = (rng.standard_normal((64, 128)) * 2).astype(np.float32)               # DeAOT: 4 query / key chunks
    K = rng.standard_normal((100, 128)).astype(np.float32)
    V = rng.standard_normal((100, 32)).astype(np.float32)
    ref = m.reference(Q.astype(np.float64), K.astype(np.float64), V.astype(np.float64), np.sqrt(128.0))
    assert np.abs(m.model_attention(Q, K, V, np.sqrt(128.0), qc=4) - ref).max() < 1e-4
    X = rng.standard_normal((128, 64)).astype(np.float32)
    assert np.array_equal(m.model_conv_a_tile(X), X.astype(np.float16).astype(np.float32))
