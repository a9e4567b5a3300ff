"""GPU: the Swin-B encoder path (BASELINE configs[3], SURVEY 8 row a19) through the C ABI -- the whole encoder against
oracle.swin_forward (bit-exact to the reference's SwinTransformer, see oracle/gen_golden.py), and the SwinB-AOTL /
SwinB-DeAOTL engines against the committed goldens of the real reference.  The window attention and patch-merge kernels
are compared with float64 in tests/test_gpu_window_envelope.py."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def test_window_attention_rejects_other_geometries():
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import AotbError
    q = torch.zeros(49, 3 * 64, device="cuda")
    with pytest.raises(AotbError):
        ops.window_attention(q, torch.zeros(192, device="cuda"), torch.zeros(1, 49, 49, device="cuda"),
                             torch.zeros(49, 64, device="cuda"), 7, 7, 1, 0)       # head dim 64


@pytest.mark.parametrize("H,W", [(64, 96), (75, 118), (144, 208)])
def test_swin_encoder_vs_oracle(H, W):
    """Whole Swin-B encoder + projector on the GPU vs the oracle (itself bit-exact to the reference's SwinTransformer).
    (75, 118) exercises patch-embed padding and odd patch merges."""
    from aot_benchmark_b200 import EngineConfig, build_vos_model, engine, plan
    from oracle import aot_oracle as O
    from oracle import weights as OW
    sd = OW.build_state_dict("swinb_aotl", seed=0)
    cfg = EngineConfig("t", "swinb_aotl")
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    img = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        want = O.encode_image(sd, O.OracleConfig("swinb_aotl"), img)
        enc = engine._Encoder(plan.get_plan(model), H, W)
        st = torch.cuda.current_stream().cuda_stream
        for rep in range(3):            # eager, captured, replayed: all three must agree with the oracle
            got = enc(img.cuda(), st)
            torch.cuda.synchronize()
            for a, b in zip(got, want):
                assert tuple(a.shape) == tuple(b.shape)
                assert (a.cpu() - b).abs().max().item() < 5e-4 * max(1.0, b.abs().max().item()), rep


@pytest.mark.parametrize("name", ["swinb_aotl_small", "swinb_deaotl_small"])
def test_swin_engine_vs_reference_golden(name, golden_dir):
    from oracle import aot_oracle as O
    from oracle import weights as OW
    from test_gpu_engine import _build_cuda_engine, _tie_band_ok
    g = torch.load(os.path.join(golden_dir, f"video_{name}.pt"))
    sd = OW.build_state_dict(g["model"], seed=g["seed"], flavour=g["flavour"])
    assert OW.checksum(sd) == g["weights_checksum"], "seeded weights are not reproducible on this machine"
    frames, mask = O.synthetic_video(g["frames"], g["H"], g["W"], g["objs"], seed=1234 + g["seed"])
    eng = _build_cuda_engine(g["model"], sd, g["gap"])
    forced = [l.float() for l in g["ref_labels"]]
    with torch.no_grad():
        lo, labels = O.run_video(eng, [f.cuda() for f in frames], mask.cuda(), g["objs"], tuple(g["out_size"]),
                                 forced_masks=forced)
    n = g["objs"] + 1
    dmax = max((a.cpu()[:, :n] - b[:, :n]).abs().max().item() for a, b in zip(lo, g["ref_logits_lo"]))
    assert dmax < 1e-3, f"max |dlogit| vs reference = {dmax}"   # north-star tolerance (fp32 logits)
    assert _tie_band_ok(lo, g["ref_logits_lo"], labels, g["ref_labels"], tuple(g["out_size"]), n, align=False) == 0
    total = sum(b.numel() for b in g["ref_labels"])
    mism = sum((a.cpu().to(torch.uint8) != b).sum().item() for a, b in zip(labels, g["ref_labels"]))
    assert mism <= 2e-4 * total


def test_full_size_cfg4_geometry_tensor_core_vs_fp32_cuda_core_paths():
    """BASELINE configs[3] geometry (SwinB-AOTL, 592x1040 -> 148x260 / 74x130 / 37x65 maps, 10 objects, gap 5) is too big for
    the CPU oracle in a test: at full size the tensor-core path (wgmma GEMMs + attention, CUDA graphs) and the fp32
    CUDA-core path (no graphs) must agree on logits and masks, the run must be deterministic, and the bank must grow as
    the reference schedule says."""
    from aot_benchmark_b200 import engine as engine_mod
    from aot_benchmark_b200 import ops
    from oracle import aot_oracle as O
    from oracle import weights as OW
    from test_gpu_engine import _build_cuda_engine
    sd = OW.build_state_dict("swinb_aotl", seed=11)
    T = 8
    frames, mask = O.synthetic_video(T, 592, 1040, 10, seed=4)
    frames = [f.cuda() for f in frames]
    mask = mask.cuda()
    runs = {}
    for name, (lt, conv, graphs) in {"tc": ("tc_exact", "tc", True), "tc2": ("tc_exact", "tc", True),
                                     "simt": ("simt", "simt", False)}.items():
        old = (engine_mod.LT_IMPL, ops.CONV_IMPL, engine_mod.USE_GRAPHS)
        engine_mod.LT_IMPL, ops.CONV_IMPL, engine_mod.USE_GRAPHS = lt, conv, graphs
        try:
            eng = _build_cuda_engine("swinb_aotl", sd, 5)
            with torch.no_grad():
                lo, labels = O.run_video(eng, frames, mask, 10, (480, 854),
                                         forced_masks=runs["tc"][1] if name != "tc" else None)
            runs[name] = (lo, labels, eng.aot_engines[0].bank_len, eng.aot_engines[0].enc_hw)
        finally:
            engine_mod.LT_IMPL, ops.CONV_IMPL, engine_mod.USE_GRAPHS = old
    lo, labels, bank_len, N = runs["tc"]
    assert N == 37 * 65 == 2405
    assert bank_len == N * (1 + (T - 1) // 5)
    for a, b in zip(lo, runs["tc2"][0]):
        assert torch.equal(a, b)                                    # run-to-run determinism
    dmax = max((a[:, :11] - b[:, :11]).abs().max().item() for a, b in zip(lo, runs["simt"][0]))
    assert dmax < 1e-3, dmax
    # label differences between the two arithmetic paths are only legitimate inside the tie band (SURVEY Appendix E)
    from test_gpu_engine import _tie_band_ok
    assert _tie_band_ok(lo, [t.cpu() for t in runs["simt"][0]], labels, runs["simt"][1], (480, 854), 11, align=False) == 0
    mism = sum((a != b).sum().item() for a, b in zip(labels, runs["simt"][1]))
    total = sum(a.numel() for a in labels)
    assert mism <= 1e-3 * total, (mism, total)
