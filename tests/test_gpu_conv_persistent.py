"""GPU: the persistent tensor-core conv (one CTA per SM walking the output tiles in a static order).

- The output does not depend on how many CTAs share the tiles: grid caps 1, 2, 3, 7 and the default give bitwise equal
  outputs in both precisions, on shapes with one, two and many tiles per CTA, tile counts that do not divide by the grid,
  partial last M tiles (M = 1674, 25773), 1x1, 3x3, strided 3x3 and the 4-channel stem gather.
- With several tiles per CTA, BN = 64, 128 and 256 stay bitwise equal to each other.
- The in-place residual linear (out aliasing res), graph replay against eager launches, and a forced split-K tiling (the
  cluster path, within the float64 envelope).
- The constant-weights opt-in changes no value, and ops.linear_tc over operand copies written by the previous kernel of the
  same graph reads the fresh copies (a smoke check; the flag itself is checked on the CPU).
- The diagnostic stamps count every tile once over the CTAs."""
import math

import pytest
import torch

import test_gpu_tc_envelope as EV

pytestmark = pytest.mark.gpu

DEV = EV.DEV
CAPS = (0, 1, 2, 3, 7)

# B, H, W, Cin, Cout, K, stride, pad, residual ("" | "res" | "alias"), act
CASES = [
    (1, 1674, 1, 256, 256, 1, 1, 0, "alias", 1),      # LSTT linear, M = 1674 (partial last tile), residual in place
    (1, 121, 213, 64, 64, 1, 1, 0, "res", 1),         # layer1 1x1 at 480p, M = 25773: 202 tiles, 2 per CTA on 132
    (1, 61, 107, 64, 128, 3, 1, 1, "res", 4),         # 3x3
    (1, 45, 61, 128, 128, 3, 2, 1, "", 0),            # strided 3x3
    (1, 97, 171, 4, 64, 7, 2, 3, "", 1),              # 7x7 stem on the 4-channel gather (Cin % 64 != 0)
    (2, 13, 17, 64, 256, 1, 1, 0, "res", 2),          # batch 2, 4 M tiles x 4 N tiles
]
IDS = ["linear1674_alias", "l1_1x1_25773", "3x3", "3x3s2", "stem7x7", "b2_1x1"]


class _Case:
    def __init__(self, case):
        from aot_benchmark_b200 import ops
        B, H, W, Cin, Cout, K, stride, pad, rmode, act = case
        self.case = case
        g = torch.Generator().manual_seed(H * 131 + W * 3 + Cin + Cout + K)
        self.x = (torch.randn(B, H, W, Cin, generator=g) * 2).to(DEV)
        w = torch.randn(Cout, Cin, K, K, generator=g) / math.sqrt(Cin * K * K)
        self.w4 = w
        self.wh, self.wl, self.ws = ops.split_fp16_scaled(EV._pack_w(w).to(DEV))
        self.b = torch.randn(Cout, generator=g).to(DEV)
        Ho, Wo = (H + 2 * pad - K) // stride + 1, (W + 2 * pad - K) // stride + 1
        self.r = torch.randn(B, Ho, Wo, Cout, generator=g).to(DEV) if rmode else None
        self.out = torch.full((B, Ho, Wo, Cout), float("nan"), device=DEV)
        self.nchunks = (K * K * Cin + 63) // 64
        self.tiles = lambda bn: ((B * Ho * Wo + 127) // 128) * (Cout // bn)

    def run(self, fp16=False, cap=0, tiling=0, const_w=False):
        from aot_benchmark_b200 import ops
        from aot_benchmark_b200._lib import lib
        B, H, W, Cin, Cout, K, stride, pad, rmode, act = self.case
        assert lib().aotb_set_conv_grid_cap(cap) == 0
        assert lib().aotb_set_conv_tiling(tiling) == 0
        try:
            self.out.fill_(float("nan"))
            if rmode == "alias":
                self.out.copy_(self.r)
            res = self.out if rmode == "alias" else self.r
            ops.conv2d_tc(self.x, self.wh, None if fp16 else self.wl, self.b, self.out, res=res, KH=K, KW=K,
                          stride=stride, pad=pad, act=act, wscale=self.ws, const_w=const_w)
            torch.cuda.synchronize()
        finally:
            lib().aotb_set_conv_tiling(0)
            lib().aotb_set_conv_grid_cap(0)
        return self.out.clone()


@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_outputs_equal_across_grid_caps(case, fp16):
    c = _Case(case)
    base = c.run(fp16)
    assert not torch.isnan(base).any()
    for cap in CAPS[1:]:
        got = c.run(fp16, cap=cap)
        assert torch.equal(got, base), f"cap {cap}: max |d| = {(got - base).abs().max().item():.3e}"
    if not fp16:      # and the values are right
        B, H, W, Cin, Cout, K, stride, pad, rmode, act = case
        ref = EV._ref_conv(c.x.cpu(), c.w4, c.b.cpu(), stride, pad, None if c.r is None else c.r.cpu(), act)
        err = (base.double().cpu() - ref).abs().max().item()
        assert err < 1e-5 * max(ref.abs().max().item(), 1.0) + 1e-5, err


@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
@pytest.mark.parametrize("cap", [1, 3, 0])
def test_n_tiles_equal_with_several_tiles_per_cta(cap, fp16):
    c = _Case(CASES[5])
    outs = {bn: c.run(fp16, cap=cap, tiling=(code << 4) | (1 << 8)) for code, bn in ((1, 64), (2, 128), (3, 256))}
    assert not torch.isnan(outs[64]).any()
    for bn, o in outs.items():
        assert torch.equal(o, outs[64]), f"BN {bn} differs from BN 64 at cap {cap}"


@pytest.mark.parametrize("cap", [0, 1, 5])
def test_inplace_residual_linear(cap):
    """ops.linear(x, W, b, out=y, res=y): every tile reads only the residual rows it then overwrites."""
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import lib
    g = torch.Generator().manual_seed(5)
    M, K, N = 1674, 256, 512
    x = torch.randn(M, K, generator=g).to(DEV)
    wk = (torch.randn(K, N, generator=g) / 16).to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    y0 = torch.randn(M, N, generator=g).to(DEV)
    ops.register_tc_weights(wk, *ops.split_fp16_scaled(wk))
    impl = ops.CONV_IMPL
    ops.CONV_IMPL = "tc"
    try:
        assert lib().aotb_set_conv_grid_cap(cap) == 0
        sep = torch.empty(M, N, device=DEV)
        ops.linear(x, wk, b, sep, res=y0)
        y = y0.clone()
        ops.linear(x, wk, b, y, res=y)
        torch.cuda.synchronize()
    finally:
        ops.CONV_IMPL = impl
        lib().aotb_set_conv_grid_cap(0)
        ops._TC_WEIGHTS.pop(wk.data_ptr(), None)
    assert torch.equal(y, sep)
    ref = x.double() @ wk.double() + b.double() + y0.double()
    assert (y.double() - ref).abs().max().item() < 1e-4


def test_graph_replay_equals_eager():
    from aot_benchmark_b200 import ops
    c = _Case(CASES[1])
    eager = c.run(const_w=True)
    B, H, W, Cin, Cout, K, stride, pad, rmode, act = c.case
    out = torch.full_like(c.out, float("nan"))
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fn = lambda: ops.conv2d_tc(c.x, c.wh, c.wl, c.b, out, res=c.r, KH=K, KW=K, stride=stride, pad=pad,  # noqa: E731
                                   act=act, wscale=c.ws, const_w=True)
        fn()
        st.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=st):
            for _ in range(3):
                fn()
        out.fill_(float("nan"))
        gr.replay()
        st.synchronize()
    assert torch.equal(out, eager)


@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
def test_forced_split_k_keeps_the_cluster_path(fp16):
    c = _Case(CASES[2])      # 9 chunks
    B, H, W, Cin, Cout, K, stride, pad, rmode, act = c.case
    ref = EV._ref_conv(c.x.cpu(), c.w4, c.b.cpu(), stride, pad, c.r.cpu(), act)
    tol = (2e-2 if fp16 else 1e-5) * max(ref.abs().max().item(), 1.0)
    for S in (2, 4, 8):
        runs = [c.run(fp16, tiling=(2 << 4) | (S << 8)) for _ in range(2)]
        err = (runs[0].double().cpu() - ref).abs().max().item()
        assert err < tol, f"S {S}: err {err:.3e}"
        assert torch.equal(runs[0], runs[1])


def test_constant_weight_opt_in_changes_nothing():
    c = _Case(CASES[4])
    for fp16 in (False, True):
        for cap in (0, 2):
            assert torch.equal(c.run(fp16, cap=cap, const_w=True), c.run(fp16, cap=cap))


def test_linear_tc_reads_bank_copies_written_just_before():
    """The DeAOT bank path end to end: split_rows refreshes the operand copies and linear_tc reads them in the next launch,
    inside one graph with programmatic dependent launch on, and sees the refreshed keys every replay.  A wrongly early
    weight fetch would only fail here through a race, so this is a smoke check; the deterministic guard of the opt-in is
    test_cpu_conv_persistent.py::test_constant_weight_flag_only_for_packed_weights (linear_tc never sets the flag)."""
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import lib
    g = torch.Generator().manual_seed(11)
    M, D, T = 700, 128, 384
    q = torch.randn(M, D, generator=g).to(DEV)
    keys = [torch.randn(T, D, generator=g).to(DEV) for _ in range(3)]
    src = torch.empty(T, D, device=DEV)
    kh = torch.zeros(T, D, dtype=torch.float16, device=DEV)
    kl = torch.zeros_like(kh)
    out = torch.empty(M, T, device=DEV)
    lib().aotb_set_pdl(1)
    try:
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            def body():
                ops.split_rows(src, kh, kl, stream=st)
                ops.linear_tc(q, kh, kl, None, out, stream=st)
            src.copy_(keys[0])
            body()
            st.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=st):
                body()
            for k in keys:
                src.copy_(k)
                gr.replay()
                st.synchronize()
                ref = q.double() @ k.double().t()
                assert (out.double() - ref).abs().max().item() < 1e-3
    finally:
        from aot_benchmark_b200 import engine
        lib().aotb_set_pdl(1 if engine.USE_PDL else 0)


def test_profile_stamps_count_every_tile_once():
    from aot_benchmark_b200 import ops
    from aot_benchmark_b200._lib import lib
    c = _Case(CASES[0])
    ws = ops._tc_workspace(DEV)
    for cap in (1, 3, 0):
        ws.zero_()
        c.run(cap=cap, tiling=4 | (1 << 4) | (1 << 8))
        st = ws.view(torch.int64)[: 12 * 4096].view(-1, 12).cpu()
        st = st[st[:, 7] != 0]
        assert st.shape[0] == (cap or min(c.tiles(64), torch.cuda.get_device_properties(0).multi_processor_count))
        assert int(st[:, 11].sum()) == c.tiles(64)
        assert (st[:, 10] >= st[:, 3]).all() and (st[:, 4] >= st[:, 10]).all()
    lib().aotb_set_conv_tiling(0)
