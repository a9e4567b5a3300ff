"""TEST INFRASTRUCTURE ONLY: CPU emulations of the batched C-ABI entry points (include/aotb200.h, the `*_batched_*` forms).

Their contract is that image b of a B-image launch equals the one-image launch on image b, so each emulation here runs the
one-image emulation already installed on `aot_benchmark_b200.ops` (tests/emu_ops.py, and the split-attention / squeeze-excite
emulations of test_cpu_resnest_host / test_cpu_mbv3_rs50_host) image by image.  A one-image call goes straight through.
"""


def _views(t, B):
    """Image b's rows of a [B, ...] tensor or of its flat [B * n] form."""
    return [t.reshape(B, -1)[b] for b in range(B)]


def install(monkeypatch):
    from aot_benchmark_b200 import ops
    one = {n: getattr(ops, n) for n in ("window_attention", "patch_merge", "splat_workspace", "splat_attention",
                                        "splat_combine", "se_gate", "gate_scale")}

    def window_attention(qkv, qkv_bias, rel_bias, out, H, W, heads, shift, window=7, stream=None, B=1):
        n = H * W
        for b in range(B):
            one["window_attention"](qkv[b * n:(b + 1) * n], qkv_bias, rel_bias, out[b * n:(b + 1) * n], H, W, heads, shift,
                                    window=window)
        return out

    def patch_merge(x, out, H, W, stream=None, B=1):
        n, m = H * W, ((H + 1) // 2) * ((W + 1) // 2)
        for b in range(B):
            one["patch_merge"](x[b * n:(b + 1) * n], out[b * m:(b + 1) * m], H, W)
        return out

    def splat_workspace(C, device, B=1):
        return one["splat_workspace"](C, device)

    def splat_attention(x, w1, b1, w2, b2, att, workspace, radix=2, stream=None):
        B = x.shape[0] if x.dim() == 4 else 1
        if B == 1:
            return one["splat_attention"](x, w1, b1, w2, b2, att, workspace, radix=radix)
        for b, a in enumerate(_views(att, B)):
            one["splat_attention"](x[b:b + 1], w1, b1, w2, b2, a, workspace, radix=radix)
        return att

    def splat_combine(x, att, out, radix=2, pool_stride=0, stream=None):
        B = x.shape[0]
        if B == 1:
            return one["splat_combine"](x, att, out, radix=radix, pool_stride=pool_stride)
        for b, a in enumerate(_views(att, B)):
            one["splat_combine"](x[b:b + 1], a, out[b:b + 1], radix=radix, pool_stride=pool_stride)
        return out

    def se_gate(x, w1, b1, w2, b2, gate, workspace, stream=None):
        B = x.shape[0] if x.dim() == 4 else 1
        if B == 1:
            return one["se_gate"](x, w1, b1, w2, b2, gate, workspace)
        for b, g in enumerate(_views(gate, B)):
            one["se_gate"](x[b:b + 1], w1, b1, w2, b2, g, workspace)
        return gate

    def gate_scale(x, gate, out, act=0, stream=None):
        B = x.shape[0]
        if B == 1:
            return one["gate_scale"](x, gate, out, act=act)
        for b, g in enumerate(_views(gate, B)):
            one["gate_scale"](x[b:b + 1], g, out[b:b + 1], act=act)
        return out

    for f in (window_attention, patch_merge, splat_workspace, splat_attention, splat_combine, se_gate, gate_scale):
        monkeypatch.setattr(ops, f.__name__, f)
