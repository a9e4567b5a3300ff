"""Thin tensor-level wrappers over the C ABI (include/aotb200.h).

PyTorch is used here only for device memory (tensors) and streams.  Every function launches
hand-written sm_90a kernels from libaotb200.so on ``stream`` (a raw cudaStream_t int, default:
torch's current stream) and raises ``AotbError`` on failure -- there is no eager fallback.

Layout conventions: activations are NHWC ``[B,H,W,C]`` or token matrices ``[rows, C]`` whose last
stride is 1; channel-sliced views are fine (the row stride is passed as ``ld``), except where a wrapper says its
operands must be contiguous (the label-map, logit post-processing and ID-embedding kernels), and there it checks.
"""
from __future__ import annotations

import contextlib
import os

import torch

from ._lib import AotbError, check, lib

ACT_NONE, ACT_RELU, ACT_GELU, ACT_SILU, ACT_RELU6, ACT_HSWISH = 0, 1, 2, 3, 4, 5
EW_COPY, EW_ADD, EW_MUL, EW_SILU, EW_SILU_MUL, EW_FILL = 0, 1, 2, 3, 4, 5


def _st(stream):
    return torch.cuda.current_stream().cuda_stream if stream is None else stream


def _chk(*ts):
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda or t.dtype != torch.float32:
            raise AotbError(f"aot_benchmark_b200 kernels need float32 CUDA tensors, got {t.dtype} on {t.device}")
        if t.dim() >= 1 and t.stride(-1) != 1:
            raise AotbError("innermost stride must be 1")


def _p(t):
    return None if t is None else t.data_ptr()


def _nhwc_ld(x):
    B, H, W, C = x.shape
    ld = x.stride(2)
    if x.stride(1) != W * ld or (B > 1 and x.stride(0) != H * W * ld):
        raise AotbError("NHWC tensor must be dense over pixels")
    return ld


# fp32 weight (by data_ptr) -> (wh, wl, wscale, w): split-fp16 [Cout, K] copies for the tensor-core conv and their
# per-channel scale (None = 1), registered by plan.py
_TC_WEIGHTS = {}
CONV_IMPL = os.environ.get("AOTB_CONV_IMPL", "tc")     # "tc" (wgmma, fp16x2 split) | "simt" (fp32 CUDA cores)
PRECISIONS = ("fp32", "fp16")
# operand precision of the tensor-core conv / linear launches issued by conv2d and linear: "fp32" = split fp16 (three MMAs,
# fp32-faithful), "fp16" = operands rounded once (the single-pass kernel).  An engine sets it around its own calls with
# `precision`, so two engines of different precision in one process each launch in their own mode.
_PRECISION = "fp32"


@contextlib.contextmanager
def precision(p):
    """Issue the tensor-core conv / linear launches of the enclosed calls in precision `p` ("fp32" | "fp16")."""
    global _PRECISION
    if p not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {p!r}")
    old, _PRECISION = _PRECISION, p
    try:
        yield
    finally:
        _PRECISION = old


_TC_WS = {}
# bench.py hook: when set to a list, every tensor-core conv / linear launch appends (start_event, end_event, flops) with
# flops = 2 * M * N * K (algorithmic: one multiply-add per weight per output) so the conv family's roofline is measured live
CONV_PROBE = None


class _ConvProbe:
    def __init__(self, flops, stream):
        self.on = CONV_PROBE is not None and stream in (None, torch.cuda.current_stream().cuda_stream)
        self.flops = flops

    def __enter__(self):
        if self.on:
            self.e0, self.e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *a):
        if self.on:
            self.e1.record()
            CONV_PROBE.append((self.e0, self.e1, self.flops))


def _tc_workspace(device):
    """Per-device scratch handed to the tensor-core conv (reserved by the C-ABI; currently unused by the kernel)."""
    ws = _TC_WS.get(device)
    if ws is None:
        ws = _TC_WS[device] = torch.zeros(1 << 20, dtype=torch.uint8, device=device)
    return ws


def register_tc_weights(w, wh, wl, wscale=None):
    _TC_WEIGHTS[w.data_ptr()] = (wh, wl, wscale, w)     # keep w alive so the pointer key stays unique


def split_fp16(w_kn):
    """fp32 [K, N] -> (hi, lo) fp16 [N, Kpad] (K zero-padded to a multiple of 64) with hi + lo ~= w to 2^-22 relative,
    but never closer than the fp16 subnormal spacing of lo (2^-25 absolute): see split_fp16_scaled."""
    K = w_kn.shape[0]
    wt = w_kn.t().contiguous()
    if K % 64:
        wt = torch.nn.functional.pad(wt, (0, 64 - K % 64))
    hi = wt.half()
    lo = (wt - hi.float()).half()
    return hi.contiguous(), lo.contiguous()


def weight_scale_exponents(w_kn):
    """fp32 [K, N] -> int32 [N]: e_n = 13 - floor(log2 max_k |w[k][n]|), so that 2^13 <= max_k |w[k][n]| 2^e_n < 2^14
    (0 for an all-zero column; at most 126 so that 2^-e_n stays a normal fp32 number)."""
    amax = w_kn.abs().amax(dim=0).float()
    _, ex = torch.frexp(amax)                      # amax = m 2^ex, m in [0.5, 1): floor(log2 amax) = ex - 1
    e = (14 - ex).clamp(max=126)
    return torch.where(amax > 0, e, torch.zeros_like(e)).to(torch.int32)


def split_fp16_scaled(w_kn):
    """fp32 [K, N] -> (hi, lo, wscale): split_fp16 of w normalised per output channel, w[:, n] 2^e_n
    (weight_scale_exponents), and wscale = 2^-e_n fp32 [N].  Both scalings are exact, and the tensor-core finish multiplies
    the accumulator by wscale: a channel of any magnitude keeps the 2^-22 relative precision of the split instead of
    hitting the absolute floor of lo."""
    e = weight_scale_exponents(w_kn)
    hi, lo = split_fp16(w_kn.float() * _pow2(e))
    return hi, lo, _pow2(-e)


def _pow2(e):
    """int32 exponents in [-126, 127] -> exact fp32 powers of two (built from the exponent bits)."""
    return ((e + 127) << 23).to(torch.int32).view(torch.float32)


# flag in the act argument of aotb_conv2d_nhwc_tc (include/aotb200.h): the weights are never written by a kernel
CONV_CONST_WEIGHTS = 256

# bench.py's encoder probe saves this flag, sets it False and restores it; no encoder path reads it
CONV_CHAIN = False


def conv2d_tc(x, wh, wl, bias, out, res=None, KH=1, KW=1, stride=1, pad=0, act=ACT_NONE, stream=None, wscale=None,
              const_w=False):
    """Tensor-core conv: x [B,H,W,Cin] fp32, wh/wl [Cout, KH*KW*Cin] fp16, wscale fp32 [Cout] or None (= 1).
    wl None: the single-pass kernel (x rounded once to fp16, wh only).  const_w: no earlier kernel in the stream writes
    wh / wl (packed model weights), so the kernel may load them before it waits for the previous kernel."""
    _chk(x, bias, out, res, wscale)
    B, H, W, Cin = x.shape
    Cout = wh.shape[0]
    ws = _tc_workspace(x.device)
    with _ConvProbe(2.0 * out.shape[0] * out.shape[1] * out.shape[2] * Cout * KH * KW * Cin, stream):
        check(lib().aotb_conv2d_nhwc_tc(_p(x), wh.data_ptr(), _p(wl), _p(bias), _p(wscale), _p(res), _p(out), B, H, W, Cin,
                                        _nhwc_ld(x), Cout, _nhwc_ld(out), _nhwc_ld(res) if res is not None else 0, KH, KW,
                                        stride, pad, act | (CONV_CONST_WEIGHTS if const_w else 0), ws.data_ptr(), ws.numel(),
                                        _st(stream)), "aotb_conv2d_nhwc_tc")
    return out


def conv2d(x, w, bias, out, res=None, KH=1, KW=1, stride=1, pad=0, dil=1, act=ACT_NONE, stream=None):
    """x [B,H,W,Cin], w [KH*KW*Cin, Cout], out [B,Ho,Wo,Cout] (+res like out)."""
    if CONV_IMPL == "tc" and dil == 1:
        t = _TC_WEIGHTS.get(w.data_ptr())
        if t is not None:
            return conv2d_tc(x, t[0], None if _PRECISION == "fp16" else t[1], bias, out, res=res, KH=KH, KW=KW, stride=stride, pad=pad, act=act,
                             stream=stream, wscale=t[2], const_w=True)
    _chk(x, w, bias, out, res)
    B, H, W, Cin = x.shape
    Cout = w.shape[1]
    check(lib().aotb_conv2d_nhwc_f32(_p(x), _p(w), _p(bias), _p(res), _p(out), B, H, W, Cin, _nhwc_ld(x), Cout,
                                     _nhwc_ld(out), _nhwc_ld(res) if res is not None else 0, KH, KW, stride, pad,
                                     dil, act, _st(stream)), "aotb_conv2d_nhwc_f32")
    return out


def linear(x, wt, bias, out, res=None, act=ACT_NONE, stream=None):
    """x [M,K], wt [K,N], out [M,N] (+res [M,N]); res may alias out (in-place accumulate)."""
    if CONV_IMPL == "tc":
        t = _TC_WEIGHTS.get(wt.data_ptr())
        if t is not None:
            _chk(x, bias, out, res, t[2])
            M, K = x.shape
            N = wt.shape[1]
            ws = _tc_workspace(x.device)
            with _ConvProbe(2.0 * M * N * K, stream):
                wl = None if _PRECISION == "fp16" else t[1]
                check(lib().aotb_conv2d_nhwc_tc(_p(x), t[0].data_ptr(), _p(wl), _p(bias), _p(t[2]), _p(res), _p(out),
                                                1, M, 1, K, x.stride(0), N, out.stride(0), res.stride(0) if res is not None else 0,
                                                1, 1, 1, 0, act | CONV_CONST_WEIGHTS, ws.data_ptr(), ws.numel(), _st(stream)),
                      "aotb_conv2d_nhwc_tc")
            return out
    _chk(x, wt, bias, out, res)
    M, K = x.shape
    N = wt.shape[1]
    check(lib().aotb_linear_f32(_p(x), _p(wt), _p(bias), _p(res), _p(out), M, K, x.stride(0), N, out.stride(0),
                                res.stride(0) if res is not None else 0, act, _st(stream)), "aotb_linear_f32")
    return out


def linear_tc(x, wh, wl, bias, out, res=None, act=ACT_NONE, stream=None):
    """out[M][N] = act(x[M][K] @ W^T + bias + res) on the tensor-core GEMM with explicitly given split-fp16 weights
    wh / wl [N][K] (K % 64 == 0, N % 64 == 0) -- e.g. operand copies of the memory bank.  Kernels of the same stream
    may write wh / wl, so the weights are read only after the previous kernel (CONV_CONST_WEIGHTS stays clear)."""
    _chk(x, bias, out, res)
    if wh.dtype != torch.float16 or wl.dtype != torch.float16 or wh.shape != wl.shape or not wh.is_contiguous() \
            or not wl.is_contiguous():
        raise AotbError("linear_tc: wh / wl must be contiguous fp16 tensors of the same shape [N, K]")
    M, K = x.shape
    N = wh.shape[0]
    if wh.shape[1] != K or K % 64 or N % 64 or out.shape[0] != M or out.shape[1] != N:
        raise AotbError(f"linear_tc: shapes x {tuple(x.shape)}, w {tuple(wh.shape)}, out {tuple(out.shape)}")
    ws = _tc_workspace(x.device)
    check(lib().aotb_conv2d_nhwc_tc(_p(x), wh.data_ptr(), wl.data_ptr(), _p(bias), None, _p(res), _p(out), 1, M, 1, K,
                                    x.stride(0), N, out.stride(0), res.stride(0) if res is not None else 0, 1, 1, 1, 0,
                                    act, ws.data_ptr(), ws.numel(), _st(stream)), "aotb_conv2d_nhwc_tc")
    return out


def split_rows(src, hi, lo, row_off=0, row_off_dev=None, stream=None):
    """src fp32 [rows, C] -> hi / lo fp16 [cap, ldw] rows [row_off, row_off + rows)."""
    _chk(src)
    rows, C = src.shape
    check(lib().aotb_split_rows_f16x2(_p(src), src.stride(0), hi.data_ptr(), lo.data_ptr(), hi.stride(0), rows, C,
                                      int(row_off), row_off_dev.data_ptr() if row_off_dev is not None else None,
                                      _st(stream)), "aotb_split_rows_f16x2")


def split_cols(src, hiT, loT, col_off=0, col_off_dev=None, stream=None):
    """src fp32 [rows, C] -> columns [col_off, col_off + rows) of hiT / loT fp16 [C, cap]."""
    _chk(src)
    rows, C = src.shape
    check(lib().aotb_split_cols_f16x2(_p(src), src.stride(0), hiT.data_ptr(), loT.data_ptr(), hiT.stride(0), rows, C,
                                      int(col_off), col_off_dev.data_ptr() if col_off_dev is not None else None,
                                      _st(stream)), "aotb_split_cols_f16x2")


def row_softmax(S, cols, Tk, scale, Tk_dev=None, stream=None):
    """In place on S [N, >= cols]: softmax(scale * S[r, :live]) in columns [0, live), zeros in [live, cols)."""
    _chk(S)
    check(lib().aotb_row_softmax_f32(_p(S), S.stride(0), S.shape[0], int(cols), int(Tk),
                                     Tk_dev.data_ptr() if Tk_dev is not None else None, float(scale), _st(stream)),
          "aotb_row_softmax_f32")
    return S


def nchw_to_nhwc(x, out, stream=None):
    _chk(x, out)
    B, C, H, W = x.shape
    check(lib().aotb_nchw_to_nhwc_f32(_p(x.contiguous()), _p(out), B, C, H * W, _st(stream)), "aotb_nchw_to_nhwc_f32")
    return out


def image_to_nhwc4(img, out, stream=None):
    """img [B,3,H,W] -> out [B,H,W,4] (4th channel zero)."""
    _chk(img, out)
    B = img.shape[0]
    if tuple(out.shape) != (B, img.shape[2], img.shape[3], 4) or not out.is_contiguous():
        raise AotbError(f"image_to_nhwc4: out must be a contiguous [{B}, H, W, 4] tensor, got {tuple(out.shape)}")
    check(lib().aotb_image_to_nhwc4_batched_f32(_p(img.contiguous()), _p(out), B, img.shape[2] * img.shape[3], _st(stream)),
          "aotb_image_to_nhwc4_f32")
    return out


def nhwc_to_nchw(x, out, stream=None):
    _chk(x, out)
    B, H, W, C = x.shape
    check(lib().aotb_nhwc_to_nchw_f32(_p(x), _p(out), B, C, H * W, _st(stream)), "aotb_nhwc_to_nchw_f32")
    return out


def maxpool3x3s2(x, out, stream=None):
    _chk(x, out)
    B, H, W, C = x.shape
    check(lib().aotb_maxpool3x3s2_nhwc_f32(_p(x), _p(out), B, H, W, C, _st(stream)), "aotb_maxpool3x3s2_nhwc_f32")
    return out


def dwconv(x, w, bias, out, K=5, stride=1, pad=2, dil=1, act=ACT_NONE, stream=None):
    """x [B,H,W,C], w [K*K, C]."""
    _chk(x, w, bias, out)
    B, H, W, C = x.shape
    check(lib().aotb_dwconv_nhwc_f32(_p(x), _p(w), _p(bias), _p(out), B, H, W, C, _nhwc_ld(x), _nhwc_ld(out), K, K,
                                     stride, pad, dil, act, _st(stream)), "aotb_dwconv_nhwc_f32")
    return out


def bilinear(x, out, align_corners, stream=None):
    _chk(x, out)
    B, H, W, C = x.shape
    check(lib().aotb_bilinear_nhwc_f32(_p(x), _p(out), B, H, W, C, out.shape[1], out.shape[2],
                                       1 if align_corners else 0, _st(stream)), "aotb_bilinear_nhwc_f32")
    return out


def eltwise(op, a, b, out, scalar=0.0, stream=None):
    """2-D strided element-wise op on [rows, cols] views."""
    _chk(a, b, out)
    rows, cols = out.shape
    check(lib().aotb_eltwise_f32(op, _p(a), a.stride(0) if a is not None else 0, _p(b),
                                 b.stride(0) if b is not None else 0, _p(out), out.stride(0), rows, cols,
                                 float(scalar), _st(stream)), "aotb_eltwise_f32")
    return out


def layernorm(x, gamma, beta, out, add=None, out2=None, stream=None):
    _chk(x, gamma, beta, out, add, out2)
    rows, C = x.shape
    check(lib().aotb_layernorm_f32(_p(x), x.stride(0), _p(gamma), _p(beta), _p(add),
                                   add.stride(0) if add is not None else 0, _p(out), out.stride(0), _p(out2),
                                   out2.stride(0) if out2 is not None else 0, rows, C, _st(stream)),
          "aotb_layernorm_f32")
    return out


def window_attention(qkv, qkv_bias, rel_bias, out, H, W, heads, shift, window=7, stream=None, B=1):
    """Swin (S)W-MSA core: qkv [B*H*W, 3C], qkv_bias [3C], rel_bias [heads, 49, 49], out [B*H*W, C] (B token maps stacked,
    each padded, shifted and cropped on its own)."""
    _chk(qkv, qkv_bias, rel_bias, out)
    C = out.shape[1]
    if qkv.shape[0] != B * H * W or qkv.shape[1] != 3 * C or out.shape[0] != B * H * W:
        raise AotbError("window_attention: qkv must be [B*H*W, 3C], out [B*H*W, C]")
    # the kernel reads rel_bias[head][i][j] and qkv_bias[2C + head * head_dim + c] densely
    T = window * window
    if tuple(rel_bias.shape) != (heads, T, T) or not rel_bias.is_contiguous():
        raise AotbError(f"window_attention: rel_bias must be contiguous [{heads}, {T}, {T}], got {tuple(rel_bias.shape)}")
    if qkv_bias.numel() != 3 * C or not qkv_bias.is_contiguous():
        raise AotbError(f"window_attention: qkv_bias must be contiguous with {3 * C} elements, got {qkv_bias.numel()}")
    check(lib().aotb_window_attention_batched_f32(_p(qkv), qkv.stride(0), _p(qkv_bias), _p(rel_bias), _p(out), out.stride(0),
                                                  B, H, W, C, heads, window, shift, _st(stream)), "aotb_window_attention_f32")
    return out


def patch_merge(x, out, H, W, stream=None, B=1):
    """x [B*H*W, C] -> out [B*ceil(H/2)*ceil(W/2), 4C] (PatchMerging gather per map)."""
    _chk(x, out)
    C = x.shape[1]
    if x.shape[0] != B * H * W or out.shape[0] != B * ((H + 1) // 2) * ((W + 1) // 2) or out.shape[1] != 4 * C:
        raise AotbError("patch_merge: shape mismatch")
    check(lib().aotb_patch_merge_batched_f32(_p(x), x.stride(0), _p(out), out.stride(0), B, H, W, C, _st(stream)),
          "aotb_patch_merge_f32")
    return out


def groupnorm_workspace(B, G, device):
    n = lib().aotb_groupnorm_workspace_bytes(B, G)
    return torch.zeros((n + 7) // 8, dtype=torch.float64, device=device)      # zero: the launch counter lives in it


def groupnorm(x, gamma, beta, out, G, act, workspace, stream=None):
    """x/out [B, P, C] (any NHWC flattened over pixels)."""
    _chk(x, gamma, beta, out)
    B, P, C = x.shape
    check(lib().aotb_groupnorm_nhwc_f32(_p(x), x.stride(1), _p(gamma), _p(beta), _p(out), out.stride(1), B, P, C, G,
                                        act, workspace.data_ptr(), _st(stream)), "aotb_groupnorm_nhwc_f32")
    return out


def splat_workspace(C, device, B=1):
    """Workspace of splat_attention / se_gate over C channels and up to B images per launch."""
    n = lib().aotb_splat_workspace_batched_bytes(C, B)
    return torch.zeros((n + 7) // 8, dtype=torch.float64, device=device)      # zero: the launch counters live in it


def _splat_rows(x):
    """x [B,H,W,C'] NHWC or [HW, C'] (one image) -> (B, pixels per image, row stride)."""
    if x.dim() == 4:
        return x.shape[0], x.shape[1] * x.shape[2], _nhwc_ld(x)
    return 1, x.shape[0], x.stride(0)


def _check_workspace(name, workspace, C, B):
    need = lib().aotb_splat_workspace_batched_bytes(C, B)
    if workspace.numel() * workspace.element_size() < need:
        raise AotbError(f"{name}: workspace of {workspace.numel() * workspace.element_size()} bytes, {B} images of {C} "
                        f"channels need {need} (splat_workspace(C, device, B))")


def splat_attention(x, w1, b1, w2, b2, att, workspace, radix=2, stream=None):
    """ResNeSt split attention per image: x [B,H,W,radix*C] NHWC (or [HW, radix*C] for one image), w1 [C, inter],
    b1 [inter], w2 [inter, radix*C], b2 [radix*C] -> att [B, radix*C] (or [radix*C]; radix-major).  `workspace` comes
    from splat_workspace(>= C, device, >= B)."""
    _chk(x, w1, b1, w2, b2, att)
    B, HW, ld = _splat_rows(x)
    C, inter = w1.shape
    if w2.shape != (inter, radix * C) or b1.numel() != inter or b2.numel() != radix * C or att.numel() != B * radix * C \
            or x.shape[-1] < radix * C or not (w1.is_contiguous() and w2.is_contiguous() and att.is_contiguous()):
        raise AotbError("splat_attention: shapes x [.., >= radix*C], w1 [C, inter], w2 [inter, radix*C], att [B, radix*C]")
    _check_workspace("splat_attention", workspace, C, B)
    check(lib().aotb_splat_attention_batched_f32(_p(x), ld, B, HW, C, radix, _p(w1), _p(b1), inter, _p(w2), _p(b2), _p(att),
                                                 workspace.data_ptr(), _st(stream)), "aotb_splat_attention_f32")
    return att


def splat_combine(x, att, out, radix=2, pool_stride=0, stream=None):
    """x [B,H,W,radix*C], att [B, radix*C] -> out [B,Ho,Wo,C] = sum_r att_r * x_r per image, avg-pooled 3x3 / pool_stride /
    pad 1 if pool_stride > 0."""
    _chk(x, att, out)
    B, H, W, _ = x.shape
    C = out.shape[3]
    Ho, Wo = (pool2d_size(H, 3, pool_stride, 1), pool2d_size(W, 3, pool_stride, 1)) if pool_stride else (H, W)
    if att.numel() != B * radix * C or x.shape[3] < radix * C or tuple(out.shape[:3]) != (B, Ho, Wo):
        raise AotbError(f"splat_combine: x {tuple(x.shape)}, att {tuple(att.shape)}, out {tuple(out.shape)}")
    check(lib().aotb_splat_combine_batched_f32(_p(x), _nhwc_ld(x), _p(att), _p(out), _nhwc_ld(out), B, H, W, C, radix,
                                               int(pool_stride), _st(stream)), "aotb_splat_combine_f32")
    return out


def se_gate(x, w1, b1, w2, b2, gate, workspace, stream=None):
    """Squeeze-excite gate per image: x [B,H,W,C] NHWC (or [HW, C] for one image), w1 [C, inter], b1 [inter], w2 [inter, C],
    b2 [C] -> gate [B, C] (or [C]) = h_sigmoid(ReLU(mean(x) @ w1 + b1) @ w2 + b2).  `workspace` comes from
    splat_workspace(>= C, device, >= B)."""
    _chk(x, w1, b1, w2, b2, gate)
    B, HW, ld = _splat_rows(x)
    C, inter = w1.shape
    if w2.shape != (inter, C) or b1.numel() != inter or b2.numel() != C or gate.numel() != B * C or x.shape[-1] != C \
            or not (w1.is_contiguous() and w2.is_contiguous() and gate.is_contiguous()):
        raise AotbError("se_gate: shapes x [.., C], w1 [C, inter], w2 [inter, C], gate [B, C]")
    _check_workspace("se_gate", workspace, C, B)
    check(lib().aotb_se_gate_batched_f32(_p(x), ld, B, HW, C, _p(w1), _p(b1), inter, _p(w2), _p(b2), _p(gate),
                                         workspace.data_ptr(), _st(stream)), "aotb_se_gate_f32")
    return gate


def gate_scale(x, gate, out, act=ACT_NONE, stream=None):
    """out [B,H,W,C] = act(gate[b, c] * x [B,H,W,C]); x / out may be channel slices."""
    _chk(x, gate, out)
    B, H, W, C = x.shape
    if tuple(out.shape) != (B, H, W, C) or gate.numel() != B * C:
        raise AotbError(f"gate_scale: x {tuple(x.shape)}, gate {tuple(gate.shape)}, out {tuple(out.shape)}")
    check(lib().aotb_gate_scale_batched_f32(_p(x), _nhwc_ld(x), _p(gate), _p(out), _nhwc_ld(out), B, H * W, C, int(act),
                                            _st(stream)), "aotb_gate_scale_f32")
    return out


def pool2d_size(n, k, s, pad=0, ceil_mode=False):
    """Output extent of nn.AvgPool2d / nn.MaxPool2d (dilation 1) along one axis, PyTorch's rule."""
    o = (n + 2 * pad - k + (s - 1 if ceil_mode else 0)) // s + 1
    if ceil_mode and (o - 1) * s >= n + pad:
        o -= 1
    return o


def avgpool(x, out, k, s, pad=0, ceil_mode=False, count_include_pad=True, stream=None):
    """nn.AvgPool2d(k, s, pad, ceil_mode, count_include_pad) on x [B,H,W,C] -> out [B,Ho,Wo,C]."""
    _chk(x, out)
    B, H, W, C = x.shape
    if tuple(out.shape) != (B, pool2d_size(H, k, s, pad, ceil_mode), pool2d_size(W, k, s, pad, ceil_mode), C):
        raise AotbError(f"avgpool: out {tuple(out.shape)} does not match x {tuple(x.shape)} pooled ({k}, {s}, {pad})")
    check(lib().aotb_avgpool_nhwc_f32(_p(x), _nhwc_ld(x), _p(out), _nhwc_ld(out), B, H, W, C, k, s, pad, 1 if ceil_mode else 0,
                                      1 if count_include_pad else 0, _st(stream)), "aotb_avgpool_nhwc_f32")
    return out


def attention(Q, K, V, O, H, d_qk, d_v, Tk=None, Tk_dev=None, Mout=None, Lout=None, stream=None):
    """Q [N, H*d_qk], K [>=Tk, H*d_qk], V [>=Tk, H*d_v], O [N, H*d_v]."""
    _chk(Q, K, V, O, Mout, Lout)
    N = Q.shape[0]
    tk = K.shape[0] if Tk is None else int(Tk)
    check(lib().aotb_attention_f32(_p(Q), Q.stride(0), _p(K), K.stride(0), _p(V), V.stride(0), _p(O), O.stride(0),
                                   N, tk, Tk_dev.data_ptr() if Tk_dev is not None else None, H, d_qk, d_v,
                                   _p(Mout), _p(Lout), _st(stream)), "aotb_attention_f32")
    return O


def attn_merge(Opart, Mpart, Lpart, O, H, d_v, stream=None):
    _chk(Opart, Mpart, Lpart, O)
    R, N = Opart.shape[0], Opart.shape[1]
    check(lib().aotb_attn_merge_f32(_p(Opart), _p(Mpart), _p(Lpart), _p(O), R, N, H, d_v, O.stride(0), _st(stream)),
          "aotb_attn_merge_f32")
    return O


def attn_merge_usage_workspace(R, device):
    """Zero-filled workspace of attn_merge_usage for up to R slots (its launch counter must start at zero)."""
    n = int(lib().aotb_attn_merge_usage_workspace_bytes(int(R)))
    return torch.zeros((n + 7) // 8, dtype=torch.float64, device=device)


def attn_merge_usage(Opart, Mpart, Lpart, O, H, d_v, U, A, live_dev, rows, layers, workspace, stream=None):
    """attn_merge over the R memory slots of a bounded bank (split r = slot r) that also adds each slot's attention mass,
    averaged over (query, head) and divided by `layers`, into U (float32 [R]); A (int32 [R] or None) gets the age tick
    A[r] += 1 for every live slot r < *live_dev / rows."""
    _chk(Opart, Mpart, Lpart, O, U)
    R, N = Opart.shape[0], Opart.shape[1]
    if U.numel() != R or not U.is_contiguous() or (A is not None and (A.dtype != torch.int32 or A.numel() != R or
                                                                      not A.is_cuda)):
        raise AotbError(f"attn_merge_usage: U must be float32 [{R}] and A int32 [{R}] CUDA tensors")
    check(lib().aotb_attn_merge_usage_f32(_p(Opart), _p(Mpart), _p(Lpart), _p(O), R, N, H, d_v, O.stride(0), _p(U), _p(A),
                                          _counter("attn_merge_usage: live_dev", live_dev) if A is not None else None,
                                          int(rows), int(layers), workspace.data_ptr(), _st(stream)),
          "aotb_attn_merge_usage_f32")
    return O


def attn_merge_peers(Oparts, Mparts, Lparts, O, splits, H, d_v, stream=None):
    """Merge split-KV partials that live in `len(Oparts)` ranks' buffers (local tensor + peer views of a symmetric-memory
    allocation): Oparts[r] [>=splits, N, H*d_v], Mparts[r] / Lparts[r] [>=splits, H, N]."""
    import ctypes
    _chk(O, *Oparts, *Mparts, *Lparts)
    R, N = len(Oparts), O.shape[0]
    arr = lambda ts: (ctypes.c_void_p * R)(*[t.data_ptr() for t in ts])
    check(lib().aotb_attn_merge_peers_f32(arr(Oparts), arr(Mparts), arr(Lparts), R, int(splits), _p(O), N, H, d_v,
                                          O.stride(0), _st(stream)), "aotb_attn_merge_peers_f32")
    return O


def local_attention(q, k, v, relk_w, relk_b, relv, out, h, w, H, d_att, d_v, stream=None):
    """q,k [hw, H*d_att], v [hw, H*d_v], out [hw, H*d_v]."""
    _chk(q, k, v, relk_w, relk_b, relv, out)
    check(lib().aotb_local_attention_f32(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(relk_w),
                                         _p(relk_b), _p(relv), _p(out), out.stride(0), h, w, H, d_att, d_v,
                                         _st(stream)), "aotb_local_attention_f32")
    return out


def local_gated_tile(q, k, v, relk_w, relk_b, out, h, w, stream=None):
    """DeAOT head shape (1 x 128 / 1024, no relative_emb_v): halo-in-shared-memory kernel; q, k [hw, 128], v / out [hw, 1024]."""
    _chk(q, k, v, relk_w, relk_b, out)
    if q.shape[1] != 128 or k.shape[1] != 128 or v.shape[1] != 1024 or out.shape[1] != 1024 or not relk_w.is_contiguous():
        raise AotbError("local_gated_tile: q / k [hw, 128], v / out [hw, 1024], contiguous relative_emb_k weights [225, 128]")
    check(lib().aotb_local_gated_tile_f32(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(relk_w), _p(relk_b),
                                          _p(out), out.stride(0), h, w, _st(stream)), "aotb_local_gated_tile_f32")
    return out


LOCAL_KERNELS = ("tile", "tc")
# kernel behind local_attention_tile: "tile" = the fp32 CUDA-core tile kernel, "tc" = the tensor-core kernel of
# local_attention_tc.  Outside `local_kernel` it is the CUDA-core kernel; the engines select theirs around their call, so
# the AOT short-term attention has one entry point whichever kernel runs.
_LOCAL_KERNEL = "tile"


@contextlib.contextmanager
def local_kernel(k):
    """Run the local_attention_tile calls of the enclosed code on kernel `k` ("tile" | "tc")."""
    global _LOCAL_KERNEL
    if k not in LOCAL_KERNELS:
        raise ValueError(f"local kernel must be one of {LOCAL_KERNELS}, got {k!r}")
    old, _LOCAL_KERNEL = _LOCAL_KERNEL, k
    try:
        yield
    finally:
        _LOCAL_KERNEL = old


def local_attention_tile(q, k, v, relk_w, relk_b, relv_t, out, h, w, H, stream=None):
    """AOT head shape (d = 32): halo-in-shared-memory kernel; relv_t [H, 225, 32].  Inside local_kernel("tc"), the
    tensor-core kernel (local_attention_tc)."""
    if _LOCAL_KERNEL == "tc":
        return local_attention_tc(q, k, v, relk_w, relk_b, relv_t, out, h, w, H, stream=stream)
    _chk(q, k, v, relk_w, relk_b, relv_t, out)
    check(lib().aotb_local_attention_tile_f32(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(relk_w),
                                              _p(relk_b), _p(relv_t), _p(out), out.stride(0), h, w, H, _st(stream)),
          "aotb_local_attention_tile_f32")
    return out


def local_attention_tc(q, k, v, relk_w, relk_b, relv_t, out, h, w, H, stream=None):
    """AOT head shape (d = 32) on the tensor cores, split fp16x2; the arguments of local_attention_tile."""
    _chk(q, k, v, relk_w, relk_b, relv_t, out)
    check(lib().aotb_local_attention_tc_f32(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(relk_w),
                                            _p(relk_b), _p(relv_t), _p(out), out.stride(0), h, w, H, _st(stream)),
          "aotb_local_attention_tc_f32")
    return out


def _id_embed_check(name, mask, table, table_shape, bias, out, C, ksize, stride, pad, ln_gamma, ln_beta):
    """The mask is read as a dense [Hm, Wm] map and the weight table as a dense array of `table_shape`; out [ho*wo, C] may
    have a row stride above C.  -> (Hm, Wm)."""
    _chk(mask, table, bias, out, ln_gamma, ln_beta)
    if mask.dim() != 2 or not mask.is_contiguous():
        raise AotbError(f"{name}: mask must be a contiguous [Hm, Wm] map, got shape {tuple(mask.shape)}, "
                        f"strides {mask.stride()}")
    Hm, Wm = mask.shape
    ho, wo = (Hm + 2 * pad - ksize) // stride + 1, (Wm + 2 * pad - ksize) // stride + 1
    if tuple(table.shape) != tuple(table_shape) or not table.is_contiguous():
        raise AotbError(f"{name}: weight table must be a contiguous {list(table_shape)}, got {tuple(table.shape)}")
    if bias.numel() != C or any(t is not None and t.numel() != C for t in (ln_gamma, ln_beta)):
        raise AotbError(f"{name}: bias and LayerNorm parameters need {C} entries")
    if out.dim() != 2 or tuple(out.shape) != (ho * wo, C):
        raise AotbError(f"{name}: out must be [{ho * wo}, {C}] for a {Hm}x{Wm} mask, got {tuple(out.shape)}")
    return Hm, Wm


def id_embed(mask, wt, bias, out, C, nid, ksize, stride, pad, ln_gamma=None, ln_beta=None, stream=None):
    """mask [Hm, Wm] float ids (contiguous) -> out [ho*wo, C]; wt [ksize*ksize*nid, C]."""
    Hm, Wm = _id_embed_check("id_embed", mask, wt, (ksize * ksize * nid, C), bias, out, C, ksize, stride, pad, ln_gamma,
                             ln_beta)
    check(lib().aotb_id_embed_f32(_p(mask), Hm, Wm, _p(wt), _p(bias), _p(ln_gamma), _p(ln_beta), _p(out),
                                  out.stride(0), C, nid, ksize, stride, pad, _st(stream)), "aotb_id_embed_f32")
    return out


def id_embed_runs(mask, wp, bias, out, C, nid, ksize, stride, pad, ln_gamma=None, ln_beta=None, stream=None):
    """Run-length form of id_embed; wp [ksize, ksize+1, nid, C] exclusive prefix sums along kx."""
    Hm, Wm = _id_embed_check("id_embed_runs", mask, wp, (ksize, ksize + 1, nid, C), bias, out, C, ksize, stride, pad,
                             ln_gamma, ln_beta)
    check(lib().aotb_id_embed_runs_f32(_p(mask), Hm, Wm, _p(wp), _p(bias), _p(ln_gamma), _p(ln_beta), _p(out),
                                       out.stride(0), C, nid, ksize, stride, pad, _st(stream)), "aotb_id_embed_runs_f32")
    return out


def _dense_maps(name, t, shape3):
    """t must be one contiguous [..., a, b, c] map (leading dims of size 1) with the given trailing shape (None: any)."""
    if t.dim() < 3 or t.numel() != t.shape[-3] * t.shape[-2] * t.shape[-1] or not t.is_contiguous() \
            or any(want is not None and got != want for got, want in zip(t.shape[-3:], shape3)):
        want = "x".join("*" if v is None else str(v) for v in shape3)
        raise AotbError(f"{name}: need one contiguous [{want}] map, got shape {tuple(t.shape)}, strides {t.stride()}")


def logits_postproc(logits_nhwc, lowres_nchw, out_nchw, obj_num, align_corners, stream=None):
    """logits_nhwc [h, w, NC] -> lowres_nchw [NC, h, w] (ids > obj_num set to -1e10) and, if given, out_nchw [NC, Ho, Wo]
    bilinearly upsampled; all three contiguous (leading dims of size 1)."""
    _chk(logits_nhwc, lowres_nchw, out_nchw)
    _dense_maps("logits_postproc logits", logits_nhwc, (None, None, None))
    h, w, NC = logits_nhwc.shape[-3:]
    _dense_maps("logits_postproc lowres", lowres_nchw, (NC, h, w))
    if out_nchw is not None:
        _dense_maps("logits_postproc out", out_nchw, (NC, None, None))
    Ho, Wo = (out_nchw.shape[-2], out_nchw.shape[-1]) if out_nchw is not None else (0, 0)
    check(lib().aotb_logits_postproc_f32(_p(logits_nhwc), _p(lowres_nchw), _p(out_nchw), h, w, NC, obj_num, Ho, Wo,
                                         1 if align_corners else 0, _st(stream)), "aotb_logits_postproc_f32")
    return out_nchw


def logits_argmax(lowres_nchw, label, align_corners, stream=None):
    """lowres_nchw [NC, h, w] -> label [Ho, Wo] = argmax over NC of the bilinear upsample; both contiguous."""
    _chk(lowres_nchw, label)
    _dense_maps("logits_argmax lowres", lowres_nchw, (None, None, None))
    NC, h, w = lowres_nchw.shape[-3:]
    Ho, Wo = label.shape[-2:]
    if label.numel() != Ho * Wo or not label.is_contiguous():
        raise AotbError(f"logits_argmax: label must be one contiguous [Ho, Wo] map, got {tuple(label.shape)}")
    check(lib().aotb_logits_argmax_f32(_p(lowres_nchw), _p(label), h, w, NC, Ho, Wo, 1 if align_corners else 0,
                                       _st(stream)), "aotb_logits_argmax_f32")
    return label


def soft_logit_aggregation(logits, out, max_obj, stream=None):
    """logits: list of E contiguous NCHW maps [1, 1 + max_obj, H, W]; out [1, 1 + E * max_obj, H, W]."""
    import ctypes
    _chk(out, *logits)
    E = len(logits)
    HW = out.shape[-2] * out.shape[-1]
    for t in logits:
        if not t.is_contiguous() or t.shape[1] != 1 + max_obj or t.shape[-2] * t.shape[-1] != HW:
            raise AotbError("soft_logit_aggregation: logit maps must be contiguous [1, 1 + max_obj, H, W] of one size")
    if not out.is_contiguous() or out.shape[1] != 1 + E * max_obj:
        raise AotbError("soft_logit_aggregation: out must be contiguous [1, 1 + E * max_obj, H, W]")
    arr = (ctypes.c_void_p * E)(*[t.data_ptr() for t in logits])
    check(lib().aotb_soft_logit_aggregation_f32(arr, E, int(max_obj), _p(out), HW, _st(stream)),
          "aotb_soft_logit_aggregation_f32")
    return out


def tta_merge(logits, flips, label, align_corners, new_label=None, prob=None, stream=None):
    """Test-time augmentation ensemble: logits = list of E (1..8) contiguous maps [NC, h_e, w_e] (leading dims of size 1, one
    NC for all), flips = E bools; label [H, W] = first argmax of the mean softmax of the bilinear upsamples (flipped ones read
    mirrored), overwritten by new_label [H, W] where that is nonzero; prob [NC, H, W] receives the mean probabilities."""
    import ctypes
    _chk(label, new_label, prob, *logits)
    E = len(logits)
    if not 1 <= E <= 8 or len(flips) != E:
        raise AotbError(f"tta_merge: 1 to 8 logit maps with one flip bit each, got {E} maps and {len(flips)} flips")
    for t in logits:
        _dense_maps("tta_merge logits", t, (logits[0].shape[-3], None, None))
    NC = int(logits[0].shape[-3])
    H, W = label.shape[-2:]
    for name, t in (("label", label), ("new_label", new_label)):
        if t is not None and (t.numel() != H * W or not t.is_contiguous() or tuple(t.shape[-2:]) != (H, W)):
            raise AotbError(f"tta_merge: {name} must be one contiguous [{H}, {W}] map, got {tuple(t.shape)}")
    if prob is not None:
        _dense_maps("tta_merge prob", prob, (NC, H, W))
    arr = (ctypes.c_void_p * E)(*[t.data_ptr() for t in logits])
    sizes = (ctypes.c_int * (2 * E))(*[int(v) for t in logits for v in t.shape[-2:]])
    fl = (ctypes.c_int * E)(*[1 if f else 0 for f in flips])
    check(lib().aotb_tta_merge_f32(arr, sizes, fl, E, NC, H, W, 1 if align_corners else 0, _p(new_label), _p(label), _p(prob),
                                   _st(stream)), "aotb_tta_merge_f32")
    return label


def tta_feedback(logits, out, output_size, align_corners, flip, new_label=None, stream=None):
    """One augmentation's memory label: out [Hi, Wi] = nearest resize from output_size (H, W) of (new_label mirrored if flip,
    where nonzero, else argmax softmax of the bilinear upsample of logits [NC, h, w] to (H, W)).  logits None: background (the
    first frame's form); new_label None: no new objects."""
    _chk(logits, out, new_label)
    H, W = int(output_size[0]), int(output_size[1])
    Hi, Wi = out.shape[-2:]
    if out.numel() != Hi * Wi or not out.is_contiguous():
        raise AotbError(f"tta_feedback: out must be one contiguous [Hi, Wi] map, got {tuple(out.shape)}")
    if new_label is not None and (new_label.numel() != H * W or not new_label.is_contiguous()
                                  or tuple(new_label.shape[-2:]) != (H, W)):
        raise AotbError(f"tta_feedback: new_label must be one contiguous [{H}, {W}] map, got {tuple(new_label.shape)}")
    NC, h, w = 0, 0, 0
    if logits is not None:
        _dense_maps("tta_feedback logits", logits, (None, None, None))
        NC, h, w = (int(v) for v in logits.shape[-3:])
    check(lib().aotb_tta_feedback_f32(_p(logits), h, w, NC, H, W, 1 if align_corners else 0, 1 if flip else 0, _p(new_label),
                                      _p(out), Hi, Wi, _st(stream)), "aotb_tta_feedback_f32")
    return out


def _label_maps(name, ts, n, H, W):
    """n optional contiguous [H, W] maps -> a ctypes pointer array (None when every entry is None)."""
    import ctypes
    if ts is None or all(t is None for t in ts):
        return None
    if len(ts) != n:
        raise AotbError(f"{name}: one entry per map, got {len(ts)} for {n}")
    for t in ts:
        _chk(t)
        if t is not None and (t.numel() != H * W or not t.is_contiguous() or tuple(t.shape[-2:]) != (H, W)):
            raise AotbError(f"{name}: each map must be one contiguous [{H}, {W}] map, got {tuple(t.shape)}")
    return (ctypes.c_void_p * n)(*[_p(t) for t in ts])


def tta_merge_batched(logits, flips, lanes, obj_nums, label, align_corners, new_labels=None, prob=None, stream=None):
    """tta_merge over n videos in one launch, reading the multi-video decoders' outputs directly.  logits = E (1..8) NHWC maps
    [lanes_e, h_e, w_e, NC] (one NC); lanes [n][E]: video b's lane in each map; obj_nums [n]: ids above obj_nums[b] are masked
    as logits_postproc masks them; label [n, H, W] (leading dims of size 1 allowed between); prob [n, NC, H, W] or None;
    new_labels: n [H, W] overlays or None entries.  Video b's label and probabilities are bit for bit logits_postproc +
    tta_merge on its lanes."""
    import ctypes
    _chk(label, prob, *logits)
    E, n = len(logits), len(lanes)
    if not 1 <= E <= 8 or len(flips) != E:
        raise AotbError(f"tta_merge_batched: 1 to 8 logit maps with one flip bit each, got {E} maps and {len(flips)} flips")
    if n < 1 or len(obj_nums) != n or any(len(r) != E for r in lanes):
        raise AotbError(f"tta_merge_batched: lanes [n][{E}] and obj_nums [n] for n >= 1 videos")
    NC = int(logits[0].shape[-1])
    for e, t in enumerate(logits):
        if t.dim() != 4 or not t.is_contiguous() or t.shape[-1] != NC:
            raise AotbError(f"tta_merge_batched: logits must be contiguous NHWC [lanes, h, w, {NC}], got {tuple(t.shape)}")
        if any(not 0 <= r[e] < t.shape[0] for r in lanes):
            raise AotbError(f"tta_merge_batched: augmentation {e}: lane out of [0, {t.shape[0]})")
    H, W = label.shape[-2:]
    if label.numel() != n * H * W or not label.is_contiguous():
        raise AotbError(f"tta_merge_batched: label must be contiguous [{n}, {H}, {W}], got {tuple(label.shape)}")
    if prob is not None and (prob.numel() != n * NC * H * W or not prob.is_contiguous() or tuple(prob.shape[-3:]) != (NC, H, W)):
        raise AotbError(f"tta_merge_batched: prob must be contiguous [{n}, {NC}, {H}, {W}], got {tuple(prob.shape)}")
    arr = (ctypes.c_void_p * E)(*[t.data_ptr() for t in logits])
    sizes = (ctypes.c_int * (2 * E))(*[int(v) for t in logits for v in t.shape[1:3]])
    fl = (ctypes.c_int * E)(*[1 if f else 0 for f in flips])
    ln = (ctypes.c_int * (n * E))(*[int(v) for r in lanes for v in r])
    ob = (ctypes.c_int * n)(*[int(v) for v in obj_nums])
    nl = _label_maps("tta_merge_batched new_labels", new_labels, n, H, W)
    check(lib().aotb_tta_merge_batched_f32(arr, sizes, fl, E, ln, ob, n, NC, H, W, 1 if align_corners else 0, nl, _p(label),
                                           _p(prob), _st(stream)), "aotb_tta_merge_batched_f32")
    return label


def tta_feedback_batched(logits, out, obj_nums, flips, output_size, align_corners, new_labels=None, stream=None):
    """tta_feedback over the first len(flips) lanes of one multi-video decoder's output in one launch.  logits [lanes, h, w, NC]
    (NHWC, lane k masked at obj_nums[k] as logits_postproc masks it) or None (background for every lane); out [>= n, Hi, Wi]
    contiguous, lane k written to out[k]; new_labels: n [H, W] maps or None entries, at output_size.  Lane k's map is bit for
    bit logits_postproc + tta_feedback on lane k."""
    import ctypes
    _chk(logits, out)
    n = len(flips)
    H, W = int(output_size[0]), int(output_size[1])
    Hi, Wi = out.shape[-2:]
    if n < 1 or not out.is_contiguous() or out.numel() < n * Hi * Wi:
        raise AotbError(f"tta_feedback_batched: out must be contiguous [>= {n}, Hi, Wi], got {tuple(out.shape)}")
    h = w = NC = 0
    ob = None
    if logits is not None:
        if logits.dim() != 4 or not logits.is_contiguous() or logits.shape[0] < n:
            raise AotbError(f"tta_feedback_batched: logits must be contiguous NHWC [>= {n}, h, w, NC], got "
                            f"{tuple(logits.shape)}")
        if obj_nums is None or len(obj_nums) != n:
            raise AotbError(f"tta_feedback_batched: one object count per lane, got {obj_nums}")
        h, w, NC = (int(v) for v in logits.shape[1:])
        ob = (ctypes.c_int * n)(*[int(v) for v in obj_nums])
    fl = (ctypes.c_int * n)(*[1 if f else 0 for f in flips])
    nl = _label_maps("tta_feedback_batched new_labels", new_labels, n, H, W)
    check(lib().aotb_tta_feedback_batched_f32(_p(logits), h, w, NC, n, ob, fl, nl, H, W, 1 if align_corners else 0, _p(out),
                                              Hi, Wi, _st(stream)), "aotb_tta_feedback_batched_f32")
    return out


def separate_labels(mask, out, max_obj, stream=None):
    """mask: contiguous label map with HW elements; out [E, ...HW...] receives the per-engine renumbered label maps."""
    _chk(mask, out)
    E, HW = out.shape[0], mask.numel()
    if not mask.is_contiguous() or not out.is_contiguous() or out.numel() != E * HW:
        raise AotbError("separate_labels: mask [HW] and out [E, HW] must be contiguous")
    check(lib().aotb_separate_labels_f32(_p(mask), E, int(max_obj), _p(out), HW, _st(stream)), "aotb_separate_labels_f32")
    return out


def soft_logit_aggregation_batched(logits, lanes, obj_nums, align_corners, out=None, labels=None, max_obj=10, stream=None):
    """soft_logit_aggregation for n videos of a multi-video pool in one launch, reading its decoder output logits [lanes, h, w,
    1 + max_obj] (NHWC, contiguous) directly.  lanes [n][k_b] (1 <= k_b <= 8): video b's lanes in sub-engine order; obj_nums
    [n][k_b]: their object counts, ids above which are masked as logits_postproc masks them.  out: n contiguous maps [1 +
    k_b max_obj, Ho, Wo] (leading dims of size 1) or None; labels: n contiguous [Ho, Wo] maps or None (entries may be None, but
    not both for one video).  Video b's map is bit for bit logits_postproc (at [Ho, Wo]) on each of its lanes followed by
    soft_logit_aggregation, its label the first argmax of that map."""
    import ctypes
    n = len(lanes)
    outs = [None] * n if out is None else list(out)
    labs = [None] * n if labels is None else list(labels)
    _chk(logits, *[t for t in outs + labs if t is not None])
    if n < 1 or len(obj_nums) != n or len(outs) != n or len(labs) != n:
        raise AotbError(f"soft_logit_aggregation_batched: lanes, obj_nums, out and labels need one entry per video, got "
                        f"{n}, {len(obj_nums)}, {len(outs)}, {len(labs)}")
    if logits.dim() != 4 or not logits.is_contiguous() or logits.shape[-1] != 1 + max_obj:
        raise AotbError(f"soft_logit_aggregation_batched: logits must be contiguous NHWC [lanes, h, w, {1 + max_obj}], got "
                        f"{tuple(logits.shape)}")
    L, h, w, NC = (int(v) for v in logits.shape)
    size = None
    for b in range(n):
        k = len(lanes[b])
        if not 1 <= k <= 8 or len(obj_nums[b]) != k or any(not 0 <= int(l) < L for l in lanes[b]):
            raise AotbError(f"soft_logit_aggregation_batched: video {b}: 1 to 8 lanes in [0, {L}) with one object count each, "
                            f"got lanes {lanes[b]}, obj_nums {obj_nums[b]}")
        if outs[b] is None and labs[b] is None:
            raise AotbError(f"soft_logit_aggregation_batched: video {b}: no output")
        for t, ch in ((outs[b], 1 + k * max_obj), (labs[b], None)):
            if t is None:
                continue
            s = tuple(int(v) for v in t.shape[-2:])
            size = size or s
            lead = t.numel() // (s[0] * s[1])
            if s != size or not t.is_contiguous() or (ch is None and lead != 1) or \
                    (ch is not None and (t.dim() < 3 or t.shape[-3] != ch or lead != ch)):
                raise AotbError(f"soft_logit_aggregation_batched: video {b}: need contiguous {'label' if ch is None else ch} "
                                f"maps of one size {size}, got {tuple(t.shape)}")
    ptr = [0]
    for r in lanes:
        ptr.append(ptr[-1] + len(r))
    lp = (ctypes.c_int * (n + 1))(*ptr)
    ln = (ctypes.c_int * ptr[-1])(*[int(v) for r in lanes for v in r])
    ob = (ctypes.c_int * ptr[-1])(*[int(v) for r in obj_nums for v in r])
    op = None if out is None else (ctypes.c_void_p * n)(*[_p(t) for t in outs])
    lb = None if labels is None else (ctypes.c_void_p * n)(*[_p(t) for t in labs])
    check(lib().aotb_soft_logit_aggregation_batched_f32(_p(logits), h, w, NC, lp, ln, ob, n, int(max_obj), size[0], size[1],
                                                        1 if align_corners else 0, op, lb, _st(stream)),
          "aotb_soft_logit_aggregation_batched_f32")
    return out, labels


def separate_labels_batched(labels, parts, out, max_obj=10, stream=None):
    """separate_labels for n lanes in one launch: out[b] (contiguous, HW elements) = labels[b]'s map for sub-engine parts[b]
    (ids (parts[b] max_obj, (parts[b] + 1) max_obj] renumbered from 1, everything else 0); labels[b] contiguous fp32 with the
    same HW elements, and an entry may repeat.  Bit for bit row parts[b] of separate_labels on labels[b]."""
    import ctypes
    n = len(labels)
    _chk(*labels, *out)
    if n < 1 or len(parts) != n or len(out) != n:
        raise AotbError(f"separate_labels_batched: one part and one output per label map, got {n}, {len(parts)}, {len(out)}")
    HW = labels[0].numel()
    for t in list(labels) + list(out):
        if t.numel() != HW or not t.is_contiguous() or t.dtype != torch.float32:
            raise AotbError(f"separate_labels_batched: every map must be contiguous fp32 with {HW} elements, got "
                            f"{tuple(t.shape)} {t.dtype}")
    if any(int(p) < 0 for p in parts):
        raise AotbError(f"separate_labels_batched: negative part in {parts}")
    lb = (ctypes.c_void_p * n)(*[_p(t) for t in labels])
    op = (ctypes.c_void_p * n)(*[_p(t) for t in out])
    pt = (ctypes.c_int * n)(*[int(p) for p in parts])
    check(lib().aotb_separate_labels_batched_f32(lb, pt, n, int(max_obj), op, HW, _st(stream)),
          "aotb_separate_labels_batched_f32")
    return out


def lane_gather(src, dst, lane_video, n_lanes, stream=None):
    """Gather up to 4 per-video maps into lane order in one launch: dst[j][l] = src[j][lane_video[l]] for l < n_lanes.  src[j]
    [videos, ...] and dst[j] [>= n_lanes, ...] contiguous fp32 with one row size (a multiple of 4 floats); lane_video: int32
    device tensor [>= n_lanes] read at run time (a captured launch follows its contents), an entry outside [0, videos) copies
    nothing."""
    import ctypes
    _chk(*src, *dst)
    m = len(src)
    if not 1 <= m <= 4 or len(dst) != m:
        raise AotbError(f"lane_gather: 1 to 4 maps with one destination each, got {m} and {len(dst)}")
    if not lane_video.is_cuda or lane_video.dtype != torch.int32 or not lane_video.is_contiguous() \
            or lane_video.numel() < n_lanes or n_lanes < 1:
        raise AotbError(f"lane_gather: lane_video must be a contiguous int32 tensor of >= {n_lanes} >= 1 entries")
    nv = int(src[0].shape[0])
    rows = []
    for s, d in zip(src, dst):
        r = s[0].numel() if s.shape[0] else 0
        if s.dtype != torch.float32 or d.dtype != torch.float32 or not s.is_contiguous() or not d.is_contiguous() \
                or s.shape[0] != nv or d.shape[0] < n_lanes or d[0].numel() != r or r % 4:
            raise AotbError(f"lane_gather: need contiguous fp32 src [{nv}, ...] and dst [>= {n_lanes}, ...] with one row size "
                            f"(a multiple of 4), got {tuple(s.shape)} and {tuple(d.shape)}")
        rows.append(r)
    sp = (ctypes.c_void_p * m)(*[_p(t) for t in src])
    dp = (ctypes.c_void_p * m)(*[_p(t) for t in dst])
    nf = (ctypes.c_int * m)(*rows)
    check(lib().aotb_lane_gather_f32(sp, dp, nf, m, _p(lane_video), int(n_lanes), nv, _st(stream)), "aotb_lane_gather_f32")
    return dst


def preprocess_bgr_u8(img_u8, out, taps=None, flip=False, stream=None):
    """img_u8 uint8 [H, W, 3] (device); out fp32 [1, 3, Ho, Wo]; taps = (ix, cx, iy, cy) device tables or None (same size)."""
    if img_u8.dtype != torch.uint8 or not img_u8.is_cuda or not img_u8.is_contiguous() or img_u8.dim() != 3 or img_u8.shape[2] != 3:
        raise AotbError("preprocess_bgr_u8: image must be a contiguous uint8 CUDA tensor [H, W, 3]")
    _chk(out)
    if out.dim() != 4 or tuple(out.shape[:2]) != (1, 3) or not out.is_contiguous():   # the kernel writes 3 * Ho * Wo floats
        raise AotbError(f"preprocess_bgr_u8: out must be contiguous [1, 3, Ho, Wo], got {tuple(out.shape)}")
    H, W = int(img_u8.shape[0]), int(img_u8.shape[1])
    Ho, Wo = int(out.shape[-2]), int(out.shape[-1])
    if taps is None:
        ptrs = (None, None, None, None)
    else:
        ix, cx, iy, cy = taps
        if ix.dtype != torch.int32 or iy.dtype != torch.int32 or cx.dtype != torch.float32 or cy.dtype != torch.float32 \
                or tuple(ix.shape) != (Wo, 4) or tuple(cx.shape) != (Wo, 4) or tuple(iy.shape) != (Ho, 4) or tuple(cy.shape) != (Ho, 4):
            raise AotbError("preprocess_bgr_u8: taps must be (int32 [Wo,4], fp32 [Wo,4], int32 [Ho,4], fp32 [Ho,4])")
        if not all(t.is_cuda and t.is_contiguous() for t in taps):
            raise AotbError("preprocess_bgr_u8: tap tables must be contiguous CUDA tensors")
        ptrs = tuple(t.data_ptr() for t in (ix, cx, iy, cy))
    check(lib().aotb_preprocess_bgr_u8(img_u8.data_ptr(), H, W, ptrs[0], ptrs[1], ptrs[2], ptrs[3], _p(out), Ho, Wo,
                                       1 if flip else 0, _st(stream)), "aotb_preprocess_bgr_u8")
    return out


def label_to_u8(label, out_u8, stream=None):
    _chk(label)
    if out_u8.dtype != torch.uint8 or not out_u8.is_cuda or not out_u8.is_contiguous() or not label.is_contiguous() \
            or out_u8.numel() != label.numel():
        raise AotbError("label_to_u8: contiguous float32 label and uint8 output of the same size on the device")
    check(lib().aotb_label_to_u8(_p(label), out_u8.data_ptr(), label.numel(), _st(stream)), "aotb_label_to_u8")
    return out_u8


def nearest_resize(x, out, stream=None):
    """x [H, W] -> out [Ho, Wo] (F.interpolate(mode='nearest')); both one contiguous map (leading dims of size 1)."""
    _chk(x, out)
    H, W = x.shape[-2:]
    Ho, Wo = out.shape[-2:]
    for t, n in ((x, H * W), (out, Ho * Wo)):
        if t.numel() != n or not t.is_contiguous():
            raise AotbError(f"nearest_resize: need contiguous single maps, got {tuple(t.shape)} with strides {t.stride()}")
    check(lib().aotb_nearest_resize_f32(_p(x), _p(out), H, W, Ho, Wo, _st(stream)), "aotb_nearest_resize_f32")
    return out


def bank_append(src, bank, offset, offset_dev=None, stream=None):
    """bank[offset + r, :cols] = src[r] for the rows of src [rows, cols]; the offset is `offset` or, if given, the int32
    device counter `offset_dev` (read when the kernel runs, so only the host offset can be checked here)."""
    _chk(src, bank)
    rows, cols = src.shape
    if bank.dim() != 2 or cols > bank.shape[1] or rows > bank.shape[0] or \
            (offset_dev is None and not 0 <= int(offset) <= bank.shape[0] - rows):
        raise AotbError(f"bank_append: {rows} x {cols} rows at offset {int(offset) if offset_dev is None else 'on device'} "
                        f"do not fit a bank of {tuple(bank.shape)}")
    check(lib().aotb_bank_append_f32(_p(src), src.stride(0), _p(bank), bank.stride(0), rows, cols, int(offset),
                                     offset_dev.data_ptr() if offset_dev is not None else None, _st(stream)),
          "aotb_bank_append_f32")
    return bank


def counter_add(counter, delta, stream=None):
    """counter: int32 CUDA tensor [1]; *counter += delta on the stream (bank row counter)."""
    if not counter.is_cuda or counter.dtype != torch.int32:
        raise AotbError("counter must be an int32 CUDA tensor")
    check(lib().aotb_counter_add(counter.data_ptr(), int(delta), _st(stream)), "aotb_counter_add")
    return counter


def _counter(name, c):
    if c is None or not c.is_cuda or c.dtype != torch.int32 or c.numel() != 1:
        raise AotbError(f"{name} must be an int32 CUDA tensor [1]")
    return c.data_ptr()


def bank_ring_store(k_src, v_src, k_bank, v_bank, k_packed, v_packed, write_dev, stream=None):
    """Bounded bank: store one memory frame's k_src [rows, Ck] / v_src [rows, Cv] at row `*write_dev` of every copy given:
    the fp32 banks k_bank [cap, >= Ck] / v_bank [cap, >= Cv] and the packed fp16 banks k_packed [Ck/32, cap, 64] / v_packed
    [Cv/32, cap, 64] (the rows tc_pack_rows writes); a copy that is None is skipped.  All copies share one capacity."""
    _chk(k_src, v_src, k_bank, v_bank)
    if k_src.dim() != 2 or v_src.dim() != 2 or k_src.shape[0] != v_src.shape[0]:
        raise AotbError("bank_ring_store: k_src and v_src must be [rows, C] with the same rows")
    rows = k_src.shape[0]
    caps = set()
    for name, src, bank, packed in (("k", k_src, k_bank, k_packed), ("v", v_src, v_bank, v_packed)):
        cols = src.shape[1]
        if bank is not None:
            if bank.dim() != 2 or bank.shape[1] < cols:
                raise AotbError(f"bank_ring_store: {name}_bank {tuple(bank.shape)} is narrower than the {cols} source channels")
            caps.add(bank.shape[0])
        if packed is not None:
            if packed.dtype != torch.float16 or not packed.is_cuda or not packed.is_contiguous() or packed.dim() != 3 or \
                    packed.shape[2] != 64 or packed.shape[0] * 32 != cols:
                raise AotbError(f"bank_ring_store: {name}_packed must be a contiguous fp16 CUDA tensor [{cols} / 32, cap, 64]")
            caps.add(packed.shape[1])
    if len(caps) != 1 or rows > min(caps):
        raise AotbError(f"bank_ring_store: the copies need one capacity of at least {rows} rows, got {sorted(caps)}")
    check(lib().aotb_bank_ring_store(_p(k_src), k_src.stride(0), k_src.shape[1], _p(v_src), v_src.stride(0), v_src.shape[1],
                                     rows, _p(k_bank), k_bank.stride(0) if k_bank is not None else 0, _p(v_bank),
                                     v_bank.stride(0) if v_bank is not None else 0, _p(k_packed), _p(v_packed), caps.pop(),
                                     _counter("bank_ring_store: write_dev", write_dev), _st(stream)), "aotb_bank_ring_store")


def ring_advance(live_dev, write_dev, rows, cap_rows, pinned_rows, stream=None):
    """Bounded bank, after a store of `rows` rows: *live_dev = min(*live_dev + rows, cap_rows); *write_dev moves on by `rows`
    and wraps to `pinned_rows` when the next store would pass `cap_rows` (both int32 CUDA tensors [1])."""
    check(lib().aotb_ring_advance(_counter("ring_advance: live_dev", live_dev), _counter("ring_advance: write_dev", write_dev),
                                  int(rows), int(cap_rows), int(pinned_rows), _st(stream)), "aotb_ring_advance")


def ring_select_usage(live_dev, write_dev, U, A, rows, cap_rows, pinned_rows, stream=None):
    """Usage policy of the bounded bank, before a store: *write_dev = the next free slot's row while *live_dev < cap_rows,
    else the row of the unpinned slot with the lowest U / A (A == 0 counts as +inf, ties to the lowest slot); that slot's
    U (float32 [cap_rows / rows]) and A (int32, same shape) restart at 0."""
    if U.dtype != torch.float32 or A.dtype != torch.int32 or not U.is_cuda or not A.is_cuda or \
            U.numel() * rows != cap_rows or A.numel() * rows != cap_rows:
        raise AotbError(f"ring_select_usage: U must be float32 and A int32 CUDA tensors of {cap_rows} / {rows} slots")
    check(lib().aotb_ring_select_usage(_counter("ring_select_usage: live_dev", live_dev),
                                       _counter("ring_select_usage: write_dev", write_dev), U.data_ptr(), A.data_ptr(),
                                       int(rows), int(cap_rows), int(pinned_rows), _st(stream)), "aotb_ring_select_usage")


# ------------------------------------------------------------------ tensor-core long-term attention
def tc_pack_rows(src, dst, row_off=0, div=1.0, row_off_dev=None, stream=None):
    """src fp32 [rows, H*32] -> dst fp16 [H, cap, 64] rows [row_off, row_off+rows) as [hi(32) | lo(32)]."""
    _chk(src)
    if dst.dtype != torch.float16 or not dst.is_cuda or not dst.is_contiguous():
        raise AotbError("packed operand buffer must be a contiguous fp16 CUDA tensor [H, cap, 64]")
    H, cap, _ = dst.shape
    rows = src.shape[0]
    check(lib().aotb_tc_pack_rows_f16x2(_p(src), src.stride(0), dst.data_ptr(), cap, rows, H, int(row_off),
                                        row_off_dev.data_ptr() if row_off_dev is not None else None, float(div),
                                        _st(stream)), "aotb_tc_pack_rows_f16x2")
    return dst


# layout of the tensor-core attention kernel (csrc/attn_tc.cuh); all compute the same maxima and, to fp32 rounding, the same P:
#   "tile"   128-query CTAs (two warpgroups of 64 rows), 64-key score tiles
#   "groups" the same CTAs with 128-key score tiles (half the tile iterations, twice the scores in registers)
#   "ahead"  64-key tiles, the scores of tile n + 1 issued on the tensor cores before the softmax of tile n
#   "pair"   64-query CTAs (one warpgroup), two co-resident per SM
LT_VARIANT = os.environ.get("AOTB_LT_VARIANT", "tile")
# 1: the mbarrier waits on the softmax -> MMA -> softmax chain poll instead of sleeping with a suspend-time hint
LT_SPIN = os.environ.get("AOTB_LT_SPIN", "0") == "1"


def lt_attn_tc_occupancy(exact=True):
    """The default ("tile") layout's kernel in one mode on the current device: (resident CTAs per SM, registers per thread,
    local-memory bytes per thread)."""
    import ctypes
    ctas, regs, local = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    check(lib().aotb_lt_attn_tc_occupancy(1 if exact else 0, ctypes.addressof(ctas), ctypes.addressof(regs),
                                          ctypes.addressof(local)), "aotb_lt_attn_tc_occupancy")
    return ctas.value, regs.value, local.value


def lt_attention_tc(Qp, Kp, Vp, N, Tk, O=None, Tk_dev=None, splits=1, exact=True, part=None, dbg=None, stream=None,
                    merge=True, variant=None):
    """Qp [H, Nq_cap, 64], Kp/Vp [H, kv_cap, 64] packed fp16x2; O [N, H*32] fp32.
    With splits > 1, `part` = (Opart [S,N,H*32], Mpart [S,H,N], Lpart [S,H,N]) and O receives the merge.
    `variant` (default: AOTB_LT_VARIANT) selects the kernel layout: "tile", "groups", "ahead" or "pair"."""
    v = LT_VARIANT if variant is None else variant
    if v not in ("tile", "groups", "ahead", "pair"):
        raise AotbError(f"unknown long-term attention variant '{v}' (tile | groups | ahead | pair)")
    mode = (1 if exact else 0) | (2 if v == "groups" else 0) | (4 if LT_SPIN else 0) | (8 if v == "ahead" else 0) | \
        (16 if v == "pair" else 0)
    H, nq_cap, _ = Qp.shape
    kv_cap = Kp.shape[1]
    if splits > 1:
        Op, Mp, Lp = part
    else:
        Op = Mp = Lp = None
    check(lib().aotb_lt_attn_tc_f16x2(Qp.data_ptr(), nq_cap, Kp.data_ptr(), Vp.data_ptr(), kv_cap, N, int(Tk),
                                      Tk_dev.data_ptr() if Tk_dev is not None else None, H,
                                      _p(O) if splits == 1 else None, O.stride(0) if O is not None else 0,
                                      _p(Op), _p(Mp), _p(Lp), splits, mode, _p(dbg), _st(stream)),
          "aotb_lt_attn_tc_f16x2")
    if splits > 1 and merge:
        attn_merge(Op, Mp, Lp, O, H, 32, stream=stream)
    return O


def gp_attention_tc(Qp, Kp, Vp, N, Tk, O=None, Tk_dev=None, splits=1, exact=True, part=None, stream=None, merge=True):
    """Fused DeAOT long-term attention: Qp [4, Nq_cap, 64], Kp [4, kv_cap, 64], Vp [dv/32, kv_cap, 64] packed
    fp16x2 (one 'head' per 32 channels); O [N, dv] fp32.  With splits > 1, `part` = (Opart [S,N,dv], Mpart [S,1,N],
    Lpart [S,1,N]) and O receives the merge."""
    nq_cap, kv_cap, dv = Qp.shape[1], Kp.shape[1], Vp.shape[0] * 32
    if splits > 1:
        Op, Mp, Lp = part
    else:
        Op = Mp = Lp = None
    mode = (1 if exact else 0) | (4 if LT_SPIN else 0)
    check(lib().aotb_gp_attn_tc_f16x2(Qp.data_ptr(), nq_cap, Kp.data_ptr(), Vp.data_ptr(), kv_cap, N, int(Tk),
                                      Tk_dev.data_ptr() if Tk_dev is not None else None, dv,
                                      _p(O) if splits == 1 else None, O.stride(0) if O is not None else 0,
                                      _p(Op), _p(Mp), _p(Lp), splits, mode, _st(stream)), "aotb_gp_attn_tc_f16x2")
    if splits > 1 and merge:
        attn_merge(Op, Mp, Lp, O, 1, dv, stream=stream)
    return O


def lt_attention_tc_slots(Qp, Kp, Vp, N, Tk_dev, slots, slot_rows, part, exact=True, stream=None):
    """lt_attention_tc over a bank of `slots` memory slots of `slot_rows` keys (default layout): split z of the partials
    `part` = (Opart [slots, N, H*32], Mpart [slots, H, N], Lpart [slots, H, N]) is slot z over the live keys *Tk_dev."""
    H, nq_cap, _ = Qp.shape
    Op, Mp, Lp = part
    _chk(Op, Mp, Lp)
    check(lib().aotb_lt_attn_tc_slots_f16x2(Qp.data_ptr(), nq_cap, Kp.data_ptr(), Vp.data_ptr(), Kp.shape[1], N, 0,
                                            _counter("lt_attention_tc_slots: Tk_dev", Tk_dev), H, _p(Op), _p(Mp), _p(Lp),
                                            int(slots), int(slot_rows), (1 if exact else 0) | (4 if LT_SPIN else 0),
                                            _st(stream)), "aotb_lt_attn_tc_slots_f16x2")


def gp_attention_tc_slots(Qp, Kp, Vp, N, Tk_dev, slots, slot_rows, part, exact=True, stream=None):
    """gp_attention_tc over a bank of `slots` memory slots of `slot_rows` keys: split z of `part` = (Opart [slots, N, dv],
    Mpart [slots, 1, N], Lpart [slots, 1, N]) is slot z over the live keys *Tk_dev."""
    Op, Mp, Lp = part
    _chk(Op, Mp, Lp)
    check(lib().aotb_gp_attn_tc_slots_f16x2(Qp.data_ptr(), Qp.shape[1], Kp.data_ptr(), Vp.data_ptr(), Kp.shape[1], N, 0,
                                            _counter("gp_attention_tc_slots: Tk_dev", Tk_dev), Vp.shape[0] * 32, _p(Op),
                                            _p(Mp), _p(Lp), int(slots), int(slot_rows),
                                            (1 if exact else 0) | (4 if LT_SPIN else 0), _st(stream)),
          "aotb_gp_attn_tc_slots_f16x2")


# ------------------------------------------------------------------ several independent videos per launch (multi_video.py)
def lt_attention_tc_batched(Qp, q_stride, Kp, Vp, kv_stride, n, N, Tk=0, Tk_dev=None, O=None, splits=1, exact=True,
                            part=None, stream=None):
    """n attentions in one launch ("tile" layout): problem b's queries are rows [b q_stride, b q_stride + N) of Qp [H, q_rows,
    64], its keys / values rows [b kv_stride, b kv_stride + Tk_dev[b]) of Kp / Vp [H, kv_rows, 64] (Tk_dev int32 [n], or Tk
    for all when None); O [n N, H*32] receives rows [b N, (b + 1) N).  With splits > 1, `part` = (Opart [splits, n N, H*32],
    Mpart [splits, H, n N], Lpart [splits, H, n N]) and O receives their merge."""
    H, q_rows, _ = Qp.shape
    if splits > 1:
        Op, Mp, Lp = part
        _chk(Op, Mp, Lp)
        if tuple(Op.shape) != (splits, n * N, H * 32) or tuple(Mp.shape) != (splits, H, n * N) or Lp.shape != Mp.shape:
            raise AotbError(f"lt_attention_tc_batched: partials must be [{splits}, {n * N}, {H * 32}] and [{splits}, {H}, "
                            f"{n * N}], got {tuple(Op.shape)}, {tuple(Mp.shape)}, {tuple(Lp.shape)}")
    else:
        Op = Mp = Lp = None
    if Tk_dev is not None and (Tk_dev.dtype != torch.int32 or not Tk_dev.is_cuda or Tk_dev.numel() != n):
        raise AotbError(f"lt_attention_tc_batched: Tk_dev must be an int32 CUDA tensor [{n}]")
    if O is None or O.shape[0] != n * N:
        raise AotbError(f"lt_attention_tc_batched: O must have {n * N} rows")
    _chk(O)
    check(lib().aotb_lt_attn_tc_batched_f16x2(Qp.data_ptr(), int(q_stride), q_rows, Kp.data_ptr(), Vp.data_ptr(),
                                              int(kv_stride), Kp.shape[1], int(n), int(N), int(Tk),
                                              Tk_dev.data_ptr() if Tk_dev is not None else None, H,
                                              _p(O) if splits == 1 else None, O.stride(0), _p(Op), _p(Mp), _p(Lp), int(splits),
                                              (1 if exact else 0) | (4 if LT_SPIN else 0), _st(stream)),
          "aotb_lt_attn_tc_batched_f16x2")
    if splits > 1:
        attn_merge(Op, Mp, Lp, O, H, 32, stream=stream)
    return O


def gp_attention_tc_batched(Qp, q_stride, Kp, Vp, kv_stride, n, N, Tk=0, Tk_dev=None, O=None, splits=1, exact=True,
                            part=None, stream=None):
    """n DeAOT attentions in one launch (gp_attention_tc's kernel): problem b's queries are rows [b q_stride, b q_stride + N)
    of Qp [4, q_rows, 64], its keys / values rows [b kv_stride, b kv_stride + Tk_dev[b]) of Kp [4, kv_rows, 64] / Vp [dv/32,
    kv_rows, 64] (Tk_dev int32 [n], or Tk for all when None); O [n N, dv] receives rows [b N, (b + 1) N).  With splits > 1,
    `part` = (Opart [splits, n N, dv], Mpart [splits, 1, n N], Lpart [splits, 1, n N]) and O receives their merge."""
    q_rows, dv = Qp.shape[1], Vp.shape[0] * 32
    if Qp.shape[0] != 4 or Kp.shape[0] != 4 or Vp.shape[1] != Kp.shape[1]:
        raise AotbError(f"gp_attention_tc_batched: Qp / Kp must be [4, rows, 64] and Vp [dv/32, kv_rows, 64], got "
                        f"{tuple(Qp.shape)}, {tuple(Kp.shape)}, {tuple(Vp.shape)}")
    if splits > 1:
        Op, Mp, Lp = part
        _chk(Op, Mp, Lp)
        if tuple(Op.shape) != (splits, n * N, dv) or tuple(Mp.shape) != (splits, 1, n * N) or Lp.shape != Mp.shape:
            raise AotbError(f"gp_attention_tc_batched: partials must be [{splits}, {n * N}, {dv}] and [{splits}, 1, {n * N}], "
                            f"got {tuple(Op.shape)}, {tuple(Mp.shape)}, {tuple(Lp.shape)}")
    else:
        Op = Mp = Lp = None
    if Tk_dev is not None and (Tk_dev.dtype != torch.int32 or not Tk_dev.is_cuda or Tk_dev.numel() != n):
        raise AotbError(f"gp_attention_tc_batched: Tk_dev must be an int32 CUDA tensor [{n}]")
    if O is None or O.shape[0] != n * N or O.shape[1] != dv:
        raise AotbError(f"gp_attention_tc_batched: O must be [{n * N}, {dv}]")
    _chk(O)
    check(lib().aotb_gp_attn_tc_batched_f16x2(Qp.data_ptr(), int(q_stride), q_rows, Kp.data_ptr(), Vp.data_ptr(),
                                              int(kv_stride), Kp.shape[1], int(n), int(N), int(Tk),
                                              Tk_dev.data_ptr() if Tk_dev is not None else None, dv,
                                              _p(O) if splits == 1 else None, O.stride(0), _p(Op), _p(Mp), _p(Lp), int(splits),
                                              (1 if exact else 0) | (4 if LT_SPIN else 0), _st(stream)),
          "aotb_gp_attn_tc_batched_f16x2")
    if splits > 1:
        attn_merge(Op, Mp, Lp, O, 1, dv, stream=stream)
    return O


def local_gated_tile_batched(q, k, v, relk_w, relk_b, out, h, w, n, stream=None):
    """local_gated_tile over n h x w maps stacked along the rows of q, k ([n h w, 128]), v and out ([n h w, 1024])."""
    _chk(q, k, v, relk_w, relk_b, out)
    if q.shape[1] != 128 or k.shape[1] != 128 or v.shape[1] != 1024 or out.shape[1] != 1024 or not relk_w.is_contiguous():
        raise AotbError("local_gated_tile_batched: q / k [n hw, 128], v / out [n hw, 1024], contiguous relative_emb_k "
                        "weights [225, 128]")
    if any(t.shape[0] != n * h * w for t in (q, k, v, out)):
        raise AotbError(f"local_gated_tile_batched: q, k, v and out need {n} x {h * w} rows")
    check(lib().aotb_local_gated_tile_batched_f32(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(relk_w),
                                                  _p(relk_b), _p(out), out.stride(0), h, w, int(n), _st(stream)),
          "aotb_local_gated_tile_batched_f32")
    return out


def local_attention_tc_batched(q, k, v, relk_w, relk_b, relv_t, out, h, w, H, n, stream=None):
    """local_attention_tc over n h x w maps stacked along the rows of q, k, v and out ([n h w, ...] each)."""
    _chk(q, k, v, relk_w, relk_b, relv_t, out)
    if any(t.shape[0] != n * h * w for t in (q, k, v, out)):
        raise AotbError(f"local_attention_tc_batched: q, k, v and out need {n} x {h * w} rows")
    check(lib().aotb_local_attention_tc_batched_f32(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(relk_w),
                                                    _p(relk_b), _p(relv_t), _p(out), out.stride(0), h, w, H, int(n),
                                                    _st(stream)), "aotb_local_attention_tc_batched_f32")
    return out


def id_embed_runs_batched(masks, wp, bias, out, C, nid, ksize, stride, pad, ln_gamma=None, ln_beta=None, stream=None):
    """id_embed_runs over n label maps masks [n, Hm, Wm] (contiguous) -> out [n ho wo, C]."""
    if masks.dim() != 3 or not masks.is_contiguous():
        raise AotbError(f"id_embed_runs_batched: masks must be contiguous [n, Hm, Wm], got {tuple(masks.shape)}")
    n, Hm, Wm = masks.shape
    ho, wo = (Hm + 2 * pad - ksize) // stride + 1, (Wm + 2 * pad - ksize) // stride + 1
    _id_embed_check("id_embed_runs_batched", masks[0], wp, (ksize, ksize + 1, nid, C), bias, out[:ho * wo], C, ksize, stride,
                    pad, ln_gamma, ln_beta)
    if out.shape[0] != n * ho * wo:
        raise AotbError(f"id_embed_runs_batched: out must have {n * ho * wo} rows, got {out.shape[0]}")
    check(lib().aotb_id_embed_runs_batched_f32(_p(masks), n, Hm, Wm, _p(wp), _p(bias), _p(ln_gamma), _p(ln_beta), _p(out),
                                               out.stride(0), C, nid, ksize, stride, pad, _st(stream)),
          "aotb_id_embed_runs_batched_f32")
    return out


def _flags(name, t, n):
    if t is None or not t.is_cuda or t.dtype != torch.int32 or t.numel() != n or not t.is_contiguous():
        raise AotbError(f"{name} must be a contiguous int32 CUDA tensor [{n}]")
    return t.data_ptr()


def bank_ring_store_batched(k_src, v_src, k_bank, v_bank, k_packed, v_packed, write_dev, store_dev, n, cap_rows, stream=None):
    """Bounded banks of n videos, stacked: video b's bank is rows [b cap_rows, (b + 1) cap_rows) of k_bank / v_bank [>= n
    cap_rows, C] and of k_packed / v_packed [C / 32, >= n cap_rows, 64] (views may start at a video's first row: the chunk
    stride is the tensor's).  Where store_dev[b] != 0, video b's rows [b rows, (b + 1) rows) of k_src / v_src [n rows, C] go to
    row write_dev[b] of its bank (int32 CUDA tensors [n])."""
    _chk(k_src, v_src, k_bank, v_bank)
    rows = k_src.shape[0] // n
    if k_src.shape[0] != n * rows or v_src.shape[0] != n * rows:
        raise AotbError(f"bank_ring_store_batched: k_src and v_src need {n} equal blocks of rows")
    head_rows = None
    for name, src, bank, packed in (("k", k_src, k_bank, k_packed), ("v", v_src, v_bank, v_packed)):
        if bank is not None and (bank.shape[0] < n * cap_rows or bank.shape[1] < src.shape[1]):
            raise AotbError(f"bank_ring_store_batched: {name}_bank {tuple(bank.shape)} holds fewer than {n} banks of "
                            f"{cap_rows} x {src.shape[1]}")
        if packed is not None:
            if packed.dtype != torch.float16 or not packed.is_cuda or packed.dim() != 3 or packed.shape[2] != 64 or \
                    packed.stride(2) != 1 or packed.stride(1) != 64 or packed.shape[0] * 32 != src.shape[1] or \
                    packed.shape[1] < n * cap_rows:
                raise AotbError(f"bank_ring_store_batched: {name}_packed must be fp16 [{src.shape[1]} / 32, >= {n * cap_rows}, "
                                f"64] with dense rows")
            hr = packed.stride(0) // 64
            if head_rows not in (None, hr):
                raise AotbError("bank_ring_store_batched: the packed copies need one chunk stride")
            head_rows = hr
    check(lib().aotb_bank_ring_store_batched(_p(k_src), k_src.stride(0), k_src.shape[1], _p(v_src), v_src.stride(0),
                                             v_src.shape[1], rows, int(n), _p(k_bank),
                                             k_bank.stride(0) if k_bank is not None else 0, _p(v_bank),
                                             v_bank.stride(0) if v_bank is not None else 0, _p(k_packed), _p(v_packed),
                                             int(cap_rows), int(head_rows if head_rows is not None else n * cap_rows),
                                             _flags("bank_ring_store_batched: write_dev", write_dev, n),
                                             _flags("bank_ring_store_batched: store_dev", store_dev, n), _st(stream)),
          "aotb_bank_ring_store_batched")


def ring_advance_batched(live_dev, write_dev, store_dev, n, rows, cap_rows, pinned_rows, stream=None):
    """ring_advance for each of n banks whose store_dev[b] != 0 (live_dev / write_dev / store_dev int32 CUDA tensors [n])."""
    check(lib().aotb_ring_advance_batched(_flags("ring_advance_batched: live_dev", live_dev, n),
                                          _flags("ring_advance_batched: write_dev", write_dev, n),
                                          _flags("ring_advance_batched: store_dev", store_dev, n), int(n), int(rows),
                                          int(cap_rows), int(pinned_rows), _st(stream)), "aotb_ring_advance_batched")
