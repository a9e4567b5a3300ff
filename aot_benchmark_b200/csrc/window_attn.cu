// Swin-B encoder pieces that are not plain linears / LayerNorms (BASELINE config 4, SURVEY 8 row a19):
//
//  * window_attn_kernel -- WindowAttention.forward (networks/encoders/swin/swin_transformer.py:158-196) fused with the
//    data movement SwinTransformerBlock.forward wraps around it (:273-316: zero padding to a multiple of the window,
//    cyclic shift by -shift, window partition, window reverse, shift back, crop) and with the shifted-window mask
//    BasicLayer.forward builds (:416-438).  The reference materialises the padded / rolled / partitioned copies and a
//    [nW, 49, 49] mask; here each CTA addresses its 49 tokens of one (window, head) in place:
//        token (ty, tx) of window (wy, wx) sits at (ys, xs) = (7 wy + ty, 7 wx + tx) of the SHIFTED padded map, which is
//        position ((ys + shift) mod Hp, (xs + shift) mod Wp) of the un-shifted one; positions outside H x W are padding.
//    Padding is applied after norm1 and before the qkv Linear (:273-278, :166), so a padded token has q = k = v = the qkv
//    bias and takes part in its window's softmax like any other key (this is what the reference computes).
//    The qkv Linear itself runs on the un-padded token matrix with the tensor-core GEMM (it is per-token, so it commutes
//    with the permutation); this kernel reads its [H*W, 3C] output.
//  * patch_merge_kernel -- the 2x2 gather of PatchMerging.forward (:339-365) in the reference's channel order
//    [(0,0) | (1,0) | (0,1) | (1,1)] with zero padding for odd maps; LayerNorm(4C) and the bias-free reduction reuse
//    layernorm_kernel and the GEMM.
//
// Both kernels take a batch of B token maps stacked densely ([B*H*W] rows, blockIdx.z / blockIdx.y = image): the padding,
// shift, mask and crop are those of each image, and every image gets the CTAs a one-image launch would give it.
//
// Bound: HBM/L2 (each qkv element is read once per use; 2*49*49*32 FMAs per (window, head) is ~1 GFLOP per frame at
// 592x1040, three orders of magnitude below the encoder's linears).
#include "common.cuh"

namespace aotb {

template <int WS, int D>
__global__ void __launch_bounds__(64) window_attn_kernel(const float* __restrict__ qkv, int ld,
                                                         const float* __restrict__ qkv_bias,
                                                         const float* __restrict__ rel_bias, float* __restrict__ out,
                                                         int ldo, int H, int W, int Hp, int Wp, int C, int shift,
                                                         float scale) {
    constexpr int T = WS * WS;
    constexpr int D4 = D / 4;
    __shared__ __align__(16) float sK[T][D];   // keys; reused as the output staging tile
    __shared__ __align__(16) float sV[T][D];
    __shared__ int sSrc[T];                    // row of the token in the un-padded [H*W] matrix, -1 = padding
    __shared__ int sReg[T];                    // region id of the shifted-window mask (0 when shift == 0)
    pdl_sync();
    qkv += (size_t)blockIdx.z * H * W * ld;          // image blockIdx.z of a batch
    out += (size_t)blockIdx.z * H * W * ldo;
    const int tid = threadIdx.x;
    const int head = blockIdx.y;
    const int nwx = Wp / WS;
    const int wy = blockIdx.x / nwx, wx = blockIdx.x - wy * nwx;
    if (tid < T) {
        const int ty = tid / WS, tx = tid - ty * WS;
        const int ys = wy * WS + ty, xs = wx * WS + tx;
        int y = ys + shift, x = xs + shift;
        if (y >= Hp) y -= Hp;
        if (x >= Wp) x -= Wp;
        sSrc[tid] = (y < H && x < W) ? y * W + x : -1;
        int ry = 0, rx = 0;
        if (shift > 0) {   // h_slices / w_slices of :421-426: [0, n-WS) -> 0, [n-WS, n-shift) -> 1, [n-shift, n) -> 2
            ry = ys < Hp - WS ? 0 : (ys < Hp - shift ? 1 : 2);
            rx = xs < Wp - WS ? 0 : (xs < Wp - shift ? 1 : 2);
        }
        sReg[tid] = ry * 3 + rx;
    }
    __syncthreads();
    const float* kb = qkv_bias + C + head * D;
    const float* vb = qkv_bias + 2 * C + head * D;
    for (int i = tid; i < T * D4; i += 64) {
        const int t = i / D4, c4 = (i - t * D4) * 4;
        const int src = sSrc[t];
        float4 k, v;
        if (src >= 0) {
            const float* r = qkv + (size_t)src * ld + head * D + c4;
            k = *reinterpret_cast<const float4*>(r + C);
            v = *reinterpret_cast<const float4*>(r + 2 * C);
        } else {
            k = __ldg(reinterpret_cast<const float4*>(kb + c4));
            v = __ldg(reinterpret_cast<const float4*>(vb + c4));
        }
        *reinterpret_cast<float4*>(&sK[t][c4]) = k;
        *reinterpret_cast<float4*>(&sV[t][c4]) = v;
    }
    __syncthreads();
    const bool active = tid < T;
    float o[D];
#pragma unroll
    for (int c = 0; c < D; ++c) o[c] = 0.f;
    if (active) {
        const int src = sSrc[tid];
        const float* qp = src >= 0 ? qkv + (size_t)src * ld + head * D : qkv_bias + head * D;
        float q[D];
#pragma unroll
        for (int c4 = 0; c4 < D; c4 += 4) {
            const float4 t4 = *reinterpret_cast<const float4*>(qp + c4);
            q[c4] = t4.x * scale; q[c4 + 1] = t4.y * scale; q[c4 + 2] = t4.z * scale; q[c4 + 3] = t4.w * scale;   // :173
        }
        const float* rb = rel_bias + ((size_t)head * T + tid) * T;
        const int myreg = sReg[tid];
        float s[T];
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < T; ++j) {
            float acc = 0.f;
#pragma unroll
            for (int c4 = 0; c4 < D; c4 += 4) {
                const float4 k4 = *reinterpret_cast<const float4*>(&sK[j][c4]);   // same address for all lanes: broadcast
                acc = fmaf(q[c4], k4.x, acc);
                acc = fmaf(q[c4 + 1], k4.y, acc);
                acc = fmaf(q[c4 + 2], k4.z, acc);
                acc = fmaf(q[c4 + 3], k4.w, acc);
            }
            acc += __ldg(rb + j);                                  // relative position bias :176-184
            if (sReg[j] != myreg) acc += -100.f;                   // shifted-window mask :436-438, :186-190
            s[j] = acc;
            m = fmaxf(m, acc);
        }
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < T; ++j) {
            s[j] = expf(s[j] - m);
            sum += s[j];
        }
        const float inv = 1.f / sum;
#pragma unroll
        for (int j = 0; j < T; ++j) {
            const float p = s[j] * inv;
#pragma unroll
            for (int c4 = 0; c4 < D; c4 += 4) {
                const float4 v4 = *reinterpret_cast<const float4*>(&sV[j][c4]);
                o[c4] = fmaf(p, v4.x, o[c4]);
                o[c4 + 1] = fmaf(p, v4.y, o[c4 + 1]);
                o[c4 + 2] = fmaf(p, v4.z, o[c4 + 2]);
                o[c4 + 3] = fmaf(p, v4.w, o[c4 + 3]);
            }
        }
    }
    __syncthreads();                 // every thread is done reading sK: reuse it to stage the output rows
    if (active) {
#pragma unroll
        for (int c4 = 0; c4 < D; c4 += 4)
            *reinterpret_cast<float4*>(&sK[tid][c4]) = make_float4(o[c4], o[c4 + 1], o[c4 + 2], o[c4 + 3]);
    }
    __syncthreads();
    for (int i = tid; i < T * D4; i += 64) {     // 8 consecutive threads write one 128-byte row
        const int t = i / D4, c4 = (i - t * D4) * 4;
        const int src = sSrc[t];
        if (src >= 0)                              // crop of :311-312: padded positions are dropped
            *reinterpret_cast<float4*>(out + (size_t)src * ldo + head * D + c4) =
                *reinterpret_cast<const float4*>(&sK[t][c4]);
    }
}

// out[(y2*W2 + x2)][q*C + c] = x[(2 y2 + (q & 1)) * W + 2 x2 + (q >> 1)][c], zero outside H x W
__global__ void patch_merge_kernel(const float* __restrict__ x, int ldx, float* __restrict__ out, int ldo, int H, int W,
                                   int H2, int W2, int C) {
    pdl_sync();
    x += (size_t)blockIdx.y * H * W * ldx;           // image blockIdx.y of a batch
    out += (size_t)blockIdx.y * H2 * W2 * ldo;
    const int C4 = C >> 2;
    const size_t total = (size_t)H2 * W2 * 4 * C4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4) * 4;
        const size_t r4 = i / C4;
        const int q = (int)(r4 & 3);
        const size_t r = r4 >> 2;
        const int y2 = (int)(r / W2), x2 = (int)(r - (size_t)y2 * W2);
        const int y = 2 * y2 + (q & 1), xx = 2 * x2 + (q >> 1);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (y < H && xx < W) v = *reinterpret_cast<const float4*>(x + ((size_t)y * W + xx) * ldx + c4);
        *reinterpret_cast<float4*>(out + r * ldo + (size_t)q * C + c4) = v;
    }
}

}  // namespace aotb

using namespace aotb;

extern "C" int aotb_window_attention_batched_f32(const float* qkv, int ldqkv, const float* qkv_bias, const float* rel_bias,
                                                 float* out, int ldo, int B, int H, int W, int C, int heads, int window,
                                                 int shift, void* stream) {
    AOTB_REQUIRE(qkv && qkv_bias && rel_bias && out && B > 0 && B <= 65535 && H > 0 && W > 0 && heads > 0,
                 "aotb_window_attention_f32: bad args");
    AOTB_REQUIRE(window == 7 && C == heads * 32,
                 "aotb_window_attention_f32: built for window 7 and head dim 32 (swin_base), got window %d, C/heads %d",
                 window, heads ? C / heads : 0);
    AOTB_REQUIRE(shift >= 0 && shift < window, "aotb_window_attention_f32: shift must be in [0, window)");
    AOTB_REQUIRE(ldqkv % 4 == 0 && ldo % 4 == 0 && ((uintptr_t)qkv % 16 == 0) && ((uintptr_t)out % 16 == 0) &&
                     ((uintptr_t)qkv_bias % 16 == 0),
                 "aotb_window_attention_f32: 16-byte alignment required");
    const int Hp = cdiv(H, window) * window, Wp = cdiv(W, window) * window;
    dim3 grid((Hp / window) * (Wp / window), heads, B);
    launch(window_attn_kernel<7, 32>, grid, dim3(64), 0, (cudaStream_t)stream, qkv, ldqkv, qkv_bias, rel_bias, out, ldo, H,
           W, Hp, Wp, C, shift, 0.17677669529663687f);   // head_dim ** -0.5 (:124)
    return check_launch("aotb_window_attention_f32");
}

extern "C" int aotb_window_attention_f32(const float* qkv, int ldqkv, const float* qkv_bias, const float* rel_bias,
                                         float* out, int ldo, int H, int W, int C, int heads, int window, int shift,
                                         void* stream) {
    return aotb_window_attention_batched_f32(qkv, ldqkv, qkv_bias, rel_bias, out, ldo, 1, H, W, C, heads, window, shift,
                                             stream);
}

extern "C" int aotb_patch_merge_batched_f32(const float* x, int ldx, float* out, int ldo, int B, int H, int W, int C,
                                            void* stream) {
    AOTB_REQUIRE(x && out && B > 0 && B <= 65535 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "aotb_patch_merge_f32: bad args");
    AOTB_REQUIRE(ldx % 4 == 0 && ldo % 4 == 0 && ((uintptr_t)x % 16 == 0) && ((uintptr_t)out % 16 == 0),
                 "aotb_patch_merge_f32: 16-byte alignment required");
    const int H2 = (H + 1) / 2, W2 = (W + 1) / 2;
    const size_t total = (size_t)H2 * W2 * C;
    size_t g = (total + 255) / 256;
    if (g > 132 * 16) g = 132 * 16;
    launch(patch_merge_kernel, dim3((unsigned)g, B), dim3(256), 0, (cudaStream_t)stream, x, ldx, out, ldo, H, W, H2, W2, C);
    return check_launch("aotb_patch_merge_f32");
}

extern "C" int aotb_patch_merge_f32(const float* x, int ldx, float* out, int ldo, int H, int W, int C, void* stream) {
    return aotb_patch_merge_batched_f32(x, ldx, out, ldo, 1, H, W, C, stream);
}
