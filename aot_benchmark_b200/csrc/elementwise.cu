// HBM-bound NHWC helpers of the per-frame path (fp32): layout transposes, max-pool, depthwise
// convolution, bilinear resize, gating/element-wise ops, strided copies.
//
// Reference sites: resnet.py:143-146 (maxpool 3x3 s2 p1), basic.py:15-57 (depthwise 5x5 of
// GNActDWConv2d / DWConv2d), mobilenetv2.py:93-101 (depthwise 3x3 + FrozenBN + ReLU6),
// fpn.py:45-54 (F.interpolate bilinear), attention.py:585-586,707,855 (SiLU, *U gating),
// transformer.py:602-611,625-626 (channel concats of the GPM block).
#include "common.cuh"

namespace aotb {

// ---------------------------------------------------------------- NCHW <-> NHWC (tiled transpose)
// in [B][R][Cc] -> out [B][Cc][R]
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int Cc) {
    pdl_sync();
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const float* ib = in + (size_t)b * R * Cc;
    float* ob = out + (size_t)b * R * Cc;
    int c = blockIdx.x * 32 + threadIdx.x;
    for (int j = threadIdx.y; j < 32; j += 8) {
        int r = blockIdx.y * 32 + j;
        if (r < R && c < Cc) tile[j][threadIdx.x] = ib[(size_t)r * Cc + c];
    }
    __syncthreads();
    int r = blockIdx.y * 32 + threadIdx.x;
    for (int j = threadIdx.y; j < 32; j += 8) {
        int cc = blockIdx.x * 32 + j;
        if (r < R && cc < Cc) ob[(size_t)cc * R + r] = tile[threadIdx.x][j];
    }
}

// image [3][HW] (NCHW, batch 1) -> [HW][4] NHWC with a zero 4th channel (so the stem conv reads 16-byte pixels)
__global__ void image_to_nhwc4_kernel(const float* __restrict__ in, float4* __restrict__ out, int HW) {
    pdl_sync();
    in += (size_t)blockIdx.y * 3 * HW;               // image blockIdx.y of a batch [B,3,H,W] -> [B,H,W,4]
    out += (size_t)blockIdx.y * HW;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x)
        out[i] = make_float4(in[i], in[HW + i], in[2 * HW + i], 0.f);
}

// ---------------------------------------------------------------- max-pool 3x3 s2 p1 (NHWC, C%4==0)
__global__ void maxpool3x3s2_kernel(const float4* __restrict__ in, float4* __restrict__ out, int B, int H, int W,
                                    int C4, int Ho, int Wo) {
    pdl_sync();
    const size_t total = (size_t)B * Ho * Wo * C4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int c = i % C4;
        size_t t = i / C4;
        int ox = t % Wo; t /= Wo;
        int oy = t % Ho;
        int b = t / Ho;
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
            int iy = oy * 2 - 1 + dy;
            if (iy < 0 || iy >= H) continue;
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                int ix = ox * 2 - 1 + dx;
                if (ix < 0 || ix >= W) continue;
                float4 v = __ldg(in + (((size_t)b * H + iy) * W + ix) * C4 + c);
                m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
            }
        }
        out[i] = m;
    }
}

// ---------------------------------------------------------------- depthwise conv (NHWC, C%4==0)
// w layout [KH*KW][C]; optional per-channel bias; optional activation.
template <bool HS = false>
__global__ void dwconv_kernel(const float* __restrict__ in, const float* __restrict__ w,
                              const float* __restrict__ bias, float* __restrict__ out, int B, int H, int W, int C,
                              int ldin, int ldout, int Ho, int Wo, int KH, int KW, int stride, int pad, int dil,
                              int act) {
    pdl_sync();
    const int C4 = C >> 2;
    const size_t total = (size_t)B * Ho * Wo * C4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int c = (i % C4) * 4;
        size_t t = i / C4;
        int ox = t % Wo; t /= Wo;
        int oy = t % Ho;
        int b = t / Ho;
        float4 acc = bias ? __ldg(reinterpret_cast<const float4*>(bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
        for (int ky = 0; ky < KH; ++ky) {
            int iy = oy * stride - pad + ky * dil;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < KW; ++kx) {
                int ix = ox * stride - pad + kx * dil;
                if (ix < 0 || ix >= W) continue;
                float4 v = __ldg(reinterpret_cast<const float4*>(in + (((size_t)b * H + iy) * W + ix) * ldin + c));
                float4 ww = __ldg(reinterpret_cast<const float4*>(w + (size_t)(ky * KW + kx) * C + c));
                acc.x = fmaf(v.x, ww.x, acc.x); acc.y = fmaf(v.y, ww.y, acc.y);
                acc.z = fmaf(v.z, ww.z, acc.z); acc.w = fmaf(v.w, ww.w, acc.w);
            }
        }
        acc.x = apply_act_or_hswish<HS>(acc.x, act); acc.y = apply_act_or_hswish<HS>(acc.y, act);
        acc.z = apply_act_or_hswish<HS>(acc.z, act); acc.w = apply_act_or_hswish<HS>(acc.w, act);
        *reinterpret_cast<float4*>(out + (((size_t)b * Ho + oy) * Wo + ox) * ldout + c) = acc;
    }
}

// Stride-1, dilation-1 K x K depthwise conv (the 5x5 of the LSTT / GPM feed-forward): one thread = 4 neighbouring
// output pixels x 4 channels.  The K+3 inputs of a filter row and its K weights are loaded once and shared by the 4
// outputs (K*(K+3) + K*K loads per 4*K*K taps instead of 2 per tap -- the generic kernel above is L1-bandwidth bound).
template <int K, bool HS = false>
__global__ void dwconv_row4_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                   const float* __restrict__ bias, float* __restrict__ out, int B, int H, int W, int C,
                                   int ldin, int ldout, int pad, int act) {
    pdl_sync();
    const int C4 = C >> 2, Ho = H + 2 * pad - K + 1, Wo = W + 2 * pad - K + 1, XB = (Wo + 3) >> 2;
    const size_t total = (size_t)B * Ho * XB * C4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (i % C4) * 4;
        size_t t = i / C4;
        const int ox0 = (t % XB) * 4; t /= XB;
        const int oy = t % Ho;
        const int b = t / Ho;
        float4 acc[4];
        const float4 b4 = bias ? __ldg(reinterpret_cast<const float4*>(bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int o = 0; o < 4; ++o) acc[o] = b4;
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
            const int iy = oy - pad + ky;
            if (iy < 0 || iy >= H) continue;
            float4 v[K + 3], ww[K];
#pragma unroll
            for (int j = 0; j < K + 3; ++j) {
                const int ix = ox0 - pad + j;
                v[j] = (ix >= 0 && ix < W) ? __ldg(reinterpret_cast<const float4*>(in + (((size_t)b * H + iy) * W + ix) * ldin + c))
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int kx = 0; kx < K; ++kx) ww[kx] = __ldg(reinterpret_cast<const float4*>(w + (size_t)(ky * K + kx) * C + c));
#pragma unroll
            for (int o = 0; o < 4; ++o)
#pragma unroll
                for (int kx = 0; kx < K; ++kx) {        // same (ky, kx) order per output as the generic kernel
                    acc[o].x = fmaf(v[o + kx].x, ww[kx].x, acc[o].x); acc[o].y = fmaf(v[o + kx].y, ww[kx].y, acc[o].y);
                    acc[o].z = fmaf(v[o + kx].z, ww[kx].z, acc[o].z); acc[o].w = fmaf(v[o + kx].w, ww[kx].w, acc[o].w);
                }
        }
#pragma unroll
        for (int o = 0; o < 4; ++o) {
            if (ox0 + o >= Wo) break;
            float4 r = acc[o];
            r.x = apply_act_or_hswish<HS>(r.x, act); r.y = apply_act_or_hswish<HS>(r.y, act);
            r.z = apply_act_or_hswish<HS>(r.z, act); r.w = apply_act_or_hswish<HS>(r.w, act);
            *reinterpret_cast<float4*>(out + (((size_t)b * Ho + oy) * Wo + ox0 + o) * ldout + c) = r;
        }
    }
}

// ---------------------------------------------------------------- bilinear resize (NHWC, C%4==0)
// PyTorch semantics (aten upsample_bilinear2d): align_corners -> src = dst*(in-1)/(out-1);
// otherwise src = max((dst+0.5)*in/out-0.5, 0).
__device__ __forceinline__ void bilinear_src(int dst, int in_sz, int out_sz, int align, int& i0, int& i1,
                                             float& l1) {
    float src;
    if (align) {
        const float scale = out_sz > 1 ? (float)(in_sz - 1) / (float)(out_sz - 1) : 0.f;
        src = scale * dst;
    } else {
        const float scale = (float)in_sz / (float)out_sz;
        src = scale * (dst + 0.5f) - 0.5f;
        if (src < 0.f) src = 0.f;
    }
    i0 = (int)src;
    if (i0 > in_sz - 1) i0 = in_sz - 1;
    i1 = i0 + (i0 < in_sz - 1 ? 1 : 0);
    l1 = src - (float)i0;
}

__global__ void bilinear_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W,
                                     int C, int Ho, int Wo, int align) {
    pdl_sync();
    const int C4 = C >> 2;
    const size_t total = (size_t)B * Ho * Wo * C4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int c = (i % C4) * 4;
        size_t t = i / C4;
        int ox = t % Wo; t /= Wo;
        int oy = t % Ho;
        int b = t / Ho;
        int y0, y1, x0, x1;
        float ly, lx;
        bilinear_src(oy, H, Ho, align, y0, y1, ly);
        bilinear_src(ox, W, Wo, align, x0, x1, lx);
        const float hy = 1.f - ly, hx = 1.f - lx;
        const float* base = in + (size_t)b * H * W * C + c;
        float4 v00 = __ldg(reinterpret_cast<const float4*>(base + ((size_t)y0 * W + x0) * C));
        float4 v01 = __ldg(reinterpret_cast<const float4*>(base + ((size_t)y0 * W + x1) * C));
        float4 v10 = __ldg(reinterpret_cast<const float4*>(base + ((size_t)y1 * W + x0) * C));
        float4 v11 = __ldg(reinterpret_cast<const float4*>(base + ((size_t)y1 * W + x1) * C));
        float4 o;
        // same association as aten: h0*(w0*a + w1*b) + h1*(w0*c + w1*d)
        o.x = hy * (hx * v00.x + lx * v01.x) + ly * (hx * v10.x + lx * v11.x);
        o.y = hy * (hx * v00.y + lx * v01.y) + ly * (hx * v10.y + lx * v11.y);
        o.z = hy * (hx * v00.z + lx * v01.z) + ly * (hx * v10.z + lx * v11.z);
        o.w = hy * (hx * v00.w + lx * v01.w) + ly * (hx * v10.w + lx * v11.w);
        *reinterpret_cast<float4*>(out + i * 4) = o;
    }
}

// ---------------------------------------------------------------- element-wise with row strides
// op: 0 copy, 1 a+b, 2 a*b, 3 silu(a), 4 silu(a)*b, 5 fill(scalar)
enum { EW_COPY = 0, EW_ADD = 1, EW_MUL = 2, EW_SILU = 3, EW_SILU_MUL = 4, EW_FILL = 5 };

__global__ void eltwise_kernel(int op, const float* __restrict__ a, int lda, const float* __restrict__ b, int ldb,
                               float* __restrict__ out, int ldo, int rows, int cols, float scalar) {
    pdl_sync();
    const size_t total = (size_t)rows * cols;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = i / cols, c = i - (size_t)r * cols;
        float x = (op == EW_FILL) ? scalar : a[(size_t)r * lda + c];
        float y = (op == EW_ADD || op == EW_MUL || op == EW_SILU_MUL) ? b[(size_t)r * ldb + c] : 0.f;
        float o;
        switch (op) {
            case EW_ADD: o = x + y; break;
            case EW_MUL: o = x * y; break;
            case EW_SILU: o = apply_act(x, ACT_SILU); break;
            case EW_SILU_MUL: o = apply_act(x, ACT_SILU) * y; break;
            default: o = x;
        }
        out[(size_t)r * ldo + c] = o;
    }
}

static inline int grid_for(size_t total, int block) {
    size_t g = (total + block - 1) / block;
    const size_t cap = 132 * 16;
    return (int)(g < cap ? (g ? g : 1) : cap);
}

}  // namespace aotb

using namespace aotb;

extern "C" int aotb_nchw_to_nhwc_f32(const float* in, float* out, int B, int C, int HW, void* stream) {
    AOTB_REQUIRE(in && out && B > 0 && C > 0 && HW > 0, "aotb_nchw_to_nhwc_f32: bad args");
    dim3 grid(cdiv(HW, 32), cdiv(C, 32), B), block(32, 8);
    launch(transpose_kernel, dim3(grid), dim3(block), 0, (cudaStream_t)stream, in, out, C, HW);
    return check_launch("aotb_nchw_to_nhwc_f32");
}

extern "C" int aotb_image_to_nhwc4_batched_f32(const float* in, float* out, int B, int HW, void* stream) {
    AOTB_REQUIRE(in && out && B > 0 && B <= 65535 && HW > 0, "aotb_image_to_nhwc4_f32: bad args");
    int g = (HW + 255) / 256;
    if (g > 132 * 8) g = 132 * 8;
    launch(image_to_nhwc4_kernel, dim3(g, B), dim3(256), 0, (cudaStream_t)stream, in, reinterpret_cast<float4*>(out), HW);
    return check_launch("aotb_image_to_nhwc4_f32");
}

extern "C" int aotb_image_to_nhwc4_f32(const float* in, float* out, int HW, void* stream) {
    return aotb_image_to_nhwc4_batched_f32(in, out, 1, HW, stream);
}

extern "C" int aotb_nhwc_to_nchw_f32(const float* in, float* out, int B, int C, int HW, void* stream) {
    AOTB_REQUIRE(in && out && B > 0 && C > 0 && HW > 0, "aotb_nhwc_to_nchw_f32: bad args");
    dim3 grid(cdiv(C, 32), cdiv(HW, 32), B), block(32, 8);
    launch(transpose_kernel, dim3(grid), dim3(block), 0, (cudaStream_t)stream, in, out, HW, C);
    return check_launch("aotb_nhwc_to_nchw_f32");
}

extern "C" int aotb_maxpool3x3s2_nhwc_f32(const float* in, float* out, int B, int H, int W, int C, void* stream) {
    AOTB_REQUIRE(in && out && C % 4 == 0, "aotb_maxpool3x3s2_nhwc_f32: C %% 4 != 0 or null");
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const size_t total = (size_t)B * Ho * Wo * (C / 4);
    launch(maxpool3x3s2_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, reinterpret_cast<const float4*>(in), reinterpret_cast<float4*>(out), B, H, W, C / 4, Ho, Wo);
    return check_launch("aotb_maxpool3x3s2_nhwc_f32");
}

extern "C" int aotb_dwconv_nhwc_f32(const float* in, const float* w, const float* bias, float* out, int B, int H,
                                    int W, int C, int ldin, int ldout, int KH, int KW, int stride, int pad, int dil,
                                    int act, void* stream) {
    AOTB_REQUIRE(in && w && out, "aotb_dwconv_nhwc_f32: null pointer");
    AOTB_REQUIRE(C % 4 == 0 && ldin % 4 == 0 && ldout % 4 == 0, "aotb_dwconv_nhwc_f32: channels must be %%4");
    const int Ho = (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
    const int Wo = (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
    if (KH == 5 && KW == 5 && stride == 1 && dil == 1) {
        const size_t tot4 = (size_t)B * Ho * ((Wo + 3) / 4) * (C / 4);
        launch(act == ACT_HSWISH ? dwconv_row4_kernel<5, true> : dwconv_row4_kernel<5>, dim3(grid_for(tot4, 128)), dim3(128), 0, (cudaStream_t)stream, in, w, bias, out, B, H, W,
               C, ldin, ldout, pad, act);
        return check_launch("aotb_dwconv_nhwc_f32");
    }
    const size_t total = (size_t)B * Ho * Wo * (C / 4);
    launch(act == ACT_HSWISH ? dwconv_kernel<true> : dwconv_kernel<>, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, in, w, bias, out, B, H, W, C, ldin, ldout,
                                                                         Ho, Wo, KH, KW, stride, pad, dil, act);
    return check_launch("aotb_dwconv_nhwc_f32");
}

extern "C" int aotb_bilinear_nhwc_f32(const float* in, float* out, int B, int H, int W, int C, int Ho, int Wo,
                                      int align_corners, void* stream) {
    AOTB_REQUIRE(in && out && C % 4 == 0 && Ho > 0 && Wo > 0, "aotb_bilinear_nhwc_f32: bad args");
    const size_t total = (size_t)B * Ho * Wo * (C / 4);
    launch(bilinear_nhwc_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, in, out, B, H, W, C, Ho, Wo,
                                                                                align_corners);
    return check_launch("aotb_bilinear_nhwc_f32");
}

extern "C" int aotb_eltwise_f32(int op, const float* a, int lda, const float* b, int ldb, float* out, int ldo,
                                int rows, int cols, float scalar, void* stream) {
    AOTB_REQUIRE(out && rows > 0 && cols > 0 && op >= 0 && op <= 5, "aotb_eltwise_f32: bad args");
    AOTB_REQUIRE(op == EW_FILL || a, "aotb_eltwise_f32: null a");
    const size_t total = (size_t)rows * cols;
    launch(eltwise_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, op, a, lda, b, ldb, out, ldo, rows, cols,
                                                                          scalar);
    return check_launch("aotb_eltwise_f32");
}
