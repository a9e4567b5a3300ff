// Implicit-GEMM convolution / linear layer, NHWC fp32, fp32-exact SIMT path.
//
//   out[m][n] = act( sum_k A(m,k) * Wt[k][n] + bias[n] + res[m][n] )
//   m -> (b, oy, ox)   k -> (ky, kx, ci)   A(m,k) = in[b, oy*s+ky*d-p, ox*s+kx*d-p, ci]  (0 outside)
//
// Replaces, on the per-frame path of the reference: every nn.Conv2d of the encoder
// (networks/encoders/resnet.py:34-54,140-157 with FrozenBatchNorm2d folded into Wt/bias,
// networks/layers/normalization.py:30-43), encoder_projector (networks/models/aot.py:19-21,83),
// the FPN convs (networks/decoders/fpn.py:34-58) and every nn.Linear of the LSTT / GPM blocks
// (networks/layers/transformer.py:321-367, 582-665; a Linear on [N,C] tokens is a 1x1 conv on
// NHWC with bs=1).  im2col is never materialised: the A tile is gathered straight from the
// NHWC activation with 128-bit loads along the channel axis.
//
// Layout: activations NHWC (pixel stride ldin/ldout/ldres may exceed the channel count so a
// kernel can read/write a channel slice of a wider buffer), weights [KH*KW*Cin][Cout].
// Tiling: BMxBNx16 per CTA, 256 threads, TMxTN register micro-tile, double-buffered smem.
#include "common.cuh"

namespace aotb {

struct ConvArgs {
    const float* in;
    const float* w;
    const float* bias;
    const float* res;
    float* out;
    int B, H, W, Cin, ldin;
    int Ho, Wo, Cout, ldout, ldres;
    int KH, KW, stride, pad, dil;
    int M, K;
    int act;
    int ovec;  // out base 16B-aligned and ldout % 4 == 0
};

template <int BM, int BN, int TM, int TN, bool AVEC, bool BVEC, bool HS = false>
__global__ void __launch_bounds__(256) conv_igemm_kernel(const ConvArgs p) {
    pdl_sync();
    constexpr int BK = 16;
    constexpr int PAD = 4;
    static_assert((BM / TM) * (BN / TN) == 256, "256 threads");
    static_assert(TM == 4 || TM == 8, "TM");
    static_assert(TN == 2 || TN == 4 || TN == 8, "TN");
    __shared__ __align__(16) float As[2][BK][BM + PAD];
    __shared__ __align__(16) float Bs[2][BK][BN + PAD];

    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int HoWo = p.Ho * p.Wo;
    const bool pointwise = (p.KH * p.KW == 1);

    // ---- per-thread A-row bookkeeping (rows are fixed across the K loop)
    constexpr int A_IT = AVEC ? (BM * BK / 4 + 255) / 256 : (BM * BK) / 256;
    int a_iy0[A_IT], a_ix0[A_IT];
    const float* a_base[A_IT];
#pragma unroll
    for (int i = 0; i < A_IT; ++i) {
        const int f = tid + i * 256;
        const int row = AVEC ? (f >> 2) : (f >> 4);
        const int m = m0 + row;
        if (m < p.M && row < BM) {
            const int b = m / HoWo;
            const int r = m - b * HoWo;
            const int oy = r / p.Wo, ox = r - oy * p.Wo;
            a_iy0[i] = oy * p.stride - p.pad;
            a_ix0[i] = ox * p.stride - p.pad;
            a_base[i] = p.in + (size_t)b * p.H * p.W * p.ldin;
        } else {
            a_iy0[i] = -(1 << 28);
            a_ix0[i] = -(1 << 28);
            a_base[i] = p.in;
        }
    }

    constexpr int B_IT = BVEC ? (BK * BN / 4 + 255) / 256 : (BK * BN + 255) / 256;
    float4 a_reg4[AVEC ? A_IT : 1];
    float a_reg1[AVEC ? 1 : A_IT];
    float4 b_reg4[BVEC ? B_IT : 1];
    float b_reg1[BVEC ? 1 : B_IT];

    auto load_tile = [&](int kt) {
        const int k0 = kt * BK;
        if constexpr (AVEC) {
            int ky = 0, kx = 0, ci0 = k0;
            if (!pointwise) {
                const int kk = k0 / p.Cin;
                ci0 = k0 - kk * p.Cin;
                ky = kk / p.KW;
                kx = kk - ky * p.KW;
            }
#pragma unroll
            for (int i = 0; i < A_IT; ++i) {
                const int f = tid + i * 256;
                const int kq = f & 3;
                const int iy = a_iy0[i] + ky * p.dil, ix = a_ix0[i] + kx * p.dil;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if ((BM * BK / 4 >= 256 * (i + 1) || f < BM * BK / 4) && iy >= 0 && iy < p.H && ix >= 0 &&
                    ix < p.W && (k0 + kq * 4) < p.K)
                    v = __ldg(reinterpret_cast<const float4*>(a_base[i] + ((size_t)iy * p.W + ix) * p.ldin + ci0 +
                                                              kq * 4));
                a_reg4[i] = v;
            }
        } else {
#pragma unroll
            for (int i = 0; i < A_IT; ++i) {
                const int f = tid + i * 256;
                const int k = k0 + (f & 15);
                float v = 0.f;
                if (k < p.K) {
                    const int kk = k / p.Cin;
                    const int ci = k - kk * p.Cin;
                    const int ky = kk / p.KW, kx = kk - ky * p.KW;
                    const int iy = a_iy0[i] + ky * p.dil, ix = a_ix0[i] + kx * p.dil;
                    if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W)
                        v = __ldg(a_base[i] + ((size_t)iy * p.W + ix) * p.ldin + ci);
                }
                a_reg1[i] = v;
            }
        }
        if constexpr (BVEC) {
#pragma unroll
            for (int i = 0; i < B_IT; ++i) {
                const int f = tid + i * 256;
                const int brow = f / (BN / 4), bq = f - brow * (BN / 4);
                const int k = k0 + brow, n = n0 + bq * 4;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (f < BK * BN / 4 && k < p.K && n < p.Cout)
                    v = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)k * p.Cout + n));
                b_reg4[i] = v;
            }
        } else {
#pragma unroll
            for (int i = 0; i < B_IT; ++i) {
                const int f = tid + i * 256;
                const int brow = f / BN, bn = f - brow * BN;
                const int k = k0 + brow, n = n0 + bn;
                float v = 0.f;
                if (f < BK * BN && k < p.K && n < p.Cout) v = __ldg(p.w + (size_t)k * p.Cout + n);
                b_reg1[i] = v;
            }
        }
    };

    auto store_tile = [&](int buf) {
        if constexpr (AVEC) {
#pragma unroll
            for (int i = 0; i < A_IT; ++i) {
                const int f = tid + i * 256;
                if (BM * BK / 4 >= 256 * (i + 1) || f < BM * BK / 4) {
                    const int row = f >> 2, kq = f & 3;
                    As[buf][kq * 4 + 0][row] = a_reg4[i].x;
                    As[buf][kq * 4 + 1][row] = a_reg4[i].y;
                    As[buf][kq * 4 + 2][row] = a_reg4[i].z;
                    As[buf][kq * 4 + 3][row] = a_reg4[i].w;
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < A_IT; ++i) {
                const int f = tid + i * 256;
                As[buf][f & 15][f >> 4] = a_reg1[i];
            }
        }
        if constexpr (BVEC) {
#pragma unroll
            for (int i = 0; i < B_IT; ++i) {
                const int f = tid + i * 256;
                if (f < BK * BN / 4) {
                    const int brow = f / (BN / 4), bq = f - brow * (BN / 4);
                    *reinterpret_cast<float4*>(&Bs[buf][brow][bq * 4]) = b_reg4[i];
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < B_IT; ++i) {
                const int f = tid + i * 256;
                if (f < BK * BN) Bs[buf][f / BN][f % BN] = b_reg1[i];
            }
        }
    };

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    const int KT = (p.K + BK - 1) / BK;
    load_tile(0);
    store_tile(0);
    __syncthreads();
    for (int kt = 0; kt < KT; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < KT) load_tile(kt + 1);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TN];
            {
                const float4 v = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
                a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
                if constexpr (TM == 8) {
                    const float4 u = *reinterpret_cast<const float4*>(&As[buf][k][BM / 2 + ty * 4]);
                    a[4] = u.x; a[5] = u.y; a[6] = u.z; a[7] = u.w;
                }
            }
            if constexpr (TN == 2) {
                const float2 v = *reinterpret_cast<const float2*>(&Bs[buf][k][tx * 2]);
                b[0] = v.x; b[1] = v.y;
            } else {
                const float4 v = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
                b[0] = v.x; b[1] = v.y; b[2] = v.z; b[3] = v.w;
                if constexpr (TN == 8) {
                    const float4 u = *reinterpret_cast<const float4*>(&Bs[buf][k][BN / 2 + tx * 4]);
                    b[4] = u.x; b[5] = u.y; b[6] = u.z; b[7] = u.w;
                }
            }
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < KT) {
            store_tile(buf ^ 1);
            __syncthreads();
        }
    }

    // ---- epilogue: bias + residual + activation
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int row = (i < 4) ? (ty * 4 + i) : (BM / 2 + ty * 4 + (i - 4));
        const int m = m0 + row;
        if (m >= p.M) continue;
        float* orow = p.out + (size_t)m * p.ldout;
        const float* rrow = p.res ? p.res + (size_t)m * p.ldres : nullptr;
#pragma unroll
        for (int jg = 0; jg < (TN == 2 ? 1 : TN / 4); ++jg) {
            constexpr int G = (TN == 2) ? 2 : 4;
            const int col = (TN == 2) ? tx * 2 : (jg == 0 ? tx * 4 : BN / 2 + tx * 4);
            const int n = n0 + col;
            float v[G];
#pragma unroll
            for (int j = 0; j < G; ++j) {
                const int nn = n + j;
                float x = acc[i][jg * 4 + j];
                if (nn < p.Cout) {
                    if (p.bias) x += __ldg(p.bias + nn);
                    if (rrow) x += rrow[nn];
                    x = apply_act_or_hswish<HS>(x, p.act);
                }
                v[j] = x;
            }
            if (BVEC && G == 4 && n + 3 < p.Cout && p.ovec) {
                *reinterpret_cast<float4*>(orow + n) = make_float4(v[0], v[1], v[2], v[3]);
            } else {
#pragma unroll
                for (int j = 0; j < G; ++j)
                    if (n + j < p.Cout) orow[n + j] = v[j];
            }
        }
    }
}

template <int BM, int BN, int TM, int TN, bool AVEC, bool BVEC>
static void launch_conv(const ConvArgs& a, cudaStream_t st) {
    dim3 grid(cdiv(a.M, BM), cdiv(a.Cout, BN));
    if (a.act == ACT_HSWISH)
        launch(conv_igemm_kernel<BM, BN, TM, TN, AVEC, BVEC, true>, dim3(grid), dim3(256), 0, st, a);
    else
        launch(conv_igemm_kernel<BM, BN, TM, TN, AVEC, BVEC>, dim3(grid), dim3(256), 0, st, a);
}

int conv2d_dispatch(const ConvArgs& a, cudaStream_t st) {
    const bool aligned_in = ((uintptr_t)a.in % 16 == 0) && (a.ldin % 4 == 0);
    const bool avec = aligned_in && (a.Cin % 4 == 0) && (a.KH * a.KW == 1 || a.Cin % 16 == 0);
    const bool bvec = (a.Cout % 4 == 0) && ((uintptr_t)a.w % 16 == 0);
    auto ctas = [&](int bm, int bn) { return (long)cdiv(a.M, bm) * cdiv(a.Cout, bn); };
    if (avec && bvec) {
        if (a.Cout >= 128 && ctas(128, 128) >= 132)
            launch_conv<128, 128, 8, 8, true, true>(a, st);
        else if (a.Cout >= 64 && ctas(128, 64) >= 132)
            launch_conv<128, 64, 8, 4, true, true>(a, st);
        else
            launch_conv<64, 64, 4, 4, true, true>(a, st);
    } else if (avec && !bvec) {
        launch_conv<128, 32, 8, 2, true, false>(a, st);
    } else if (!avec && bvec) {
        if (ctas(128, 64) >= 132)
            launch_conv<128, 64, 8, 4, false, true>(a, st);
        else
            launch_conv<64, 64, 4, 4, false, true>(a, st);
    } else {
        launch_conv<128, 32, 8, 2, false, false>(a, st);
    }
    return check_launch("aotb_conv2d_nhwc_f32");
}

}  // namespace aotb

extern "C" int aotb_conv2d_nhwc_f32(const float* in, const float* w, const float* bias, const float* res,
                                    float* out, int B, int H, int W, int Cin, int ldin, int Cout, int ldout,
                                    int ldres, int KH, int KW, int stride, int pad, int dil, int act,
                                    void* stream) {
    using namespace aotb;
    AOTB_REQUIRE(in && w && out, "aotb_conv2d_nhwc_f32: null pointer");
    AOTB_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && KH > 0 && KW > 0 && stride > 0 && dil > 0,
                 "aotb_conv2d_nhwc_f32: bad shape");
    AOTB_REQUIRE(ldin >= Cin && ldout >= Cout && (!res || ldres >= Cout), "aotb_conv2d_nhwc_f32: bad ld");
    ConvArgs a;
    a.in = in; a.w = w; a.bias = bias; a.res = res; a.out = out;
    a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.ldin = ldin;
    a.Ho = (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
    a.Wo = (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
    AOTB_REQUIRE(a.Ho > 0 && a.Wo > 0, "aotb_conv2d_nhwc_f32: empty output");
    a.Cout = Cout; a.ldout = ldout; a.ldres = ldres;
    a.KH = KH; a.KW = KW; a.stride = stride; a.pad = pad; a.dil = dil;
    a.M = B * a.Ho * a.Wo; a.K = KH * KW * Cin; a.act = act;
    a.ovec = ((uintptr_t)out % 16 == 0) && (ldout % 4 == 0);
    return conv2d_dispatch(a, (cudaStream_t)stream);
}

// Linear layer on [M, K] tokens: out[M, N] = act(in @ Wt + bias + res); Wt is [K][N].
extern "C" int aotb_linear_f32(const float* in, const float* wt, const float* bias, const float* res, float* out,
                               int M, int K, int ldin, int N, int ldout, int ldres, int act, void* stream) {
    return aotb_conv2d_nhwc_f32(in, wt, bias, res, out, 1, M, 1, K, ldin, N, ldout, ldres, 1, 1, 1, 0, 1, act, stream);
}
