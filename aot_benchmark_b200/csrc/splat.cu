// Split-attention (ResNeSt), squeeze-excite (MobileNetV3) and average pooling, NHWC fp32.
//
// Reference sites: networks/encoders/resnest/splat.py:88-115 (SplAtConv2d.forward after its grouped conv + bn0 + ReLU:
// gap, fc1 + bn1 + ReLU, fc2, rSoftMax :118-132, the attention-weighted sum of the radix splits),
// networks/encoders/resnest/resnet.py:72-73,152-153 (avd AvgPool2d(3, stride, padding=1) after conv2) and :330-342
// (avg_down AvgPool2d(stride, stride, ceil_mode=True, count_include_pad=False) in front of the downsample conv);
// networks/encoders/mobilenetv3.py:51-65 (SELayer: mean over the map, fc1 + ReLU, fc2 + h_sigmoid, x * gate).
//
// The pixel reduction of the split attention spans many CTAs.  Each CTA writes the per-channel sum of its fixed pixel range
// to its own slot of the workspace (double), and the CTA that takes the last ticket of the launch counter adds the slots in
// CTA order, runs the two small GEMVs and the final gate (radix softmax or h_sigmoid), and resets the counter: the result
// does not depend on CTA scheduling, and every launch (or graph replay) starts from a zero counter.
//
// Every kernel here also takes a batch of B images stacked densely over pixels (blockIdx.y = image): each image of a batch
// gets the grid, pixel ranges, workspace partials and counter a one-image launch would give it, so image b of a batched
// launch is bitwise equal to a one-image launch on image b.
#include "common.cuh"
#include <cstdint>

namespace aotb {

constexpr int SPLAT_THREADS = 256;
constexpr int SPLAT_MAX_CTAS = 264;          // 2 per SM
constexpr int SPLAT_MAX_C = 1024;         // one float4 channel group per thread: C / 4 <= SPLAT_THREADS
constexpr int SPLAT_MAX_RADIX = 4;
constexpr size_t SPLAT_HDR = 256;            // launch counter

enum Gate { GATE_RSOFTMAX = 0, GATE_HSIGMOID = 1 };

// x [HW][ldx] holds radix splits of C channels: split r = channels [r*C, (r+1)*C).
// w1 [C][inter] (fc1 with bn1 folded), b1 [inter], w2 [inter][radix*C] (fc2), b2 [radix*C] -> att [radix*C] (radix-major).
// GATE_RSOFTMAX: softmax across the radix (ResNeSt); GATE_HSIGMOID: radix 1, att = h_sigmoid(logit) (squeeze-excite).
template <int GATE>
__global__ void __launch_bounds__(SPLAT_THREADS)
splat_attention_kernel(const float* __restrict__ x, int ldx, int HW, int C, int radix, const float* __restrict__ w1,
                       const float* __restrict__ b1, int inter, const float* __restrict__ w2, const float* __restrict__ b2,
                       float* __restrict__ att, double* __restrict__ partial, unsigned* __restrict__ counter) {
    pdl_sync();
    // image blockIdx.y: its pixels here, its CTA partials, its own launch counter and its gate where they are used
    x += (size_t)blockIdx.y * HW * ldx;
    __shared__ float4 red[SPLAT_THREADS];
    __shared__ float gap[SPLAT_MAX_C];
    __shared__ float hid[SPLAT_MAX_C];
    __shared__ float logit[SPLAT_MAX_RADIX * SPLAT_MAX_C];
    __shared__ unsigned last;
    const int tid = threadIdx.x;
    const int C4 = C >> 2, R = SPLAT_THREADS / C4;                 // R pixel rows per pass, one float4 channel group per thread
    const int cg = tid % C4, pr = tid / C4;
    const int per = (HW + gridDim.x - 1) / gridDim.x;
    const int p0 = blockIdx.x * per, p1 = min(HW, p0 + per);
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (pr < R) {
        for (int p = p0 + pr; p < p1; p += R) {
            const float* xp = x + (size_t)p * ldx + cg * 4;
            for (int r = 0; r < radix; ++r) {
                const float4 v = *reinterpret_cast<const float4*>(xp + r * C);
                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
            }
        }
    }
    red[tid] = s;
    __syncthreads();
    // per-CTA channel sums: rows added in a fixed order
    const float* redf = reinterpret_cast<const float*>(red);
    for (int c = tid; c < C; c += SPLAT_THREADS) {
        double a = 0.0;
        for (int r = 0; r < R; ++r) a += (double)redf[r * C + c];
        partial[((size_t)blockIdx.y * SPLAT_MAX_CTAS + blockIdx.x) * C + c] = a;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) last = atomicAdd(counter + blockIdx.y, 1u) == gridDim.x - 1 ? 1u : 0u;
    __syncthreads();
    if (!last) return;
    __threadfence();
    // ---- last CTA: gap = mean over pixels of the sum of the splits (CTA partials in CTA order)
    const volatile double* pv = partial + (size_t)blockIdx.y * SPLAT_MAX_CTAS * C;
    for (int c = tid; c < C; c += SPLAT_THREADS) {
        double a = 0.0;
        for (int b = 0; b < (int)gridDim.x; ++b) a += pv[(size_t)b * C + c];
        gap[c] = (float)(a / (double)HW);
    }
    __syncthreads();
    // fc1 (bn1 folded) + ReLU
    for (int j = tid; j < inter; j += SPLAT_THREADS) {
        float a = b1[j];
        for (int c = 0; c < C; ++c) a = fmaf(gap[c], w1[(size_t)c * inter + j], a);
        hid[j] = fmaxf(a, 0.f);
    }
    __syncthreads();
    // fc2
    const int RC = radix * C;
    for (int k = tid; k < RC; k += SPLAT_THREADS) {
        float a = b2[k];
        for (int j = 0; j < inter; ++j) a = fmaf(hid[j], w2[(size_t)j * RC + k], a);
        logit[k] = a;
    }
    __syncthreads();
    att += (size_t)blockIdx.y * radix * C;
    counter += blockIdx.y;
    if (GATE == GATE_HSIGMOID) {
        for (int c = tid; c < C; c += SPLAT_THREADS) att[c] = hsigmoid(logit[c]);
        if (tid == 0) *counter = 0u;
        return;
    }
    // rSoftMax: softmax across the radix for every channel (cardinality 1), written radix-major
    for (int c = tid; c < C; c += SPLAT_THREADS) {
        float m = logit[c];
        for (int r = 1; r < radix; ++r) m = fmaxf(m, logit[r * C + c]);
        float e[SPLAT_MAX_RADIX], den = 0.f;
        for (int r = 0; r < radix; ++r) { e[r] = expf(logit[r * C + c] - m); den += e[r]; }
        for (int r = 0; r < radix; ++r) att[r * C + c] = e[r] / den;
    }
    if (tid == 0) *counter = 0u;          // ready for the next launch
}

// nn.AvgPool2d window of output (oy, ox) with PyTorch's divisor rule: the padded extent is clipped at H + pad, the divisor is
// its size (count_include_pad) or the size of the part inside the map.
struct PoolWin {
    int y0, y1, x0, x1;
    float div;
};
__device__ __forceinline__ PoolWin pool_window(int oy, int ox, int H, int W, int k, int s, int pad, int include_pad) {
    int y0 = oy * s - pad, x0 = ox * s - pad;
    int y1 = min(y0 + k, H + pad), x1 = min(x0 + k, W + pad);
    const int padded = (y1 - y0) * (x1 - x0);
    y0 = max(y0, 0); x0 = max(x0, 0);
    y1 = min(y1, H); x1 = min(x1, W);
    const int div = include_pad ? padded : (y1 - y0) * (x1 - x0);
    return PoolWin{y0, y1, x0, x1, (float)div};
}

// out [Ho][Wo][ldo] (C channels) = act(sum_r att[r*C + c] * x[r*C + c]), optionally average-pooled 3x3 / stride / pad 1 with
// padding counted before the activation (pool_stride 0: no pool, Ho = H, Wo = W).  The radix is a template argument so the
// weights stay in registers.  With radix 1 the sum is the single rounded product att * x, as the reference's x * y computes it.
template <int RADIX>
__global__ void splat_combine_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ att, float* __restrict__ out,
                                     int ldo, int H, int W, int C, int pool_stride, int Ho, int Wo, int act) {
    pdl_sync();
    x += (size_t)blockIdx.y * H * W * ldx;              // image blockIdx.y of a batch
    att += (size_t)blockIdx.y * RADIX * C;
    out += (size_t)blockIdx.y * Ho * Wo * ldo;
    const int C4 = C >> 2;
    const size_t total = (size_t)Ho * Wo * C4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4) * 4;
        const size_t t = i / C4;
        const int ox = (int)(t % Wo), oy = (int)(t / Wo);
        float4 a[RADIX];
#pragma unroll
        for (int r = 0; r < RADIX; ++r) a[r] = __ldg(reinterpret_cast<const float4*>(att + r * C + c));
        auto comb = [&](int y, int xx) {
            const float* xp = x + ((size_t)y * W + xx) * ldx + c;
            float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int r = 0; r < RADIX; ++r) {
                const float4 v = *reinterpret_cast<const float4*>(xp + r * C);
                o.x = fmaf(a[r].x, v.x, o.x); o.y = fmaf(a[r].y, v.y, o.y);
                o.z = fmaf(a[r].z, v.z, o.z); o.w = fmaf(a[r].w, v.w, o.w);
            }
            return o;
        };
        float4 o;
        if (pool_stride == 0) {
            o = comb(oy, ox);
        } else {
            const PoolWin pw = pool_window(oy, ox, H, W, 3, pool_stride, 1, 1);
            o = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int y = pw.y0; y < pw.y1; ++y)
                for (int xx = pw.x0; xx < pw.x1; ++xx) {
                    const float4 v = comb(y, xx);
                    o.x += v.x; o.y += v.y; o.z += v.z; o.w += v.w;
                }
            o.x /= pw.div; o.y /= pw.div; o.z /= pw.div; o.w /= pw.div;
        }
        o.x = apply_act_hs(o.x, act); o.y = apply_act_hs(o.y, act); o.z = apply_act_hs(o.z, act); o.w = apply_act_hs(o.w, act);
        *reinterpret_cast<float4*>(out + ((size_t)oy * Wo + ox) * ldo + c) = o;
    }
}

__global__ void avgpool_kernel(const float* __restrict__ in, int ldin, float* __restrict__ out, int ldo, int B, int H, int W,
                               int C, int Ho, int Wo, int k, int s, int pad, int include_pad) {
    pdl_sync();
    const int C4 = C >> 2;
    const size_t total = (size_t)B * Ho * Wo * C4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4) * 4;
        size_t t = i / C4;
        const int ox = (int)(t % Wo);
        t /= Wo;
        const int oy = (int)(t % Ho), b = (int)(t / Ho);
        const PoolWin pw = pool_window(oy, ox, H, W, k, s, pad, include_pad);
        const float* ib = in + (size_t)b * H * W * ldin + c;
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int y = pw.y0; y < pw.y1; ++y)
            for (int x = pw.x0; x < pw.x1; ++x) {
                const float4 v = *reinterpret_cast<const float4*>(ib + ((size_t)y * W + x) * ldin);
                o.x += v.x; o.y += v.y; o.z += v.z; o.w += v.w;
            }
        o.x /= pw.div; o.y /= pw.div; o.z /= pw.div; o.w /= pw.div;
        *reinterpret_cast<float4*>(out + (((size_t)b * Ho + oy) * Wo + ox) * ldo + c) = o;
    }
}

// nn.AvgPool2d output extent (pooling_output_shape of PyTorch, dilation 1)
static int pool_out(int n, int k, int s, int pad, int ceil_mode) {
    int o = (n + 2 * pad - k + (ceil_mode ? s - 1 : 0)) / s + 1;
    if (ceil_mode && (o - 1) * s >= n + pad) --o;
    return o;
}

static int grid_for(size_t total) {
    size_t g = (total + 255) / 256;
    return (int)(g > 132 * 16 ? 132 * 16 : (g < 1 ? 1 : g));
}

}  // namespace aotb

using namespace aotb;

// B counters in the header, then SPLAT_MAX_CTAS partial rows per image; B = 1 is the one-image layout
extern "C" size_t aotb_splat_workspace_batched_bytes(int C, int B) {
    const size_t b = B > 0 ? (size_t)B : 0;
    const size_t hdr = (b * sizeof(unsigned) + SPLAT_HDR - 1) / SPLAT_HDR * SPLAT_HDR;
    return (hdr > SPLAT_HDR ? hdr : SPLAT_HDR) + b * (size_t)SPLAT_MAX_CTAS * (size_t)(C > 0 ? C : 0) * sizeof(double);
}

extern "C" size_t aotb_splat_workspace_bytes(int C) { return aotb_splat_workspace_batched_bytes(C, 1); }

static double* splat_partials(void* workspace, int B) {
    const size_t hdr = ((size_t)B * sizeof(unsigned) + SPLAT_HDR - 1) / SPLAT_HDR * SPLAT_HDR;
    return (double*)((uint8_t*)workspace + (hdr > SPLAT_HDR ? hdr : SPLAT_HDR));
}

extern "C" int aotb_splat_attention_batched_f32(const float* x, int ldx, int B, int HW, int C, int radix, const float* w1,
                                                const float* b1, int inter, const float* w2, const float* b2, float* att,
                                                void* workspace, void* stream) {
    AOTB_REQUIRE(x && w1 && b1 && w2 && b2 && att && workspace, "aotb_splat_attention_f32: null pointer");
    AOTB_REQUIRE(B > 0 && B <= 65535 && HW > 0 && C > 0 && C % 4 == 0 && C <= SPLAT_MAX_C && inter > 0 &&
                     inter <= SPLAT_MAX_C && radix >= 2 && radix <= SPLAT_MAX_RADIX && ldx >= radix * C,
                 "aotb_splat_attention_f32: need B > 0, HW > 0, C %% 4 == 0, C and inter <= %d, 2 <= radix <= %d, "
                 "ldx >= radix * C", SPLAT_MAX_C, SPLAT_MAX_RADIX);
    AOTB_REQUIRE(ldx % 4 == 0 && (uintptr_t)x % 16 == 0, "aotb_splat_attention_f32: x needs 16-byte aligned rows");
    const int rows = (SPLAT_THREADS / (C / 4)) * 8;          // ~8 float4 loads per thread and split
    int ctas = cdiv(HW, rows);
    ctas = ctas > SPLAT_MAX_CTAS ? SPLAT_MAX_CTAS : ctas;
    launch(splat_attention_kernel<GATE_RSOFTMAX>, dim3(ctas, B), dim3(SPLAT_THREADS), 0, (cudaStream_t)stream, x, ldx, HW,
           C, radix, w1, b1, inter, w2, b2, att, splat_partials(workspace, B), (unsigned*)workspace);
    return check_launch("aotb_splat_attention_f32");
}

extern "C" int aotb_splat_attention_f32(const float* x, int ldx, int HW, int C, int radix, const float* w1, const float* b1,
                                        int inter, const float* w2, const float* b2, float* att, void* workspace,
                                        void* stream) {
    return aotb_splat_attention_batched_f32(x, ldx, 1, HW, C, radix, w1, b1, inter, w2, b2, att, workspace, stream);
}

extern "C" int aotb_splat_combine_batched_f32(const float* x, int ldx, const float* att, float* out, int ldo, int B, int H,
                                              int W, int C, int radix, int pool_stride, void* stream) {
    AOTB_REQUIRE(x && att && out, "aotb_splat_combine_f32: null pointer");
    AOTB_REQUIRE(B > 0 && B <= 65535 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && radix >= 1 && radix <= SPLAT_MAX_RADIX &&
                     ldx >= radix * C && ldo >= C && pool_stride >= 0,
                 "aotb_splat_combine_f32: bad shape");
    AOTB_REQUIRE(ldx % 4 == 0 && ldo % 4 == 0 && (uintptr_t)x % 16 == 0 && (uintptr_t)out % 16 == 0 &&
                     (uintptr_t)att % 16 == 0,
                 "aotb_splat_combine_f32: 16-byte alignment required");
    const int Ho = pool_stride ? pool_out(H, 3, pool_stride, 1, 0) : H;
    const int Wo = pool_stride ? pool_out(W, 3, pool_stride, 1, 0) : W;
    const size_t total = (size_t)Ho * Wo * (C / 4);
    auto kernel = radix == 1 ? splat_combine_kernel<1> : radix == 2 ? splat_combine_kernel<2>
                : radix == 3 ? splat_combine_kernel<3> : splat_combine_kernel<4>;
    launch(kernel, dim3(grid_for(total), B), dim3(256), 0, (cudaStream_t)stream, x, ldx, att, out, ldo, H, W, C, pool_stride,
           Ho, Wo, (int)ACT_NONE);
    return check_launch("aotb_splat_combine_f32");
}

extern "C" int aotb_splat_combine_f32(const float* x, int ldx, const float* att, float* out, int ldo, int H, int W, int C,
                                      int radix, int pool_stride, void* stream) {
    return aotb_splat_combine_batched_f32(x, ldx, att, out, ldo, 1, H, W, C, radix, pool_stride, stream);
}

extern "C" int aotb_se_gate_batched_f32(const float* x, int ldx, int B, int HW, int C, const float* w1, const float* b1,
                                        int inter, const float* w2, const float* b2, float* gate, void* workspace,
                                        void* stream) {
    AOTB_REQUIRE(x && w1 && b1 && w2 && b2 && gate && workspace, "aotb_se_gate_f32: null pointer");
    AOTB_REQUIRE(B > 0 && B <= 65535 && HW > 0 && C > 0 && C % 4 == 0 && C <= SPLAT_MAX_C && inter > 0 &&
                     inter <= SPLAT_MAX_C && ldx >= C,
                 "aotb_se_gate_f32: need B > 0, HW > 0, C %% 4 == 0, C and inter <= %d, ldx >= C", SPLAT_MAX_C);
    AOTB_REQUIRE(ldx % 4 == 0 && (uintptr_t)x % 16 == 0, "aotb_se_gate_f32: x needs 16-byte aligned rows");
    const int rows = (SPLAT_THREADS / (C / 4)) * 8;
    int ctas = cdiv(HW, rows);
    ctas = ctas > SPLAT_MAX_CTAS ? SPLAT_MAX_CTAS : ctas;
    launch(splat_attention_kernel<GATE_HSIGMOID>, dim3(ctas, B), dim3(SPLAT_THREADS), 0, (cudaStream_t)stream, x, ldx, HW, C,
           1, w1, b1, inter, w2, b2, gate, splat_partials(workspace, B), (unsigned*)workspace);
    return check_launch("aotb_se_gate_f32");
}

extern "C" int aotb_se_gate_f32(const float* x, int ldx, int HW, int C, const float* w1, const float* b1, int inter,
                                const float* w2, const float* b2, float* gate, void* workspace, void* stream) {
    return aotb_se_gate_batched_f32(x, ldx, 1, HW, C, w1, b1, inter, w2, b2, gate, workspace, stream);
}

extern "C" int aotb_gate_scale_batched_f32(const float* x, int ldx, const float* gate, float* out, int ldo, int B, int HW,
                                           int C, int act, void* stream) {
    AOTB_REQUIRE(x && gate && out, "aotb_gate_scale_f32: null pointer");
    AOTB_REQUIRE(B > 0 && B <= 65535 && HW > 0 && C > 0 && C % 4 == 0 && ldx >= C && ldo >= C && act >= ACT_NONE &&
                     act <= ACT_HSWISH,
                 "aotb_gate_scale_f32: bad shape or activation");
    AOTB_REQUIRE(ldx % 4 == 0 && ldo % 4 == 0 && (uintptr_t)x % 16 == 0 && (uintptr_t)out % 16 == 0 &&
                     (uintptr_t)gate % 16 == 0,
                 "aotb_gate_scale_f32: 16-byte alignment required");
    const size_t total = (size_t)HW * (C / 4);
    launch(splat_combine_kernel<1>, dim3(grid_for(total), B), dim3(256), 0, (cudaStream_t)stream, x, ldx, gate, out, ldo, 1,
           HW, C, 0, 1, HW, act);
    return check_launch("aotb_gate_scale_f32");
}

extern "C" int aotb_gate_scale_f32(const float* x, int ldx, const float* gate, float* out, int ldo, int HW, int C, int act,
                                   void* stream) {
    return aotb_gate_scale_batched_f32(x, ldx, gate, out, ldo, 1, HW, C, act, stream);
}

extern "C" int aotb_avgpool_nhwc_f32(const float* in, int ldin, float* out, int ldo, int B, int H, int W, int C, int k,
                                     int s, int pad, int ceil_mode, int count_include_pad, void* stream) {
    AOTB_REQUIRE(in && out, "aotb_avgpool_nhwc_f32: null pointer");
    AOTB_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && ldin >= C && ldo >= C && k > 0 && s > 0 && pad >= 0 &&
                     2 * pad <= k,
                 "aotb_avgpool_nhwc_f32: bad shape (pad must be at most half the kernel, as in nn.AvgPool2d)");
    AOTB_REQUIRE(ldin % 4 == 0 && ldo % 4 == 0 && (uintptr_t)in % 16 == 0 && (uintptr_t)out % 16 == 0,
                 "aotb_avgpool_nhwc_f32: 16-byte alignment required");
    const int Ho = pool_out(H, k, s, pad, ceil_mode), Wo = pool_out(W, k, s, pad, ceil_mode);
    AOTB_REQUIRE(Ho > 0 && Wo > 0, "aotb_avgpool_nhwc_f32: empty output");
    const size_t total = (size_t)B * Ho * Wo * (C / 4);
    launch(avgpool_kernel, dim3(grid_for(total)), dim3(256), 0, (cudaStream_t)stream, in, ldin, out, ldo, B, H, W, C, Ho, Wo,
           k, s, pad, count_include_pad ? 1 : 0);
    return check_launch("aotb_avgpool_nhwc_f32");
}
