// Identity-bank embedding (K4), logit post-processing (K9) and memory-bank append (K10).
//
// K4  one_hot_mask (utils/image.py:69-74) -> patch_wise_id_bank Conv2d(11->C, k17 s16 p8 | k16 s16 p0)
//     (networks/models/aot.py:50-63,76-79; aot_engine.py:168-179) [+ LayerNorm over C for DeAOT,
//     deaot.py:51-55].  A convolution of a one-hot image is a gather-sum of weight columns:
//        id[y,x,c] = b[c] + sum_{ky,kx in frame} W[c, mask[s*y+ky-p, s*x+kx-p], ky, kx]
//     so the [1,11,H,W] one-hot tensor (18 MB/frame at 480p) and 96 % of the conv FLOPs vanish.
// K9  aot_engine.py:367-378: ids > obj_num are set to -1e10 at stride-4 resolution, then
//     F.interpolate(bilinear, align_corners=cfg) to the output size (NCHW result for the caller).
// K10 aot_engine.py:291-305 re-copies the whole bank with torch.cat on every update; here the new
//     frame's rows are written in place into a pre-allocated bank (row order is append, not the
//     reference's prepend -- softmax attention is permutation invariant over keys).
#include "common.cuh"

#include <cuda_fp16.h>

namespace aotb {

// weights re-laid out as wt[(ky*KW + kx) * NID + id][C]
template <bool LN>
__global__ void __launch_bounds__(256) id_embed_kernel(const float* __restrict__ mask, int Hm, int Wm,
                                                       const float* __restrict__ wt, const float* __restrict__ bias,
                                                       const float* __restrict__ ln_g, const float* __restrict__ ln_b,
                                                       float* __restrict__ out, int ldo, int ho, int wo, int C,
                                                       int NID, int KS, int stride, int pad) {
    pdl_sync();
    __shared__ int ids[17 * 17];
    __shared__ float red[2][8];
    const int pix = blockIdx.x;
    const int oy = pix / wo, ox = pix - oy * wo;
    for (int t = threadIdx.x; t < KS * KS; t += blockDim.x) {
        const int ky = t / KS, kx = t - ky * KS;
        const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
        int id = -1;
        if (iy >= 0 && iy < Hm && ix >= 0 && ix < Wm) {
            const float v = __ldg(mask + (size_t)iy * Wm + ix);
            const int iv = (int)v;
            if ((float)iv == v && iv >= 0 && iv < NID) id = iv;   // (mask == arange).float()
        }
        ids[t] = id;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float acc = 0.f;
        for (int t = 0; t < KS * KS; ++t) {
            const int id = ids[t];
            if (id >= 0) acc += __ldg(wt + ((size_t)t * NID + id) * C + c);
        }
        acc += __ldg(bias + c);
        if constexpr (!LN) out[(size_t)pix * ldo + c] = acc;
        else {
            // C == blockDim.x == 256 in the LN variant (checked on the host)
            float s = warp_sum(acc);
            const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
            if (lane == 0) red[0][wid] = s;
            __syncthreads();
            float tot = 0.f;
            for (int w2 = 0; w2 < 8; ++w2) tot += red[0][w2];
            const float mean = tot / (float)C;
            const float d = acc - mean;
            float q = warp_sum(d * d);
            if (lane == 0) red[1][wid] = q;
            __syncthreads();
            float tq = 0.f;
            for (int w2 = 0; w2 < 8; ++w2) tq += red[1][w2];
            const float rstd = rsqrtf(tq / (float)C + 1e-5f);
            out[(size_t)pix * ldo + c] = d * rstd * __ldg(ln_g + c) + __ldg(ln_b + c);
        }
    }
}

// Run-length variant: a label map is piecewise constant, so along each of the KS window rows the ids form a few runs.
// With wp[ky][j][id][c] = sum_{kx < j} W[c, id, ky, kx] (exclusive prefix along kx, built in float64 by the host) a run
// [a, b) of one id contributes wp[ky][b][id] - wp[ky][a][id]: ~2 table rows per run instead of one per tap
// (typically ~40 instead of 289 one-KB rows per output pixel).
template <bool LN>
__device__ __forceinline__ void id_embed_runs_cta(const float* __restrict__ mask, int Hm, int Wm,
                                                  const float* __restrict__ wp, const float* __restrict__ bias,
                                                  const float* __restrict__ ln_g, const float* __restrict__ ln_b,
                                                  float* __restrict__ out, int ldo, int ho, int wo, int C,
                                                  int NID, int KS, int stride, int pad) {
    pdl_sync();
    __shared__ int ids[17 * 17];
    __shared__ int run_pos[17 * 18];     // per row: up to KS runs, stored as (start | end<<8 | id<<16)
    __shared__ int run_cnt[17];
    __shared__ float red[2][8];
    const int pix = blockIdx.x;
    const int oy = pix / wo, ox = pix - oy * wo;
    for (int t = threadIdx.x; t < KS * KS; t += blockDim.x) {
        const int ky = t / KS, kx = t - ky * KS;
        const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
        int id = -1;
        if (iy >= 0 && iy < Hm && ix >= 0 && ix < Wm) {
            const float v = __ldg(mask + (size_t)iy * Wm + ix);
            const int iv = (int)v;
            if ((float)iv == v && iv >= 0 && iv < NID) id = iv;
        }
        ids[t] = id;
    }
    __syncthreads();
    if (threadIdx.x < KS) {
        const int ky = threadIdx.x;
        int n = 0, start = 0, cur = ids[ky * KS];
        for (int kx = 1; kx <= KS; ++kx) {
            const int v = (kx < KS) ? ids[ky * KS + kx] : -2;
            if (v != cur) {
                if (cur >= 0) run_pos[ky * 18 + n++] = start | (kx << 8) | (cur << 16);
                start = kx;
                cur = v;
            }
        }
        run_cnt[ky] = n;
    }
    __syncthreads();
    const int c = threadIdx.x;      // C == blockDim.x == 256 (checked on the host)
    float acc = 0.f;
    for (int ky = 0; ky < KS; ++ky) {
        const int n = run_cnt[ky];
        const float* row = wp + (size_t)ky * (KS + 1) * NID * C + c;
        for (int r = 0; r < n; ++r) {
            const int e = run_pos[ky * 18 + r];
            const int a = e & 0xff, b = (e >> 8) & 0xff, id = e >> 16;
            acc += __ldg(row + ((size_t)b * NID + id) * C) - __ldg(row + ((size_t)a * NID + id) * C);
        }
    }
    acc += __ldg(bias + c);
    if constexpr (!LN) out[(size_t)pix * ldo + c] = acc;
    else {
        float s = warp_sum(acc);
        const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
        if (lane == 0) red[0][wid] = s;
        __syncthreads();
        float tot = 0.f;
        for (int w2 = 0; w2 < 8; ++w2) tot += red[0][w2];
        const float mean = tot / (float)C;
        const float d = acc - mean;
        float q = warp_sum(d * d);
        if (lane == 0) red[1][wid] = q;
        __syncthreads();
        float tq = 0.f;
        for (int w2 = 0; w2 < 8; ++w2) tq += red[1][w2];
        const float rstd = rsqrtf(tq / (float)C + 1e-5f);
        out[(size_t)pix * ldo + c] = d * rstd * __ldg(ln_g + c) + __ldg(ln_b + c);
    }
}

template <bool LN>
__global__ void __launch_bounds__(256) id_embed_runs_kernel(const float* __restrict__ mask, int Hm, int Wm,
                                                            const float* __restrict__ wp, const float* __restrict__ bias,
                                                            const float* __restrict__ ln_g, const float* __restrict__ ln_b,
                                                            float* __restrict__ out, int ldo, int ho, int wo, int C,
                                                            int NID, int KS, int stride, int pad) {
    id_embed_runs_cta<LN>(mask, Hm, Wm, wp, bias, ln_g, ln_b, out, ldo, ho, wo, C, NID, KS, stride, pad);
}

// n label maps [n][Hm][Wm] in one launch: map b = blockIdx.y writes output rows [b ho wo, (b + 1) ho wo).
template <bool LN>
__global__ void __launch_bounds__(256) id_embed_runs_batched_kernel(const float* __restrict__ mask, int Hm, int Wm,
                                                                    const float* __restrict__ wp, const float* __restrict__ bias,
                                                                    const float* __restrict__ ln_g, const float* __restrict__ ln_b,
                                                                    float* __restrict__ out, int ldo, int ho, int wo, int C,
                                                                    int NID, int KS, int stride, int pad) {
    const size_t b = blockIdx.y;
    id_embed_runs_cta<LN>(mask + b * Hm * Wm, Hm, Wm, wp, bias, ln_g, ln_b, out + b * ho * wo * ldo, ldo, ho, wo, C, NID, KS,
                          stride, pad);
}

__device__ __forceinline__ void bl_src(int dst, int in_sz, int out_sz, int align, int& i0, int& i1, float& l1) {
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

// logits_nhwc [h][w][NC] -> lowres NCHW [NC][h][w] with ids > obj_num masked to -1e10
__global__ void logits_mask_kernel(const float* __restrict__ in, float* __restrict__ lo, int h, int w, int NC,
                                   int obj_num) {
    pdl_sync();
    const int total = NC * h * w;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int c = i / (h * w), r = i - c * h * w;
        lo[i] = (c > obj_num) ? -1e10f : __ldg(in + (size_t)r * NC + c);
    }
}

// lowres NCHW [NC][h][w] -> out NCHW [NC][Ho][Wo], bilinear
__global__ void logits_upsample_kernel(const float* __restrict__ lo, float* __restrict__ out, int h, int w, int NC,
                                       int Ho, int Wo, int align) {
    pdl_sync();
    const size_t total = (size_t)NC * Ho * Wo;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ox = i % Wo;
        const size_t t = i / Wo;
        const int oy = t % Ho, c = t / Ho;
        int y0, y1, x0, x1;
        float ly, lx;
        bl_src(oy, h, Ho, align, y0, y1, ly);
        bl_src(ox, w, Wo, align, x0, x1, lx);
        const float* b = lo + (size_t)c * h * w;
        const float hy = 1.f - ly, hx = 1.f - lx;
        out[i] = hy * (hx * b[y0 * w + x0] + lx * b[y0 * w + x1]) + ly * (hx * b[y1 * w + x0] + lx * b[y1 * w + x1]);
    }
}

// fused K9 fast path: bilinear upsample of the masked low-res logits + argmax over ids -> label map
// (evaluator.py:339-361 collapses to argmax(logits) for one engine without TTA).  First maximum
// wins on ties, like torch.argmax.
__global__ void logits_argmax_kernel(const float* __restrict__ lo, float* __restrict__ label, int h, int w, int NC,
                                     int Ho, int Wo, int align) {
    pdl_sync();
    const int total = Ho * Wo;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int oy = i / Wo, ox = i - oy * Wo;
        int y0, y1, x0, x1;
        float ly, lx;
        bl_src(oy, h, Ho, align, y0, y1, ly);
        bl_src(ox, w, Wo, align, x0, x1, lx);
        const float hy = 1.f - ly, hx = 1.f - lx;
        float best = -INFINITY;
        int bi = 0;
        for (int c = 0; c < NC; ++c) {
            const float* b = lo + (size_t)c * h * w;
            const float v =
                hy * (hx * b[y0 * w + x0] + lx * b[y0 * w + x1]) + ly * (hx * b[y1 * w + x0] + lx * b[y1 * w + x1]);
            if (v > best) { best = v; bi = c; }
        }
        label[i] = (float)bi;
    }
}

// nearest-neighbour resize of a label map (F.interpolate(mode='nearest'), evaluator.py:418-421):
// src = floor(dst * in / out)
__global__ void nearest_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, int Ho, int Wo) {
    pdl_sync();
    const int total = Ho * Wo;
    const float sy = (float)H / (float)Ho, sx = (float)W / (float)Wo;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int oy = i / Wo, ox = i - oy * Wo;
        int iy = (int)floorf(oy * sy), ix = (int)floorf(ox * sx);
        iy = iy < H - 1 ? iy : H - 1;
        ix = ix < W - 1 ? ix : W - 1;
        out[i] = in[(size_t)iy * W + ix];
    }
}

// Test-time augmentation (networks/managers/evaluator.py:265-446 with TEST_FLIP / TEST_MULTISCALE): E augmentations, each an
// engine on its own resized and possibly mirrored copy of the frame.  Both kernels sample an augmentation's logit map with the
// bilinear arithmetic of logits_argmax_kernel; a map already at the output size is read unchanged (bl_src gives weights 1 and
// 0 there for either align_corners).
struct TTAArgs {
    const float* logits[8];     // [NC][h][w] per augmentation
    int h[8], w[8];
    int flip[8];
};

__device__ __forceinline__ float tta_sample(const float* __restrict__ b, int w, int y0, int y1, int x0, int x1, float ly,
                                            float lx) {
    const float hy = 1.f - ly, hx = 1.f - lx;
    return hy * (hx * b[y0 * w + x0] + lx * b[y0 * w + x1]) + ly * (hx * b[y1 * w + x0] + lx * b[y1 * w + x1]);
}

// Up to TTA_BATCH videos (merge) or lanes (feedback) per launch, one per blockIdx.y; the entry points launch once per chunk.
constexpr int TTA_BATCH = 32;

struct TTAMergeBatchArgs {
    const float* logits[8];     // per augmentation: its scale's decoder output [lanes][h][w][NC]
    int h[8], w[8];
    int flip[8];
    int lane[TTA_BATCH][8];     // video b's lane in augmentation e's map
    int obj[TTA_BATCH];
    const float* new_label[TTA_BATCH];
};

// Tap loaders of the two TTA bodies below.  A loader gives a map's channel c blended at the four bilinear taps with
// tta_sample's arithmetic, so a body never sees the logit layout.
//   NCHW forms (the one-video kernels): masked low-resolution maps [NC][h][w].
//   NHWC forms (the batched kernels): one lane of a multi-video decoder's output [lanes][h][w][NC], with the post-processing
//   mask applied at every tap: a channel above the video's object count reads -1e10, the value aotb_logits_postproc_f32
//   writes, and blended with tta_sample's roundings, so every sampled logit is bit for bit the one-video form's.
__device__ __forceinline__ float tta_sample_nhwc(const float* __restrict__ b, int w, int NC, int c, int obj, int y0, int y1,
                                                 int x0, int x1, float ly, float lx) {
    auto tap = [&](int y, int x) { return c > obj ? -1e10f : __ldg(b + ((y * w + x) * NC + c)); };   // a lane < 2^31
    const float hy = 1.f - ly, hx = 1.f - lx;
    // tta_sample's blend with its contraction spelled out: nvcc compiles tta_sample in the one-video kernels to
    // fma(hx, v0, lx * v1) per row and fma(hy, row0, ly * row1) across rows, and left to itself it contracts this copy the
    // other way round at some sites, one ulp apart.
    const float r0 = __fmaf_rn(hx, tap(y0, x0), __fmul_rn(lx, tap(y0, x1)));
    const float r1 = __fmaf_rn(hx, tap(y1, x0), __fmul_rn(lx, tap(y1, x1)));
    return __fmaf_rn(hy, r0, __fmul_rn(ly, r1));
}

// One map's channels: c -> channel c blended at the taps.
struct TTANchwMap {
    const float* lo;
    size_t plane;
    int w;
    __device__ __forceinline__ float operator()(int c, int y0, int y1, int x0, int x1, float ly, float lx) const {
        return tta_sample(lo + c * plane, w, y0, y1, x0, x1, ly, lx);
    }
};

struct TTANhwcMap {
    const float* b;             // the lane's [h][w][NC]
    int w, NC, obj;
    __device__ __forceinline__ float operator()(int c, int y0, int y1, int x0, int x1, float ly, float lx) const {
        return tta_sample_nhwc(b, w, NC, c, obj, y0, y1, x0, x1, ly, lx);
    }
};

struct TTAMergeNhwc {           // video b's lanes of E augmentations' maps
    const TTAMergeBatchArgs& a;
    int b, NC;
    __device__ __forceinline__ int h(int e) const { return a.h[e]; }
    __device__ __forceinline__ int w(int e) const { return a.w[e]; }
    __device__ __forceinline__ int flip(int e) const { return a.flip[e]; }
    __device__ __forceinline__ TTANhwcMap channels(int e) const {
        return TTANhwcMap{a.logits[e] + (size_t)a.lane[b][e] * a.h[e] * a.w[e] * NC, a.w[e], NC, a.obj[b]};
    }
    __device__ __forceinline__ float operator()(int e, int c, int y0, int y1, int x0, int x1, float ly, float lx) const {
        return channels(e)(c, y0, y1, x0, x1, ly, lx);
    }
};

struct TTAFeedbackNchw {        // one map, or none (lo null)
    const float* lo;
    int h, w;
    __device__ __forceinline__ bool live() const { return lo; }
    __device__ __forceinline__ TTANchwMap channels() const { return TTANchwMap{lo, (size_t)h * w, w}; }
};

struct TTAFeedbackNhwc {        // one lane, or none (lane null)
    TTANhwcMap lane;
    __device__ __forceinline__ bool live() const { return lane.b; }
    __device__ __forceinline__ const TTANhwcMap& channels() const { return lane; }
};

// evaluator.py:332-361: per output pixel, every augmentation's upsampled logits (read at the mirrored column for a flipped
// one, :336-337) -> softmax over NC (:339) -> mean over the augmentations in order (:355-358) -> first argmax (:359-361),
// then the new-object overlay n != 0 ? n : label (:363-369).  The mean probabilities go to prob [NC][H][W] when it is given.
// Three passes over the channels per augmentation (max, sum, probability): the E x NC logits stay in L1 / L2, nothing but the
// label (and the optional probabilities) is written.  This is pixel i of one video.
template <class Maps>
__device__ __forceinline__ void tta_merge_pixel(const Maps& a, int E, int NC, int Ho, int Wo, int align, int i, int total,
                                                float inv_e, const float* __restrict__ new_label, float* __restrict__ label,
                                                float* __restrict__ prob) {
    const int oy = i / Wo, ox = i - oy * Wo;
    int y0[8], y1[8], x0[8], x1[8];
    float ly[8], lx[8], m[8], s[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        if (e < E) {
            bl_src(oy, a.h(e), Ho, align, y0[e], y1[e], ly[e]);
            bl_src(a.flip(e) ? Wo - 1 - ox : ox, a.w(e), Wo, align, x0[e], x1[e], lx[e]);
            const auto ch = a.channels(e);
            float mx = -INFINITY;
            for (int c = 0; c < NC; ++c) mx = fmaxf(mx, ch(c, y0[e], y1[e], x0[e], x1[e], ly[e], lx[e]));
            float sum = 0.f;
            for (int c = 0; c < NC; ++c) sum += expf(ch(c, y0[e], y1[e], x0[e], x1[e], ly[e], lx[e]) - mx);
            m[e] = mx;
            s[e] = sum;
        }
    }
    float best = -INFINITY;
    int bi = 0;
    for (int c = 0; c < NC; ++c) {
        float acc = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            if (e < E) acc += expf(a(e, c, y0[e], y1[e], x0[e], x1[e], ly[e], lx[e]) - m[e]) / s[e];
        }
        const float p = acc * inv_e;
        if (prob) prob[(size_t)c * total + i] = p;
        if (p > best) { best = p; bi = c; }
    }
    const float n = new_label ? new_label[i] : 0.f;
    label[i] = n != 0.f ? n : (float)bi;
}

__global__ void tta_merge_kernel(const TTAArgs a, int E, int NC, int Ho, int Wo, int align,
                                 const float* __restrict__ new_label, float* __restrict__ label, float* __restrict__ prob) {
    pdl_sync();
    const int total = Ho * Wo;
    const float inv_e = 1.f / (float)E;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int oy = i / Wo, ox = i - oy * Wo;
        int y0[8], y1[8], x0[8], x1[8];
        float ly[8], lx[8], m[8], s[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            if (e < E) {
                bl_src(oy, a.h[e], Ho, align, y0[e], y1[e], ly[e]);
                bl_src(a.flip[e] ? Wo - 1 - ox : ox, a.w[e], Wo, align, x0[e], x1[e], lx[e]);
                const size_t plane = (size_t)a.h[e] * a.w[e];
                float mx = -INFINITY;
                for (int c = 0; c < NC; ++c)
                    mx = fmaxf(mx, tta_sample(a.logits[e] + c * plane, a.w[e], y0[e], y1[e], x0[e], x1[e], ly[e], lx[e]));
                float sum = 0.f;
                for (int c = 0; c < NC; ++c)
                    sum += expf(tta_sample(a.logits[e] + c * plane, a.w[e], y0[e], y1[e], x0[e], x1[e], ly[e], lx[e]) - mx);
                m[e] = mx;
                s[e] = sum;
            }
        }
        float best = -INFINITY;
        int bi = 0;
        for (int c = 0; c < NC; ++c) {
            float acc = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                if (e < E) {
                    const float* b = a.logits[e] + c * (size_t)a.h[e] * a.w[e];
                    acc += expf(tta_sample(b, a.w[e], y0[e], y1[e], x0[e], x1[e], ly[e], lx[e]) - m[e]) / s[e];
                }
            }
            const float p = acc * inv_e;
            if (prob) prob[(size_t)c * total + i] = p;
            if (p > best) { best = p; bi = c; }
        }
        const float n = new_label ? new_label[i] : 0.f;
        label[i] = n != 0.f ? n : (float)bi;
    }
}

// tta_merge_kernel over n videos: video b = blockIdx.y reads its own lane of every augmentation's map, masked at its own
// object count, and writes label [b][H][W] (and prob [b][NC][H][W]).
__global__ void tta_merge_batched_kernel(const TTAMergeBatchArgs a, int E, int NC, int Ho, int Wo, int align,
                                         float* __restrict__ label, float* __restrict__ prob) {
    pdl_sync();
    const int b = blockIdx.y;
    const int total = Ho * Wo;
    const float inv_e = 1.f / (float)E;
    float* lb = label + (size_t)b * total;
    float* pb = prob ? prob + (size_t)b * NC * total : nullptr;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x)
        tta_merge_pixel(TTAMergeNhwc{a, b, NC}, E, NC, Ho, Wo, align, i, total, inv_e, a.new_label[b], lb, pb);
}

// evaluator.py:346-353, :363-422 for one augmentation: the label its engine stores in memory.  For input pixel (y, x) the
// nearest source (sy, sx) at the output size follows nearest_kernel; base = argmax softmax of the upsampled logits at (sy, sx)
// in the augmentation's own orientation (the flip of :336-337 and the flip back of :373-376 / :402-406 cancel), n = the
// new-object label at the mirrored column for a flipped augmentation (mirror at output size first, then nearest: the two do not
// commute), out = n != 0 ? n : base.  No logits: base = 0 (the first frame's label, :315-319); no new label: n = 0.  This is
// input pixel i of one augmentation.
template <class Map>
__device__ __forceinline__ void tta_feedback_pixel(const Map& lo, int h, int w, int NC, int H, int W, int align, int flip,
                                                   const float* __restrict__ new_label, float* __restrict__ out, int i,
                                                   int Wi, float sy, float sx) {
    const int oy = i / Wi, ox = i - oy * Wi;
    int iy = (int)floorf(oy * sy), ix = (int)floorf(ox * sx);
    iy = iy < H - 1 ? iy : H - 1;
    ix = ix < W - 1 ? ix : W - 1;
    int base = 0;
    if (lo.live()) {
        int y0, y1, x0, x1;
        float ly, lx;
        bl_src(iy, h, H, align, y0, y1, ly);
        bl_src(ix, w, W, align, x0, x1, lx);
        const auto ch = lo.channels();
        float mx = -INFINITY;
        for (int c = 0; c < NC; ++c) mx = fmaxf(mx, ch(c, y0, y1, x0, x1, ly, lx));
        float sum = 0.f;
        for (int c = 0; c < NC; ++c) sum += expf(ch(c, y0, y1, x0, x1, ly, lx) - mx);
        float best = -INFINITY;
        for (int c = 0; c < NC; ++c) {
            const float p = expf(ch(c, y0, y1, x0, x1, ly, lx) - mx) / sum;
            if (p > best) { best = p; base = c; }
        }
    }
    const float n = new_label ? new_label[(size_t)iy * W + (flip ? W - 1 - ix : ix)] : 0.f;
    out[i] = n != 0.f ? n : (float)base;
}

__global__ void tta_feedback_kernel(const float* __restrict__ lo, int h, int w, int NC, int H, int W, int align, int flip,
                                    const float* __restrict__ new_label, float* __restrict__ out, int Hi, int Wi) {
    pdl_sync();
    const int total = Hi * Wi;
    const float sy = (float)H / (float)Hi, sx = (float)W / (float)Wi;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x)
        tta_feedback_pixel(TTAFeedbackNchw{lo, h, w}, h, w, NC, H, W, align, flip, new_label, out, i, Wi, sy, sx);
}

struct TTAFeedbackBatchArgs {
    int obj[TTA_BATCH];
    int flip[TTA_BATCH];
    const float* new_label[TTA_BATCH];
};

// tta_feedback_kernel over n lanes of one multi-video pool: lane k = blockIdx.y reads its rows of the decoder output
// [lanes][h][w][NC] (masked at its object count; lg null: the no-logits form) and writes its memory label into out [k][Hi][Wi].
__global__ void tta_feedback_batched_kernel(const float* __restrict__ lg, int h, int w, int NC, int H, int W, int align,
                                            const TTAFeedbackBatchArgs a, float* __restrict__ out, int Hi, int Wi) {
    pdl_sync();
    const int k = blockIdx.y;
    const int total = Hi * Wi;
    const float sy = (float)H / (float)Hi, sx = (float)W / (float)Wi;
    const TTAFeedbackNhwc lane{{lg ? lg + (size_t)k * h * w * NC : nullptr, w, NC, a.obj[k]}};
    float* ok = out + (size_t)k * total;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x)
        tta_feedback_pixel(lane, h, w, NC, H, W, align, a.flip[k], a.new_label[k], ok, i, Wi, sy, sx);
}


// soft_logit_aggregation (aot_engine.py:565-582) for E sub-engines of max_obj objects each, fused: per output pixel
//   prob_e = softmax over the 1 + max_obj channels of engine e;  bg = prod_e prob_e[0];
//   merged = clamp([bg, prob_0[1:], prob_1[1:], ...], 1e-5, 1 - 1e-5);  out = log(merged / (1 - merged))   (torch.logit)
// One thread per pixel: the E x (1 + max_obj) logits of a pixel are read once (channel planes are HW apart, so a warp reads
// 128 contiguous bytes per channel) and the 1 + E * max_obj merged logits written once.  The reference materialises E softmax
// tensors, two concatenations, a product, a clamp and a logit (7 passes over E x 18 MB at 480p).
struct AggArgs { const float* logits[8]; };

// One output pixel of soft_logit_aggregation for the batched kernel: ld(e, c) is engine e's logit of channel c at the pixel;
// emit.engine(e).fg(c, v) receives the merged logit of engine e's object c (c >= 1), emit.bg(v) the merged background.  It
// performs soft_logit_aggregation_kernel's operations in the same order, so every merged logit is bit for bit the one-video
// kernel's; that kernel keeps its own copy of them because inlining this body there changes its compiled code.
template <int NC, class Load, class Emit>
__device__ __forceinline__ void soft_logit_aggregation_pixel(const Load& ld, int E, Emit& emit) {
    float bg = 1.f;
    for (int e = 0; e < E; ++e) {
        float v[NC];
        float m = -INFINITY;
#pragma unroll
        for (int c = 0; c < NC; ++c) { v[c] = ld(e, c); m = fmaxf(m, v[c]); }
        float sum = 0.f;
#pragma unroll
        for (int c = 0; c < NC; ++c) { v[c] = expf(v[c] - m); sum += v[c]; }
        bg *= v[0] / sum;
        auto o = emit.engine(e);
#pragma unroll
        for (int c = 1; c < NC; ++c) {
            const float p = fminf(fmaxf(v[c] / sum, 1e-5f), 1.f - 1e-5f);
            o.fg(c, logf(p / (1.f - p)));
        }
    }
    const float p = fminf(fmaxf(bg, 1e-5f), 1.f - 1e-5f);
    emit.bg(logf(p / (1.f - p)));
}

template <int NC>
__global__ void soft_logit_aggregation_kernel(const AggArgs a, int E, float* __restrict__ out, int HW) {
    pdl_sync();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        float bg = 1.f;
        for (int e = 0; e < E; ++e) {
            const float* l = a.logits[e] + i;
            float v[NC];
            float m = -INFINITY;
#pragma unroll
            for (int c = 0; c < NC; ++c) { v[c] = l[(size_t)c * HW]; m = fmaxf(m, v[c]); }
            float sum = 0.f;
#pragma unroll
            for (int c = 0; c < NC; ++c) { v[c] = expf(v[c] - m); sum += v[c]; }
            bg *= v[0] / sum;
            float* o = out + (size_t)(1 + e * (NC - 1)) * HW + i;
#pragma unroll
            for (int c = 1; c < NC; ++c) {
                const float p = fminf(fmaxf(v[c] / sum, 1e-5f), 1.f - 1e-5f);
                o[(size_t)(c - 1) * HW] = logf(p / (1.f - p));
            }
        }
        const float p = fminf(fmaxf(bg, 1e-5f), 1.f - 1e-5f);
        out[i] = logf(p / (1.f - p));
    }
}

// logits_upsample_kernel's value at one output pixel, read from one lane [h][w][NC] of a decoder output with
// logits_mask_kernel's mask applied at every tap (a channel above obj reads -1e10).  The blend spells out the contraction nvcc
// gives logits_upsample_kernel, fma(lx, v1, hx * v0) per row and fma(hy, row0, ly * row1) across rows, so every value is bit
// for bit aotb_logits_postproc_f32's.
__device__ __forceinline__ float upsample_nhwc(const float* __restrict__ b, int w, int NC, int c, int obj, int y0, int y1,
                                               int x0, int x1, float ly, float lx) {
    auto tap = [&](int y, int x) { return c > obj ? -1e10f : __ldg(b + ((y * w + x) * NC + c)); };   // a lane < 2^31
    const float hy = 1.f - ly, hx = 1.f - lx;
    const float r0 = __fmaf_rn(lx, tap(y0, x1), __fmul_rn(hx, tap(y0, x0)));
    const float r1 = __fmaf_rn(lx, tap(y1, x1), __fmul_rn(hx, tap(y1, x0)));
    return __fmaf_rn(hy, r0, __fmul_rn(ly, r1));
}

// soft_logit_aggregation over several videos of a multi-video pool, reading the decoder output [lanes][h][w][NC] directly:
// video b = blockIdx.y aggregates its k[b] lanes in sub-engine order, each masked at its own object count and sampled at
// [Ho][Wo] as aotb_logits_postproc_f32 does (upsample_nhwc; read unchanged when the size is [h][w]).  Writes the merged map out[b] [1 + k (NC - 1)][Ho][Wo] and / or label[b] [Ho][Wo], the map's first argmax; the
// label compares the very values the map receives.
constexpr int AGG_BATCH = 32;

struct AggBatchArgs {
    int lane[AGG_BATCH][8];
    int obj[AGG_BATCH][8];
    int k[AGG_BATCH];
    float* out[AGG_BATCH];
    float* label[AGG_BATCH];
};

template <int NC>
struct AggBatchOut {
    float* out;                 // null: label only
    size_t total;
    int i;
    float best;
    int bi;
    struct Engine {
        AggBatchOut& s;
        int ch0;
        __device__ __forceinline__ void fg(int c, float v) {
            const int ch = ch0 + c - 1;
            if (s.out) s.out[ch * s.total + s.i] = v;
            if (v > s.best) { s.best = v; s.bi = ch; }
        }
    };
    __device__ __forceinline__ Engine engine(int e) { return Engine{*this, 1 + e * (NC - 1)}; }
    __device__ __forceinline__ void bg(float v) {
        if (out) out[i] = v;
        if (!(best > v)) bi = 0;          // channel 0 comes first: it wins a tie
    }
};

template <int NC>
__global__ void soft_logit_aggregation_batched_kernel(const float* __restrict__ lg, int h, int w, int Ho, int Wo, int align,
                                                      const AggBatchArgs a) {
    pdl_sync();
    const int b = blockIdx.y;
    const int E = a.k[b];
    const int total = Ho * Wo;
    const bool same = Ho == h && Wo == w;
    const size_t lane = (size_t)h * w * NC;
    float* label = a.label[b];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int oy = i / Wo, ox = i - oy * Wo;
        int y0, y1, x0, x1;
        float ly, lx;
        bl_src(oy, h, Ho, align, y0, y1, ly);
        bl_src(ox, w, Wo, align, x0, x1, lx);
        auto ld = [&](int e, int c) {
            const float* base = lg + (size_t)a.lane[b][e] * lane;
            const int obj = a.obj[b][e];
            if (same) return c > obj ? -1e10f : __ldg(base + ((size_t)(oy * w + ox) * NC + c));
            return upsample_nhwc(base, w, NC, c, obj, y0, y1, x0, x1, ly, lx);
        };
        AggBatchOut<NC> emit{a.out[b], (size_t)total, i, -INFINITY, 0};
        soft_logit_aggregation_pixel<NC>(ld, E, emit);
        if (label) label[i] = (float)emit.bi;
    }
}

// separate_mask for label maps (aot_engine.py:515-533): engine e keeps ids [e*max_obj + 1, (e+1)*max_obj], renumbered from 1,
// everything else becomes background.  One pass writes all E maps (the reference builds E boolean masks and 3 E temporaries).
__global__ void separate_labels_kernel(const float* __restrict__ mask, int E, int max_obj, float* __restrict__ out, int HW) {
    pdl_sync();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        const float m = mask[i];
        for (int e = 0; e < E; ++e) {
            const float lo = (float)(e * max_obj + 1), hi = (float)((e + 1) * max_obj);
            out[(size_t)e * HW + i] = (m >= lo && m <= hi) ? m - lo + 1.f : 0.f;
        }
    }
}

// separate_labels_kernel for the lanes of several videos: entry b = blockIdx.y writes out[b] = part[b]'s map of label[b].  The
// per-element arithmetic is separate_labels_kernel's, which keeps its own copy so that its compiled code is unchanged.
__device__ __forceinline__ float separate_label(float m, int e, int max_obj) {
    const float lo = (float)(e * max_obj + 1), hi = (float)((e + 1) * max_obj);
    return (m >= lo && m <= hi) ? m - lo + 1.f : 0.f;
}

constexpr int SEP_BATCH = 32;

struct SepBatchArgs {
    const float* label[SEP_BATCH];
    float* out[SEP_BATCH];
    int part[SEP_BATCH];
};

__global__ void separate_labels_batched_kernel(const SepBatchArgs a, int max_obj, int HW) {
    pdl_sync();
    const int b = blockIdx.y;
    const float* __restrict__ mask = a.label[b];
    float* __restrict__ out = a.out[b];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x)
        out[i] = separate_label(mask[i], a.part[b], max_obj);
}

// Gather of up to four per-video maps into lane order: for every map j, lane l = blockIdx.y copies video lane_video[l]'s
// n4[j] float4s from src[j] into its own rows of dst[j].  A table entry outside [0, n_videos) copies nothing.
struct LaneGatherArgs {
    const float* src[4];
    float* dst[4];
    int n4[4];
};

__global__ void __launch_bounds__(256) lane_gather_kernel(const LaneGatherArgs a, int n_maps, const int* __restrict__ lane_video,
                                                          int n_videos) {
    pdl_sync();
    const int l = blockIdx.y;
    const int v = lane_video[l];
    if (v < 0 || v >= n_videos) return;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j < n_maps) {
            const size_t n4 = a.n4[j];
            const float4* __restrict__ s = reinterpret_cast<const float4*>(a.src[j]) + (size_t)v * n4;
            float4* __restrict__ d = reinterpret_cast<float4*>(a.dst[j]) + (size_t)l * n4;
            for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
                d[i] = __ldg(s + i);
        }
    }
}

// rows x cols copy into bank at row offset (host value or device counter)
__global__ void bank_append_kernel(const float* __restrict__ src, int lds, float* __restrict__ bank, int ldb,
                                   int rows, int cols4, int offset, const int* __restrict__ offset_dev) {
    pdl_sync();
    const int off = offset_dev ? *offset_dev : offset;
    const size_t total = (size_t)rows * cols4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = i / cols4, c = (i - (size_t)r * cols4) * 4;
        *reinterpret_cast<float4*>(bank + (size_t)(off + r) * ldb + c) =
            *reinterpret_cast<const float4*>(src + (size_t)r * lds + c);
    }
}

__global__ void counter_add_kernel(int* ctr, int delta) {
    pdl_sync(); *ctr += delta; }

// Bounded bank (a pinned first frame + a FIFO ring of the newest frames): one launch stores a memory frame's K and V rows into
// every copy of the bank the attention kernels read, at the ring's device-resident write offset.
struct RingStoreArgs {
    const float* src[2];    // K, V rows [rows][ld]
    float* bank[2];         // fp32 banks [cap_rows][ldb] (nullptr: no such copy)
    __half* packed[2];      // split-fp16 banks [cols / 32][cap_rows][64] (nullptr: no such copy)
    int ld[2], ldb[2], c4[2];   // c4: float4 groups per row
};

// One thread per (row, 4 channels) of K then V: the source is read once; the packed rows are the bytes of pack_rows64_kernel
// with div == 1 (hi = fp16(x), lo = fp16(x - hi), [hi(32) | lo(32)] per 32-channel chunk).  Bank
// rows from `off`; the packed banks' 32-channel chunks are head_rows rows apart.
__device__ __forceinline__ void ring_store_rows(const RingStoreArgs& a, int rows, int head_rows, int off) {
    const int per_row = a.c4[0] + a.c4[1];
    const size_t total = (size_t)rows * per_row;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = i / per_row;
        int j = i - (size_t)r * per_row;
        const bool isv = j >= a.c4[0];                    // selects, not indexing: the arguments stay in constant memory
        if (isv) j -= a.c4[0];
        const float* src = isv ? a.src[1] : a.src[0];
        float* bank = isv ? a.bank[1] : a.bank[0];
        __half* packed = isv ? a.packed[1] : a.packed[0];
        const int ld = isv ? a.ld[1] : a.ld[0], ldb = isv ? a.ldb[1] : a.ldb[0];
        const float4 v = __ldg(reinterpret_cast<const float4*>(src + (size_t)r * ld + j * 4));
        if (bank) *reinterpret_cast<float4*>(bank + (size_t)(off + r) * ldb + j * 4) = v;
        if (packed) {
            const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
            const __half2 l0 = __floats2half2_rn(v.x - __low2float(h0), v.y - __high2float(h0));
            const __half2 l1 = __floats2half2_rn(v.z - __low2float(h1), v.w - __high2float(h1));
            __half* d = packed + ((size_t)(j >> 3) * head_rows + off + r) * 64 + (j & 7) * 4;
            uint2 hi, lo;
            hi.x = *reinterpret_cast<const unsigned*>(&h0); hi.y = *reinterpret_cast<const unsigned*>(&h1);
            lo.x = *reinterpret_cast<const unsigned*>(&l0); lo.y = *reinterpret_cast<const unsigned*>(&l1);
            *reinterpret_cast<uint2*>(d) = hi;
            *reinterpret_cast<uint2*>(d + 32) = lo;
        }
    }
}

__global__ void __launch_bounds__(256) bank_ring_store_kernel(const RingStoreArgs a, int rows, int cap_rows,
                                                              const int* __restrict__ write) {
    pdl_sync();
    const int off = *write;
    if (off < 0 || off + rows > cap_rows) return;      // never write outside the bank, whatever the counter holds
    ring_store_rows(a, rows, cap_rows, off);
}

// n banks of cap_rows rows each, stacked (bank b = rows [b cap_rows, (b + 1) cap_rows) of every copy; the packed copies'
// chunks are head_rows = n_banks cap_rows apart): bank b = blockIdx.y stores source rows [b rows, (b + 1) rows) at its own
// write offset write[b] when store[b] != 0.
__global__ void __launch_bounds__(256) bank_ring_store_batched_kernel(const RingStoreArgs a, int rows, int cap_rows,
                                                                      int head_rows, const int* __restrict__ write,
                                                                      const int* __restrict__ store) {
    pdl_sync();
    const int b = blockIdx.y;
    if (!store[b]) return;
    const int off = write[b];
    if (off < 0 || off + rows > cap_rows) return;
    RingStoreArgs ab = a;
    for (int i = 0; i < 2; ++i) {
        ab.src[i] += (size_t)b * rows * a.ld[i];
        if (ab.bank[i]) ab.bank[i] += (size_t)b * cap_rows * a.ldb[i];
        if (ab.packed[i]) ab.packed[i] += (size_t)b * cap_rows * 64;
    }
    ring_store_rows(ab, rows, head_rows, off);
}

// After a store of `rows` rows: one more frame is live until the bank is full; the write offset moves on by one frame and
// wraps to the first unpinned row when the next frame would not fit.
__global__ void ring_advance_kernel(int* live, int* write, int rows, int cap_rows, int pinned_rows) {
    pdl_sync();
    *live = min(*live + rows, cap_rows);
    int w = *write + rows;
    if (w + rows > cap_rows) w = pinned_rows;
    *write = w;
}

// ring_advance_kernel for n banks, bank b only when store[b] != 0.
__global__ void ring_advance_batched_kernel(int* live, int* write, const int* store, int n, int rows, int cap_rows,
                                            int pinned_rows) {
    pdl_sync();
    const int b = threadIdx.x;
    if (b >= n || !store[b]) return;
    live[b] = min(live[b] + rows, cap_rows);
    int w = write[b] + rows;
    if (w + rows > cap_rows) w = pinned_rows;
    write[b] = w;
}

// Usage policy of the bounded bank, before a store: the next free slot while the bank is not full, else the unpinned slot
// with the lowest mean attention mass U / A (A == 0 counts as +inf, ties go to the lowest slot); that slot's counters restart.
__global__ void ring_select_usage_kernel(const int* live, int* write, float* U, int* A, int rows, int cap_rows,
                                         int pinned_rows) {
    pdl_sync();
    const int slots = cap_rows / rows, used = max(*live, 0) / rows;
    int s = used;
    if (used >= slots) {
        float best = 0.f;
        s = -1;
        for (int c = pinned_rows / rows; c < slots; ++c) {
            const float score = A[c] > 0 ? U[c] / (float)A[c] : INFINITY;
            if (s < 0 || score < best) { s = c; best = score; }
        }
    }
    *write = s * rows;
    U[s] = 0.f;
    A[s] = 0;
}

}  // namespace aotb

using namespace aotb;

extern "C" int aotb_id_embed_f32(const float* mask, int Hm, int Wm, const float* wt, const float* bias,
                                 const float* ln_gamma, const float* ln_beta, float* out, int ldo, int C, int nid,
                                 int ksize, int stride, int pad, void* stream) {
    AOTB_REQUIRE(mask && wt && bias && out && Hm > 0 && Wm > 0, "aotb_id_embed_f32: bad args");
    AOTB_REQUIRE(ksize <= 17 && ksize > 0 && stride > 0, "aotb_id_embed_f32: kernel size > 17");
    const int ho = (Hm + 2 * pad - ksize) / stride + 1, wo = (Wm + 2 * pad - ksize) / stride + 1;
    AOTB_REQUIRE(ho > 0 && wo > 0, "aotb_id_embed_f32: empty output");
    cudaStream_t st = (cudaStream_t)stream;
    if (ln_gamma) {
        AOTB_REQUIRE(C == 256 && ln_beta, "aotb_id_embed_f32: fused LayerNorm needs C == 256");
        launch(id_embed_kernel<true>, dim3(ho * wo), dim3(256), 0, st, mask, Hm, Wm, wt, bias, ln_gamma, ln_beta, out, ldo, ho, wo, C,
                                                       nid, ksize, stride, pad);
    } else {
        launch(id_embed_kernel<false>, dim3(ho * wo), dim3(256), 0, st, mask, Hm, Wm, wt, bias, nullptr, nullptr, out, ldo, ho, wo, C,
                                                        nid, ksize, stride, pad);
    }
    return check_launch("aotb_id_embed_f32");
}

// wp: exclusive prefix sums of the ID-bank weights along kx: [KS][KS+1][nid][C] (C must be 256).
extern "C" int aotb_id_embed_runs_f32(const float* mask, int Hm, int Wm, const float* wp, const float* bias,
                                      const float* ln_gamma, const float* ln_beta, float* out, int ldo, int C, int nid,
                                      int ksize, int stride, int pad, void* stream) {
    AOTB_REQUIRE(mask && wp && bias && out && Hm > 0 && Wm > 0, "aotb_id_embed_runs_f32: bad args");
    AOTB_REQUIRE(ksize <= 17 && ksize > 0 && stride > 0 && C == 256 && nid < 128, "aotb_id_embed_runs_f32: unsupported shape");
    const int ho = (Hm + 2 * pad - ksize) / stride + 1, wo = (Wm + 2 * pad - ksize) / stride + 1;
    AOTB_REQUIRE(ho > 0 && wo > 0, "aotb_id_embed_runs_f32: empty output");
    cudaStream_t st = (cudaStream_t)stream;
    if (ln_gamma) {
        AOTB_REQUIRE(ln_beta, "aotb_id_embed_runs_f32: ln_beta");
        launch(id_embed_runs_kernel<true>, dim3(ho * wo), dim3(256), 0, st, mask, Hm, Wm, wp, bias, ln_gamma, ln_beta, out, ldo, ho, wo,
                                                            C, nid, ksize, stride, pad);
    } else {
        launch(id_embed_runs_kernel<false>, dim3(ho * wo), dim3(256), 0, st, mask, Hm, Wm, wp, bias, nullptr, nullptr, out, ldo, ho, wo,
                                                             C, nid, ksize, stride, pad);
    }
    return check_launch("aotb_id_embed_runs_f32");
}

extern "C" int aotb_logits_postproc_f32(const float* logits_nhwc, float* lowres_nchw, float* out_nchw, int h, int w,
                                        int NC, int obj_num, int Ho, int Wo, int align_corners, void* stream) {
    AOTB_REQUIRE(logits_nhwc && lowres_nchw && h > 0 && w > 0 && NC > 0, "aotb_logits_postproc_f32: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    launch(logits_mask_kernel, dim3(cdiv(NC * h * w, 256)), dim3(256), 0, st, logits_nhwc, lowres_nchw, h, w, NC, obj_num);
    if (out_nchw) {
        AOTB_REQUIRE(Ho > 0 && Wo > 0, "aotb_logits_postproc_f32: bad output size");
        const size_t total = (size_t)NC * Ho * Wo;
        int g = (int)((total + 255) / 256);
        if (g > 132 * 16) g = 132 * 16;
        launch(logits_upsample_kernel, dim3(g), dim3(256), 0, st, lowres_nchw, out_nchw, h, w, NC, Ho, Wo, align_corners);
    }
    return check_launch("aotb_logits_postproc_f32", out_nchw ? 2 : 1);
}

extern "C" int aotb_logits_argmax_f32(const float* lowres_nchw, float* label, int h, int w, int NC, int Ho, int Wo,
                                      int align_corners, void* stream) {
    AOTB_REQUIRE(lowres_nchw && label && h > 0 && w > 0 && NC > 0 && Ho > 0 && Wo > 0,
                 "aotb_logits_argmax_f32: bad args");
    launch(logits_argmax_kernel, dim3(cdiv(Ho * Wo, 256)), dim3(256), 0, (cudaStream_t)stream, lowres_nchw, label, h, w, NC, Ho, Wo,
                                                                               align_corners);
    return check_launch("aotb_logits_argmax_f32");
}

extern "C" int aotb_nearest_resize_f32(const float* in, float* out, int H, int W, int Ho, int Wo, void* stream) {
    AOTB_REQUIRE(in && out && H > 0 && W > 0 && Ho > 0 && Wo > 0, "aotb_nearest_resize_f32: bad args");
    launch(nearest_kernel, dim3(cdiv(Ho * Wo, 256)), dim3(256), 0, (cudaStream_t)stream, in, out, H, W, Ho, Wo);
    return check_launch("aotb_nearest_resize_f32");
}

extern "C" int aotb_tta_merge_f32(const float* const* logits, const int* sizes, const int* flips, int n_augs, int NC, int H,
                                  int W, int align_corners, const float* new_label, float* label, float* pred_prob,
                                  void* stream) {
    AOTB_REQUIRE(logits && sizes && flips && label && NC > 0 && H > 0 && W > 0, "aotb_tta_merge_f32: bad args");
    AOTB_REQUIRE(n_augs >= 1 && n_augs <= 8, "aotb_tta_merge_f32: 1 to 8 augmentations (got %d)", n_augs);
    TTAArgs a;
    for (int e = 0; e < 8; ++e) {
        const bool live = e < n_augs;
        a.logits[e] = live ? logits[e] : nullptr;
        a.h[e] = live ? sizes[2 * e] : 1;
        a.w[e] = live ? sizes[2 * e + 1] : 1;
        a.flip[e] = live ? (flips[e] != 0) : 0;
        AOTB_REQUIRE(!live || (a.logits[e] && a.h[e] > 0 && a.w[e] > 0), "aotb_tta_merge_f32: augmentation %d: bad map", e);
    }
    launch(tta_merge_kernel, dim3(cdiv(H * W, 256)), dim3(256), 0, (cudaStream_t)stream, a, n_augs, NC, H, W, align_corners,
           new_label, label, pred_prob);
    return check_launch("aotb_tta_merge_f32");
}

extern "C" int aotb_tta_feedback_f32(const float* logits, int h, int w, int NC, int H, int W, int align_corners, int flip,
                                     const float* new_label, float* out, int Hi, int Wi, void* stream) {
    AOTB_REQUIRE(out && H > 0 && W > 0 && Hi > 0 && Wi > 0, "aotb_tta_feedback_f32: bad args");
    AOTB_REQUIRE(!logits || (h > 0 && w > 0 && NC > 0), "aotb_tta_feedback_f32: bad logit map");
    launch(tta_feedback_kernel, dim3(cdiv(Hi * Wi, 256)), dim3(256), 0, (cudaStream_t)stream, logits, h, w, NC, H, W,
           align_corners, flip ? 1 : 0, new_label, out, Hi, Wi);
    return check_launch("aotb_tta_feedback_f32");
}

extern "C" int aotb_tta_merge_batched_f32(const float* const* logits, const int* sizes, const int* flips, int n_augs,
                                          const int* lanes, const int* obj_nums, int n, int NC, int H, int W,
                                          int align_corners, const float* const* new_labels, float* label, float* pred_prob,
                                          void* stream) {
    AOTB_REQUIRE(logits && sizes && flips && lanes && obj_nums && label && n > 0 && NC > 0 && H > 0 && W > 0,
                 "aotb_tta_merge_batched_f32: bad args");
    AOTB_REQUIRE(n_augs >= 1 && n_augs <= 8, "aotb_tta_merge_batched_f32: 1 to 8 augmentations (got %d)", n_augs);
    TTAMergeBatchArgs a;
    for (int e = 0; e < 8; ++e) {
        const bool live = e < n_augs;
        a.logits[e] = live ? logits[e] : nullptr;
        a.h[e] = live ? sizes[2 * e] : 1;
        a.w[e] = live ? sizes[2 * e + 1] : 1;
        a.flip[e] = live ? (flips[e] != 0) : 0;
        AOTB_REQUIRE(!live || (a.logits[e] && a.h[e] > 0 && a.w[e] > 0), "aotb_tta_merge_batched_f32: augmentation %d: bad map",
                     e);
        AOTB_REQUIRE(!live || (size_t)a.h[e] * a.w[e] * NC < (1u << 31), "aotb_tta_merge_batched_f32: augmentation %d: lane "
                     "too large", e);
    }
    const size_t plane = (size_t)H * W;
    int launches = 0;
    for (int v0 = 0; v0 < n; v0 += TTA_BATCH, ++launches) {
        const int nb = n - v0 < TTA_BATCH ? n - v0 : TTA_BATCH;
        for (int b = 0; b < nb; ++b) {
            for (int e = 0; e < 8; ++e) {
                a.lane[b][e] = e < n_augs ? lanes[(size_t)(v0 + b) * n_augs + e] : 0;
                AOTB_REQUIRE(a.lane[b][e] >= 0, "aotb_tta_merge_batched_f32: video %d: negative lane", v0 + b);
            }
            a.obj[b] = obj_nums[v0 + b];
            a.new_label[b] = new_labels ? new_labels[v0 + b] : nullptr;
        }
        launch(tta_merge_batched_kernel, dim3(cdiv(H * W, 256), nb), dim3(256), 0, (cudaStream_t)stream, a, n_augs, NC, H, W,
               align_corners, label + v0 * plane, pred_prob ? pred_prob + v0 * NC * plane : nullptr);
    }
    return check_launch("aotb_tta_merge_batched_f32", launches);
}

extern "C" int aotb_tta_feedback_batched_f32(const float* logits, int h, int w, int NC, int n_lanes, const int* obj_nums,
                                             const int* flips, const float* const* new_labels, int H, int W,
                                             int align_corners, float* out, int Hi, int Wi, void* stream) {
    AOTB_REQUIRE(out && flips && n_lanes > 0 && H > 0 && W > 0 && Hi > 0 && Wi > 0, "aotb_tta_feedback_batched_f32: bad args");
    AOTB_REQUIRE(!logits || (obj_nums && h > 0 && w > 0 && NC > 0 && (size_t)h * w * NC < (1u << 31)),
                 "aotb_tta_feedback_batched_f32: bad logit map");
    const size_t lane = (size_t)h * w * NC, plane = (size_t)Hi * Wi;
    TTAFeedbackBatchArgs a;
    int launches = 0;
    for (int k0 = 0; k0 < n_lanes; k0 += TTA_BATCH, ++launches) {
        const int nb = n_lanes - k0 < TTA_BATCH ? n_lanes - k0 : TTA_BATCH;
        for (int k = 0; k < nb; ++k) {
            a.obj[k] = obj_nums ? obj_nums[k0 + k] : 0;
            a.flip[k] = flips[k0 + k] != 0;
            a.new_label[k] = new_labels ? new_labels[k0 + k] : nullptr;
        }
        launch(tta_feedback_batched_kernel, dim3(cdiv(Hi * Wi, 256), nb), dim3(256), 0, (cudaStream_t)stream,
               logits ? logits + k0 * lane : nullptr, h, w, NC, H, W, align_corners, a, out + k0 * plane, Hi, Wi);
    }
    return check_launch("aotb_tta_feedback_batched_f32", launches);
}


// logits: E device pointers to NCHW fp32 maps [1 + max_obj][HW] (the sub-engines' upsampled logits); out [1 + E*max_obj][HW].
extern "C" int aotb_soft_logit_aggregation_f32(const float* const* logits, int n_engines, int max_obj, float* out, int HW,
                                               void* stream) {
    AOTB_REQUIRE(logits && out && n_engines >= 1 && n_engines <= 8 && HW > 0, "aotb_soft_logit_aggregation_f32: bad args");
    AOTB_REQUIRE(max_obj == 10, "aotb_soft_logit_aggregation_f32: built for MODEL_MAX_OBJ_NUM = 10 (got %d)", max_obj);
    AggArgs a;
    for (int e = 0; e < 8; ++e) a.logits[e] = e < n_engines ? logits[e] : nullptr;
    for (int e = 0; e < n_engines; ++e) AOTB_REQUIRE(a.logits[e], "aotb_soft_logit_aggregation_f32: null logit map");
    int g = cdiv(HW, 256);
    if (g > 132 * 8) g = 132 * 8;
    launch(soft_logit_aggregation_kernel<11>, dim3(g), dim3(256), 0, (cudaStream_t)stream, a, n_engines, out, HW);
    return check_launch("aotb_soft_logit_aggregation_f32");
}


extern "C" int aotb_separate_labels_f32(const float* mask, int n_engines, int max_obj, float* out, int HW, void* stream) {
    AOTB_REQUIRE(mask && out && n_engines >= 1 && max_obj >= 1 && HW > 0, "aotb_separate_labels_f32: bad args");
    int g = cdiv(HW, 256);
    if (g > 132 * 8) g = 132 * 8;
    launch(separate_labels_kernel, dim3(g), dim3(256), 0, (cudaStream_t)stream, mask, n_engines, max_obj, out, HW);
    return check_launch("aotb_separate_labels_f32");
}

// logits: decoder output [lanes][h][w][NC] (NHWC); video b's k[b] = lane_ptr[b + 1] - lane_ptr[b] lanes are
// lanes[lane_ptr[b] ..], with object counts obj_nums[lane_ptr[b] ..]; out / label: n_videos pointers or null arrays.
extern "C" int aotb_soft_logit_aggregation_batched_f32(const float* logits, int h, int w, int NC, const int* lane_ptr,
                                                       const int* lanes, const int* obj_nums, int n_videos, int max_obj,
                                                       int Ho, int Wo, int align_corners, float* const* out,
                                                       float* const* label, void* stream) {
    AOTB_REQUIRE(logits && lane_ptr && lanes && obj_nums && n_videos > 0 && h > 0 && w > 0 && Ho > 0 && Wo > 0 && (out || label),
                 "aotb_soft_logit_aggregation_batched_f32: bad args");
    AOTB_REQUIRE(max_obj == 10 && NC == 11, "aotb_soft_logit_aggregation_batched_f32: built for MODEL_MAX_OBJ_NUM = 10 (got "
                 "max_obj %d, NC %d)", max_obj, NC);
    AOTB_REQUIRE((size_t)h * w * NC < (1u << 31), "aotb_soft_logit_aggregation_batched_f32: lane too large");
    const size_t plane = (size_t)Ho * Wo;
    AggBatchArgs a;
    int launches = 0;
    for (int v0 = 0; v0 < n_videos; v0 += AGG_BATCH, ++launches) {
        const int nb = n_videos - v0 < AGG_BATCH ? n_videos - v0 : AGG_BATCH;
        for (int b = 0; b < nb; ++b) {
            const int p = lane_ptr[v0 + b], k = lane_ptr[v0 + b + 1] - p;
            AOTB_REQUIRE(k >= 1 && k <= 8, "aotb_soft_logit_aggregation_batched_f32: video %d: 1 to 8 lanes (got %d)", v0 + b, k);
            for (int e = 0; e < 8; ++e) {
                a.lane[b][e] = e < k ? lanes[p + e] : 0;
                a.obj[b][e] = e < k ? obj_nums[p + e] : 0;
                AOTB_REQUIRE(a.lane[b][e] >= 0, "aotb_soft_logit_aggregation_batched_f32: video %d: negative lane", v0 + b);
            }
            a.k[b] = k;
            a.out[b] = out ? out[v0 + b] : nullptr;
            a.label[b] = label ? label[v0 + b] : nullptr;
            AOTB_REQUIRE(a.out[b] || a.label[b], "aotb_soft_logit_aggregation_batched_f32: video %d: no output", v0 + b);
        }
        int g = cdiv((int)plane, 256);
        if (g > 132 * 8) g = 132 * 8;
        launch(soft_logit_aggregation_batched_kernel<11>, dim3(g, nb), dim3(256), 0, (cudaStream_t)stream, logits, h, w, Ho, Wo,
               align_corners, a);
    }
    return check_launch("aotb_soft_logit_aggregation_batched_f32", launches);
}

extern "C" int aotb_separate_labels_batched_f32(const float* const* labels, const int* parts, int n, int max_obj,
                                                float* const* out, int HW, void* stream) {
    AOTB_REQUIRE(labels && parts && out && n > 0 && max_obj >= 1 && HW > 0, "aotb_separate_labels_batched_f32: bad args");
    SepBatchArgs a;
    int g = cdiv(HW, 256);
    if (g > 132 * 8) g = 132 * 8;
    int launches = 0;
    for (int b0 = 0; b0 < n; b0 += SEP_BATCH, ++launches) {
        const int nb = n - b0 < SEP_BATCH ? n - b0 : SEP_BATCH;
        for (int b = 0; b < nb; ++b) {
            a.label[b] = labels[b0 + b];
            a.out[b] = out[b0 + b];
            a.part[b] = parts[b0 + b];
            AOTB_REQUIRE(a.label[b] && a.out[b] && a.part[b] >= 0, "aotb_separate_labels_batched_f32: entry %d: bad map or part",
                         b0 + b);
        }
        launch(separate_labels_batched_kernel, dim3(g, nb), dim3(256), 0, (cudaStream_t)stream, a, max_obj, HW);
    }
    return check_launch("aotb_separate_labels_batched_f32", launches);
}

extern "C" int aotb_lane_gather_f32(const float* const* src, float* const* dst, const int* n_floats, int n_maps,
                                    const int* lane_video, int n_lanes, int n_videos, void* stream) {
    AOTB_REQUIRE(src && dst && n_floats && lane_video && n_maps >= 1 && n_maps <= 4 && n_lanes >= 1 && n_lanes <= 65535 &&
                 n_videos >= 1, "aotb_lane_gather_f32: bad args");
    LaneGatherArgs a;
    int most = 0;
    for (int j = 0; j < 4; ++j) {
        const bool live = j < n_maps;
        a.src[j] = live ? src[j] : nullptr;
        a.dst[j] = live ? dst[j] : nullptr;
        a.n4[j] = live ? n_floats[j] / 4 : 0;
        AOTB_REQUIRE(!live || (a.src[j] && a.dst[j] && n_floats[j] > 0 && n_floats[j] % 4 == 0 &&
                               ((uintptr_t)a.src[j] | (uintptr_t)a.dst[j]) % 16 == 0),
                     "aotb_lane_gather_f32: map %d: null, unaligned or not a multiple of 4 floats", j);
        if (a.n4[j] > most) most = a.n4[j];
    }
    int g = cdiv(most, 256);
    if (g > 132 * 4) g = 132 * 4;
    launch(lane_gather_kernel, dim3(g, n_lanes), dim3(256), 0, (cudaStream_t)stream, a, n_maps, lane_video, n_videos);
    return check_launch("aotb_lane_gather_f32");
}

extern "C" int aotb_bank_append_f32(const float* src, int lds, float* bank, int ldb, int rows, int cols, int offset,
                                    const int* offset_dev, void* stream) {
    AOTB_REQUIRE(src && bank && rows > 0 && cols > 0 && cols % 4 == 0 && lds % 4 == 0 && ldb % 4 == 0,
                 "aotb_bank_append_f32: bad args");
    const size_t total = (size_t)rows * (cols / 4);
    int g = (int)((total + 255) / 256);
    if (g > 132 * 8) g = 132 * 8;
    launch(bank_append_kernel, dim3(g), dim3(256), 0, (cudaStream_t)stream, src, lds, bank, ldb, rows, cols / 4, offset, offset_dev);
    return check_launch("aotb_bank_append_f32");
}

extern "C" int aotb_counter_add(int* counter, int delta, void* stream) {
    AOTB_REQUIRE(counter, "aotb_counter_add: null");
    launch(counter_add_kernel, dim3(1), dim3(1), 0, (cudaStream_t)stream, counter, delta);
    return check_launch("aotb_counter_add");
}

extern "C" int aotb_bank_ring_store(const float* k_src, int ldk, int k_cols, const float* v_src, int ldv, int v_cols, int rows,
                                    float* k_bank, int ldkb, float* v_bank, int ldvb, void* k_packed, void* v_packed,
                                    int cap_rows, const int* write, void* stream) {
    AOTB_REQUIRE(k_src && v_src && write && rows > 0 && rows <= cap_rows, "aotb_bank_ring_store: bad args");
    AOTB_REQUIRE(k_bank || v_bank || k_packed || v_packed, "aotb_bank_ring_store: no destination");
    AOTB_REQUIRE(k_cols > 0 && v_cols > 0 && k_cols % 4 == 0 && v_cols % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 &&
                 ldk >= k_cols && ldv >= v_cols, "aotb_bank_ring_store: columns and row strides must be multiples of 4");
    AOTB_REQUIRE((!k_bank || (ldkb % 4 == 0 && ldkb >= k_cols)) && (!v_bank || (ldvb % 4 == 0 && ldvb >= v_cols)),
                 "aotb_bank_ring_store: bank row stride");
    AOTB_REQUIRE((!k_packed || k_cols % 32 == 0) && (!v_packed || v_cols % 32 == 0),
                 "aotb_bank_ring_store: a packed copy needs a multiple of 32 channels");
    AOTB_REQUIRE(((uintptr_t)k_src | (uintptr_t)v_src | (uintptr_t)k_bank | (uintptr_t)v_bank | (uintptr_t)k_packed |
                  (uintptr_t)v_packed) % 16 == 0, "aotb_bank_ring_store: alignment");
    RingStoreArgs a;
    a.src[0] = k_src; a.src[1] = v_src; a.bank[0] = k_bank; a.bank[1] = v_bank;
    a.packed[0] = (__half*)k_packed; a.packed[1] = (__half*)v_packed;
    a.ld[0] = ldk; a.ld[1] = ldv; a.ldb[0] = ldkb; a.ldb[1] = ldvb; a.c4[0] = k_cols / 4; a.c4[1] = v_cols / 4;
    const size_t total = (size_t)rows * (a.c4[0] + a.c4[1]);
    int g = (int)((total + 255) / 256);
    if (g > 132 * 8) g = 132 * 8;
    launch(bank_ring_store_kernel, dim3(g), dim3(256), 0, (cudaStream_t)stream, a, rows, cap_rows, write);
    return check_launch("aotb_bank_ring_store");
}

extern "C" int aotb_ring_advance(int* live, int* write, int rows, int cap_rows, int pinned_rows, void* stream) {
    AOTB_REQUIRE(live && write, "aotb_ring_advance: null counter");
    AOTB_REQUIRE(rows > 0 && pinned_rows >= 0 && (long long)pinned_rows + rows <= cap_rows &&
                 (cap_rows - pinned_rows) % rows == 0,
                 "aotb_ring_advance: need rows > 0, pinned_rows + rows <= cap_rows and (cap_rows - pinned_rows) %% rows == 0 "
                 "(got rows %d, cap_rows %d, pinned_rows %d)", rows, cap_rows, pinned_rows);
    launch(ring_advance_kernel, dim3(1), dim3(1), 0, (cudaStream_t)stream, live, write, rows, cap_rows, pinned_rows);
    return check_launch("aotb_ring_advance");
}

extern "C" int aotb_ring_select_usage(const int* live, int* write, float* U, int* A, int rows, int cap_rows, int pinned_rows,
                                      void* stream) {
    AOTB_REQUIRE(live && write && U && A, "aotb_ring_select_usage: null pointer");
    AOTB_REQUIRE(rows > 0 && pinned_rows >= 0 && pinned_rows % rows == 0 && cap_rows % rows == 0 &&
                     pinned_rows + rows <= cap_rows,
                 "aotb_ring_select_usage: need rows > 0, pinned_rows and cap_rows multiples of rows and pinned_rows + rows <= "
                 "cap_rows (rows %d, cap_rows %d, pinned_rows %d)", rows, cap_rows, pinned_rows);
    launch(ring_select_usage_kernel, dim3(1), dim3(1), 0, (cudaStream_t)stream, live, write, U, A, rows, cap_rows, pinned_rows);
    return check_launch("aotb_ring_select_usage");
}

extern "C" int aotb_id_embed_runs_batched_f32(const float* mask, int n, int Hm, int Wm, const float* wp, const float* bias,
                                              const float* ln_gamma, const float* ln_beta, float* out, int ldo, int C, int nid,
                                              int ksize, int stride, int pad, void* stream) {
    AOTB_REQUIRE(mask && wp && bias && out && n >= 1 && n <= 65535 && Hm > 0 && Wm > 0,
                 "aotb_id_embed_runs_batched_f32: bad args");
    AOTB_REQUIRE(ksize <= 17 && ksize > 0 && stride > 0 && C == 256 && nid < 128,
                 "aotb_id_embed_runs_batched_f32: unsupported shape");
    const int ho = (Hm + 2 * pad - ksize) / stride + 1, wo = (Wm + 2 * pad - ksize) / stride + 1;
    AOTB_REQUIRE(ho > 0 && wo > 0, "aotb_id_embed_runs_batched_f32: empty output");
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid(ho * wo, n);
    if (ln_gamma) {
        AOTB_REQUIRE(ln_beta, "aotb_id_embed_runs_batched_f32: ln_beta");
        launch(id_embed_runs_batched_kernel<true>, grid, dim3(256), 0, st, mask, Hm, Wm, wp, bias, ln_gamma, ln_beta, out, ldo,
               ho, wo, C, nid, ksize, stride, pad);
    } else {
        launch(id_embed_runs_batched_kernel<false>, grid, dim3(256), 0, st, mask, Hm, Wm, wp, bias, nullptr, nullptr, out, ldo,
               ho, wo, C, nid, ksize, stride, pad);
    }
    return check_launch("aotb_id_embed_runs_batched_f32");
}

extern "C" int aotb_bank_ring_store_batched(const float* k_src, int ldk, int k_cols, const float* v_src, int ldv, int v_cols,
                                            int rows, int n, float* k_bank, int ldkb, float* v_bank, int ldvb, void* k_packed,
                                            void* v_packed, int cap_rows, int head_rows, const int* write, const int* store,
                                            void* stream) {
    AOTB_REQUIRE(k_src && v_src && write && store && rows > 0 && rows <= cap_rows && n >= 1 && n <= 65535,
                 "aotb_bank_ring_store_batched: bad args");
    AOTB_REQUIRE(k_bank || v_bank || k_packed || v_packed, "aotb_bank_ring_store_batched: no destination");
    AOTB_REQUIRE((long long)n * cap_rows <= head_rows, "aotb_bank_ring_store_batched: packed chunk stride");
    AOTB_REQUIRE(k_cols > 0 && v_cols > 0 && k_cols % 4 == 0 && v_cols % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 &&
                 ldk >= k_cols && ldv >= v_cols, "aotb_bank_ring_store_batched: columns and row strides must be multiples of 4");
    AOTB_REQUIRE((!k_bank || (ldkb % 4 == 0 && ldkb >= k_cols)) && (!v_bank || (ldvb % 4 == 0 && ldvb >= v_cols)),
                 "aotb_bank_ring_store_batched: bank row stride");
    AOTB_REQUIRE((!k_packed || k_cols % 32 == 0) && (!v_packed || v_cols % 32 == 0),
                 "aotb_bank_ring_store_batched: a packed copy needs a multiple of 32 channels");
    AOTB_REQUIRE(((uintptr_t)k_src | (uintptr_t)v_src | (uintptr_t)k_bank | (uintptr_t)v_bank | (uintptr_t)k_packed |
                  (uintptr_t)v_packed) % 16 == 0, "aotb_bank_ring_store_batched: alignment");
    RingStoreArgs a;
    a.src[0] = k_src; a.src[1] = v_src; a.bank[0] = k_bank; a.bank[1] = v_bank;
    a.packed[0] = (__half*)k_packed; a.packed[1] = (__half*)v_packed;
    a.ld[0] = ldk; a.ld[1] = ldv; a.ldb[0] = ldkb; a.ldb[1] = ldvb; a.c4[0] = k_cols / 4; a.c4[1] = v_cols / 4;
    const size_t total = (size_t)rows * (a.c4[0] + a.c4[1]);
    int g = (int)((total + 255) / 256);
    if (g > 132 * 8) g = 132 * 8;
    launch(bank_ring_store_batched_kernel, dim3(g, n), dim3(256), 0, (cudaStream_t)stream, a, rows, cap_rows, head_rows, write,
           store);
    return check_launch("aotb_bank_ring_store_batched");
}

extern "C" int aotb_ring_advance_batched(int* live, int* write, const int* store, int n, int rows, int cap_rows, int pinned_rows,
                                         void* stream) {
    AOTB_REQUIRE(live && write && store && n >= 1 && n <= 1024, "aotb_ring_advance_batched: bad args");
    AOTB_REQUIRE(rows > 0 && pinned_rows >= 0 && (long long)pinned_rows + rows <= cap_rows &&
                 (cap_rows - pinned_rows) % rows == 0,
                 "aotb_ring_advance_batched: need rows > 0, pinned_rows + rows <= cap_rows and (cap_rows - pinned_rows) %% rows "
                 "== 0 (got rows %d, cap_rows %d, pinned_rows %d)", rows, cap_rows, pinned_rows);
    launch(ring_advance_batched_kernel, dim3(1), dim3(32 * ((n + 31) / 32)), 0, (cudaStream_t)stream, live, write, store, n, rows,
           cap_rows, pinned_rows);
    return check_launch("aotb_ring_advance_batched");
}
