// LayerNorm over channels and GroupNorm over (pixels x channels-in-group), NHWC fp32.
//
// Reference sites: nn.LayerNorm(256) norm1/norm2/norm3, decoder_norms, id_norm*
// (transformer.py:274,293,297,85-93,530,537,565-566; deaot.py:39,53); with_pos_embed
// (transformer.py:305-310,322: q = k = LN(x) + pos -> emitted as a second output here);
// GroupNorm(32,1024)+GELU of the FFN (basic.py:18,30-32), GroupNorm(8,C)+ReLU of ConvGN
// (basic.py:75-85, fpn.py:41-56), GroupNorm1D(512, groups=2) (basic.py:6-12, transformer.py:197-200).
// eps = 1e-5 everywhere (PyTorch default).
//
// GroupNorm statistics are reduced deterministically (fixed partial layout, double precision
// partials) so replicated ranks stay bit-identical (SURVEY 7.6).
#include "common.cuh"
#include <cstdint>

namespace aotb {

// one warp per row; C % 4 == 0; C <= 4096
__global__ void layernorm_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, const float* __restrict__ add, int ldadd,
                                 float* __restrict__ out, int ldo, float* __restrict__ out2, int ldo2, int rows,
                                 int C, float eps) {
    pdl_sync();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const float* xr = x + (size_t)warp * ldx;
    float s = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
        float4 v = *reinterpret_cast<const float4*>(xr + c);
        s += (v.x + v.y) + (v.z + v.w);
    }
    s = warp_sum(s);
    const float mean = s / (float)C;
    float q = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
        float4 v = *reinterpret_cast<const float4*>(xr + c);
        float a = v.x - mean, b = v.y - mean, cc = v.z - mean, d = v.w - mean;
        q += (a * a + b * b) + (cc * cc + d * d);
    }
    q = warp_sum(q);
    const float rstd = rsqrtf(q / (float)C + eps);
    for (int c = lane * 4; c < C; c += 128) {
        float4 v = *reinterpret_cast<const float4*>(xr + c);
        float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
        float4 b = __ldg(reinterpret_cast<const float4*>(beta + c));
        float4 o;
        o.x = (v.x - mean) * rstd * g.x + b.x;
        o.y = (v.y - mean) * rstd * g.y + b.y;
        o.z = (v.z - mean) * rstd * g.z + b.z;
        o.w = (v.w - mean) * rstd * g.w + b.w;
        *reinterpret_cast<float4*>(out + (size_t)warp * ldo + c) = o;
        if (out2) {
            float4 p = __ldg(reinterpret_cast<const float4*>(add + (size_t)warp * ldadd + c));
            o.x += p.x; o.y += p.y; o.z += p.z; o.w += p.w;
            *reinterpret_cast<float4*>(out2 + (size_t)warp * ldo2 + c) = o;
        }
    }
}

// ---- GroupNorm, stage 1: partial (sum, sumsq) per (b, g, chunk) in double
// x [B][P][ldx] (P pixels), group g covers channels [g*Cg, (g+1)*Cg)
constexpr int GN_CHUNKS = 64;

// `chunks` (a multiple of 8, <= GN_CHUNKS) pixel ranges per (b, g): enough blocks to fill the GPU on the large decoder maps, few
// enough on the 31 x 54 token maps that a block has more than one load per thread (2 048 blocks of 208 float4 took 9.8 us).
//
// The sums are taken about a shift K = x[b][0][g*Cg], the first element of the group: S = sum(v - K), Q = sum((v - K)^2), and
// the finaliser forms mean = K + S/n, var = Q/n - (S/n)^2.  The raw sums sum(v), sum(v^2) cancel catastrophically in
// E[v^2] - mean^2 once |mean| is large next to the standard deviation (on the FFN shape at mean/std = 1000, gamma = 1, the
// raw-sum form was off by 4.8e-2 on an H100, the shifted one by 4.1e-5); about K the cancellation is only that of
// (K - mean)^2, a few variances.  Every block reads the same K, so the result does not
// depend on the launch.
__global__ void groupnorm_stats_kernel(const float* __restrict__ x, int ldx, int P, int G, int Cg,
                                       double* __restrict__ partial, float* __restrict__ stat, unsigned* __restrict__ counter,
                                       float eps) {
    pdl_sync();
    const int chunk = blockIdx.x, g = blockIdx.y, b = blockIdx.z, chunks = gridDim.x;
    const int per = (P + chunks - 1) / chunks;
    const int p0 = chunk * per, p1 = min(P, p0 + per);
    const float* xb = x + (size_t)b * P * ldx + (size_t)g * Cg;
    const float K = xb[0];
    const int Cg4 = Cg >> 2;
    float s = 0.f, q = 0.f;
    const int n = (p1 > p0 ? (p1 - p0) : 0) * Cg4;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int p = p0 + i / Cg4, c = (i % Cg4) * 4;
        const float4 v = *reinterpret_cast<const float4*>(xb + (size_t)p * ldx + c);
        const float a = v.x - K, bb = v.y - K, cc = v.z - K, d = v.w - K;
        s += (a + bb) + (cc + d);
        q += (a * a + bb * bb) + (cc * cc + d * d);
    }
    __shared__ double sh[2][8];
    __shared__ unsigned last;
    double ds = (double)warp_sum(s), dq = (double)warp_sum(q);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) { sh[0][wid] = ds; sh[1][wid] = dq; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, c = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { a += sh[0][w]; c += sh[1][w]; }
        double* o = partial + (((size_t)b * G + g) * GN_CHUNKS + chunk) * 2;
        o[0] = a; o[1] = c;
        __threadfence();
        last = atomicAdd(counter, 1u) == gridDim.x * gridDim.y * gridDim.z - 1 ? 1u : 0u;
    }
    __syncthreads();
    if (!last) return;
    // The block that arrives last turns the partials into (mean, rstd) per (b, g) -- ONCE, in a fixed order (8 threads per group
    // sum 8 chunks each in order, then a fixed xor tree), whichever block it is.  The apply kernel used to redo this in every one
    // of its ~1200 blocks (32 KB of double partials each: 17 us per launch for 14 MB of payload).
    __threadfence();
    const int BG = gridDim.z * G;
    for (int g0 = 0; g0 < BG; g0 += blockDim.x / 8) {
        const int bg = g0 + (threadIdx.x >> 3), sub = threadIdx.x & 7;
        double ss = 0, qq = 0;
        if (bg < BG) {
            const int cps = chunks / 8;                      // chunks per summing thread
            const volatile double* pp = partial + ((size_t)bg * GN_CHUNKS + sub * cps) * 2;
            for (int c = 0; c < cps; ++c) { ss += pp[2 * c]; qq += pp[2 * c + 1]; }
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
            ss += __shfl_xor_sync(0xffffffffu, ss, o);
            qq += __shfl_xor_sync(0xffffffffu, qq, o);
        }
        if (bg < BG && sub == 0) {
            // the shift of this (b, g), as its stats blocks read it: x is not written before the apply kernel runs
            const double shift = x[(size_t)(bg / G) * P * ldx + (size_t)(bg % G) * Cg];
            const double nn = (double)P * Cg;
            const double dm = ss / nn;
            double var = qq / nn - dm * dm;
            if (var < 0) var = 0;
            stat[2 * bg] = (float)(shift + dm);
            stat[2 * bg + 1] = (float)(1.0 / sqrt(var + (double)eps));
        }
    }
    if (threadIdx.x == 0) *counter = 0u;          // ready for the next launch
}

// ---- stage 2: normalise + affine + activation
__global__ void groupnorm_apply_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, const float* __restrict__ gstat,
                                       float* __restrict__ out, int ldo, int P, int C, int G, int Cg, int act) {
    pdl_sync();
    extern __shared__ float stat[];  // [G][2] mean, rstd for this batch element (finalised by the stats kernel's last block)
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) stat[i] = gstat[(size_t)b * 2 * G + i];
    __syncthreads();
    const int C4 = C >> 2;
    const size_t total = (size_t)P * C4;
    const float* xb = x + (size_t)b * P * ldx;
    float* ob = out + (size_t)b * P * ldo;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int p = i / C4, c = (i - (size_t)p * C4) * 4;
        const int g = c / Cg;
        const float mean = stat[2 * g], rstd = stat[2 * g + 1];
        float4 v = *reinterpret_cast<const float4*>(xb + (size_t)p * ldx + c);
        float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c));
        float4 be = __ldg(reinterpret_cast<const float4*>(beta + c));
        float4 o;
        o.x = apply_act((v.x - mean) * rstd * ga.x + be.x, act);
        o.y = apply_act((v.y - mean) * rstd * ga.y + be.y, act);
        o.z = apply_act((v.z - mean) * rstd * ga.z + be.z, act);
        o.w = apply_act((v.w - mean) * rstd * ga.w + be.w, act);
        *reinterpret_cast<float4*>(ob + (size_t)p * ldo + c) = o;
    }
}

}  // namespace aotb

using namespace aotb;

extern "C" int aotb_layernorm_f32(const float* x, int ldx, const float* gamma, const float* beta, const float* add,
                                  int ldadd, float* out, int ldo, float* out2, int ldo2, int rows, int C,
                                  void* stream) {
    AOTB_REQUIRE(x && gamma && beta && out && rows > 0, "aotb_layernorm_f32: bad args");
    AOTB_REQUIRE(C % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0, "aotb_layernorm_f32: C/ld must be %%4");
    AOTB_REQUIRE(!out2 || (add && ldadd % 4 == 0 && ldo2 % 4 == 0), "aotb_layernorm_f32: out2 needs add");
    const int warps_per_block = 8;
    launch(layernorm_kernel, dim3(cdiv(rows, warps_per_block)), dim3(warps_per_block * 32), 0, (cudaStream_t)stream, x, ldx, gamma, beta, add, ldadd, out, ldo, out2, ldo2, rows, C, 1e-5f);
    return check_launch("aotb_layernorm_f32");
}

// workspace = [launch counter, 256 B][(mean, rstd) floats: 8 KB per batch element][double partials]; it must be ZERO when first
// used (the counter) and is left ready for the next call.
static constexpr size_t GN_HDR = 256, GN_STAT = 8192;

extern "C" size_t aotb_groupnorm_workspace_bytes(int B, int G) {
    return GN_HDR + (size_t)B * GN_STAT + (size_t)B * G * GN_CHUNKS * 2 * sizeof(double);
}

extern "C" int aotb_groupnorm_nhwc_f32(const float* x, int ldx, const float* gamma, const float* beta, float* out,
                                       int ldo, int B, int P, int C, int G, int act, void* workspace,
                                       void* stream) {
    AOTB_REQUIRE(x && gamma && beta && out && workspace, "aotb_groupnorm_nhwc_f32: null pointer");
    AOTB_REQUIRE(G > 0 && C % G == 0 && (C / G) % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0 && G <= 1024,
                 "aotb_groupnorm_nhwc_f32: unsupported channel/group configuration");
    AOTB_REQUIRE(act >= ACT_NONE && act <= ACT_RELU6, "aotb_groupnorm_nhwc_f32: activation %d not supported (0-4)", act);
    const int Cg = C / G;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned* counter = (unsigned*)workspace;
    float* stat = (float*)((uint8_t*)workspace + GN_HDR);
    double* partial = (double*)((uint8_t*)workspace + GN_HDR + (size_t)B * GN_STAT);
    int chunks = (int)(((size_t)P * (Cg / 4) + 1023) / 1024);          // ~4 float4 loads per thread and block
    chunks = ((chunks + 7) / 8) * 8;
    chunks = chunks < 8 ? 8 : (chunks > GN_CHUNKS ? GN_CHUNKS : chunks);
    launch(groupnorm_stats_kernel, dim3(dim3(chunks, G, B)), dim3(256), 0, st, x, ldx, P, G, Cg, partial, stat, counter, 1e-5f);
    const size_t total = (size_t)P * (C / 4);
    int gx = (int)((total + 255) / 256);
    if (gx > 132 * 8) gx = 132 * 8;
    launch(groupnorm_apply_kernel, dim3(dim3(gx, B)), dim3(256), 2 * G * sizeof(float), st, x, ldx, gamma, beta,
                                                                             (const float*)stat, out, ldo, P, C, G, Cg, act);
    return check_launch("aotb_groupnorm_nhwc_f32", 2);
}
