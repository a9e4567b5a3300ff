// Fused softmax(Q K^T / T) V, fp32-exact SIMT flash-style kernel (scores never materialised).
//
// Restates the arithmetic core of MultiheadAttention.forward (networks/layers/attention.py:82-117:
// Q / T true division :82, per-head Q K^T :97, softmax over keys :107, @V :113) and of
// GatedPropagation.forward (:672-704) for every head layout the reference uses:
//   AOT  long-term / self-attention : H = 8, d_qk = 32,  d_v = 32   (transformer.py:278-281,294)
//   DeAOT long-term / self-attention: H = 1, d_qk = 128, d_v = 1024 (transformer.py:541-548,567-570)
// This is the reference-precision path (and the in-library cross-check for the tensor-core kernel in
// lt_attn_tc.cu); Q/K/V/O are [rows][ld] fp32 with head h at columns h*d.
//
// CTA = 64 queries x one head x one DVC-wide value chunk; 256 threads as 16x16, each owning a
// 4x4 score micro-tile and a 4 x (DVC/16) output micro-tile; K/V streamed in 64-key tiles.
#include "common.cuh"

namespace aotb {

struct AttnArgs {
    const float* Q; int ldq;
    const float* K; int ldk;
    const float* V; int ldv;
    float* O; int ldo;
    int N, Tk;
    const int* Tk_dev;   // optional device-resident key count (CUDA-graph friendly)
    float T;             // sqrt(d_att); scores use (q / T) . k
    int dv_head;         // value width per head
    float* Mout;         // optional split-KV partial statistics [H][N] (row max, row sum)
    float* Lout;
    int kv_begin_frames; // unused (reserved)
};

template <int DQK, int DVC>
__global__ void __launch_bounds__(256) attn_f32_kernel(const AttnArgs p) {
    pdl_sync();
    constexpr int BM = 64, BN = 64, LDS_ = BM + 4;
    constexpr int TNV = DVC / 16;
    extern __shared__ __align__(16) float smem[];
    float* Qt = smem;                       // [DQK][LDS_]
    float* Kt = Qt + DQK * LDS_;            // [DQK][LDS_]
    float* Pt = Kt + DQK * LDS_;            // [BN][LDS_]   (P transposed: [key][query])
    float* Vs = Pt + BN * LDS_;             // [BN][DVC + 4]
    constexpr int LDV = DVC + 4;

    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int q0 = blockIdx.x * BM, h = blockIdx.y, vc = blockIdx.z;
    const int Tk = p.Tk_dev ? *p.Tk_dev : p.Tk;
    const float* Qh = p.Q + (size_t)h * DQK;
    const float* Kh = p.K + (size_t)h * DQK;
    const float* Vh = p.V + (size_t)h * p.dv_head + (size_t)vc * DVC;

    // ---- Q tile, scaled by true division (attention.py:82), stored transposed
    for (int f = tid; f < BM * (DQK / 4); f += 256) {
        const int row = f / (DQK / 4), kq = (f % (DQK / 4)) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q0 + row < p.N) v = *reinterpret_cast<const float4*>(Qh + (size_t)(q0 + row) * p.ldq + kq);
        Qt[(kq + 0) * LDS_ + row] = v.x / p.T;
        Qt[(kq + 1) * LDS_ + row] = v.y / p.T;
        Qt[(kq + 2) * LDS_ + row] = v.z / p.T;
        Qt[(kq + 3) * LDS_ + row] = v.w / p.T;
    }

    float m_run[4], l_run[4], o[4][TNV];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        m_run[i] = -INFINITY;
        l_run[i] = 0.f;
#pragma unroll
        for (int j = 0; j < TNV; ++j) o[i][j] = 0.f;
    }

    for (int k0 = 0; k0 < Tk; k0 += BN) {
        __syncthreads();  // previous tile fully consumed (also covers the Q tile on first trip)
        for (int f = tid; f < BN * (DQK / 4); f += 256) {
            const int row = f / (DQK / 4), kq = (f % (DQK / 4)) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k0 + row < Tk) v = __ldg(reinterpret_cast<const float4*>(Kh + (size_t)(k0 + row) * p.ldk + kq));
            Kt[(kq + 0) * LDS_ + row] = v.x;
            Kt[(kq + 1) * LDS_ + row] = v.y;
            Kt[(kq + 2) * LDS_ + row] = v.z;
            Kt[(kq + 3) * LDS_ + row] = v.w;
        }
        for (int f = tid; f < BN * (DVC / 4); f += 256) {
            const int row = f / (DVC / 4), c = (f % (DVC / 4)) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k0 + row < Tk) v = __ldg(reinterpret_cast<const float4*>(Vh + (size_t)(k0 + row) * p.ldv + c));
            *reinterpret_cast<float4*>(Vs + row * LDV + c) = v;
        }
        __syncthreads();

        // ---- S = (Q/T) K^T micro-tile
        float s[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
        for (int k = 0; k < DQK; ++k) {
            const float4 a = *reinterpret_cast<const float4*>(Qt + k * LDS_ + ty * 4);
            const float4 b = *reinterpret_cast<const float4*>(Kt + k * LDS_ + tx * 4);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s[i][j] = fmaf(av[i], bv[j], s[i][j]);
        }
        // ---- online softmax (rows are shared by the 16 tx-lanes of a half warp)
        float corr[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (k0 + tx * 4 + j >= Tk) s[i][j] = -INFINITY;
                mx = fmaxf(mx, s[i][j]);
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            const float m_new = fmaxf(m_run[i], mx);
            corr[i] = (m_run[i] == -INFINITY) ? 0.f : expf(m_run[i] - m_new);
            float rs = 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float e = expf(s[i][j] - m_new);  // exp(-inf) == 0 for masked keys
                s[i][j] = e;
                rs += e;
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
            l_run[i] = l_run[i] * corr[i] + rs;
            m_run[i] = m_new;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
            *reinterpret_cast<float4*>(Pt + (tx * 4 + j) * LDS_ + ty * 4) =
                make_float4(s[0][j], s[1][j], s[2][j], s[3][j]);
        __syncthreads();

        // ---- O = O * corr + P V
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < TNV; ++j) o[i][j] *= corr[i];
#pragma unroll 4
        for (int kk = 0; kk < BN; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(Pt + kk * LDS_ + ty * 4);
            const float av[4] = {a.x, a.y, a.z, a.w};
            float bv[TNV];
            if constexpr (TNV == 2) {
                const float2 b = *reinterpret_cast<const float2*>(Vs + kk * LDV + tx * 2);
                bv[0] = b.x; bv[1] = b.y;
            } else {
#pragma unroll
                for (int g = 0; g < TNV / 4; ++g) {
                    const float4 b = *reinterpret_cast<const float4*>(Vs + kk * LDV + g * 64 + tx * 4);
                    bv[g * 4 + 0] = b.x; bv[g * 4 + 1] = b.y; bv[g * 4 + 2] = b.z; bv[g * 4 + 3] = b.w;
                }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < TNV; ++j) o[i][j] = fmaf(av[i], bv[j], o[i][j]);
        }
    }

    // ---- epilogue
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int q = q0 + ty * 4 + i;
        if (q >= p.N) continue;
        const bool partial = (p.Mout != nullptr);
        const float inv = partial ? 1.f : 1.f / l_run[i];
        float* orow = p.O + (size_t)q * p.ldo + (size_t)h * p.dv_head + (size_t)vc * DVC;
        if constexpr (TNV == 2) {
            *reinterpret_cast<float2*>(orow + tx * 2) = make_float2(o[i][0] * inv, o[i][1] * inv);
        } else {
#pragma unroll
            for (int g = 0; g < TNV / 4; ++g)
                *reinterpret_cast<float4*>(orow + g * 64 + tx * 4) =
                    make_float4(o[i][g * 4] * inv, o[i][g * 4 + 1] * inv, o[i][g * 4 + 2] * inv, o[i][g * 4 + 3] * inv);
        }
        if (partial && tx == 0 && vc == 0) {
            p.Mout[(size_t)h * p.N + q] = m_run[i];
            p.Lout[(size_t)h * p.N + q] = l_run[i];
        }
    }
}

template <int DQK, int DVC>
static int launch_attn(const AttnArgs& a, int H, cudaStream_t st) {
    constexpr int LDS_ = 64 + 4;
    const size_t smem = sizeof(float) * (size_t)(2 * DQK * LDS_ + 64 * LDS_ + 64 * (DVC + 4));
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(attn_f32_kernel<DQK, DVC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem);
        if (e != cudaSuccess) {
            set_error("aotb_attention_f32: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    dim3 grid(cdiv(a.N, 64), H, a.dv_head / DVC);
    launch(attn_f32_kernel<DQK, DVC>, dim3(grid), dim3(256), smem, st, a);
    return check_launch("aotb_attention_f32");
}

}  // namespace aotb

using namespace aotb;

// Q [N][ldq], K [Tk][ldk], V [Tk][ldv], O [N][ldo]; head h uses Q/K columns [h*d_qk, (h+1)*d_qk)
// and V/O columns [h*d_v, (h+1)*d_v).  If Mout/Lout are given the un-normalised partial
// (m, l, O) of a split-KV shard is written instead (merged by aotb_attn_merge_f32).
extern "C" int aotb_attention_f32(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                                  float* O, int ldo, int N, int Tk, const int* Tk_dev, int H, int d_qk, int d_v,
                                  float* Mout, float* Lout, void* stream) {
    AOTB_REQUIRE(Q && K && V && O && N > 0 && (Tk > 0 || Tk_dev) && H > 0, "aotb_attention_f32: bad args");
    AOTB_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0, "aotb_attention_f32: ld %% 4");
    AOTB_REQUIRE((Mout == nullptr) == (Lout == nullptr), "aotb_attention_f32: Mout/Lout go together");
    AttnArgs a;
    a.Q = Q; a.ldq = ldq; a.K = K; a.ldk = ldk; a.V = V; a.ldv = ldv; a.O = O; a.ldo = ldo;
    a.N = N; a.Tk = Tk; a.Tk_dev = Tk_dev; a.T = sqrtf((float)d_qk); a.dv_head = d_v;
    a.Mout = Mout; a.Lout = Lout; a.kv_begin_frames = 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (d_qk == 32 && d_v == 32) return launch_attn<32, 32>(a, H, st);
    if (d_qk == 128 && d_v % 256 == 0) return launch_attn<128, 256>(a, H, st);
    if (d_qk == 32 && d_v % 64 == 0) return launch_attn<32, 64>(a, H, st);
    set_error("aotb_attention_f32: unsupported head shape d_qk=%d d_v=%d", d_qk, d_v);
    return AOTB_ERR_UNSUPPORTED;
}

// ---------------------------------------------------------------- split-KV merge (cfg4 row e)
// O = sum_r exp(m_r - m) O_r / sum_r exp(m_r - m) l_r  with m = max_r m_r  (exact LSE merge)
namespace aotb {
// USAGE (aotb_attn_merge_usage_f32): split r is memory slot r, and the merge also adds each slot's attention mass
// l_r exp(m_r - m) / L over its (query, head) pairs into the usage counters; see the entry point.
constexpr int MERGE_USAGE_MAX_SLOTS = 32;
constexpr size_t MERGE_USAGE_HDR = 256;            // launch counter, then the per-CTA slot sums (double [gridDim.x][R])
struct MergeUsage {
    float* U;             // [R] += mass / (layers H N)
    int* A;               // [R] += 1 for every live slot (nullptr: no age tick in this launch)
    const int* live;      // live rows of the bank
    int rows;             // rows per slot
    double scale;         // 1 / (layers H N)
    unsigned* counter;
    double* partial;
};

template <bool USAGE>
__global__ void attn_merge_kernel(const float* __restrict__ Opart, const float* __restrict__ Mpart,
                                  const float* __restrict__ Lpart, float* __restrict__ O, int R, int N, int H,
                                  int dv, int ldo, const MergeUsage u) {
    pdl_sync();
    extern __shared__ float usage_red[];         // USAGE: [R][blockDim.x], thread t's mass sums in column t
    if (USAGE)
        for (int r = 0; r < R; ++r) usage_red[r * blockDim.x + threadIdx.x] = 0.f;
    // Opart [R][N][H*dv], Mpart/Lpart [R][H][N]; one thread per 4 channels (dv % 4 == 0): the weights of a (query, head) are
    // computed once per float4 instead of once per scalar (same arithmetic and order per element as the scalar form)
    const int dv4 = dv >> 2;
    const size_t total = (size_t)N * H * dv4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (i % dv4) * 4;
        const int h = (i / dv4) % H;
        const int q = i / ((size_t)dv4 * H);
        float m = -INFINITY;
        for (int r = 0; r < R; ++r) m = fmaxf(m, Mpart[((size_t)r * H + h) * N + q]);
        float4 num = make_float4(0.f, 0.f, 0.f, 0.f);
        float den = 0.f;
        for (int r = 0; r < R; ++r) {
            const float mr = Mpart[((size_t)r * H + h) * N + q];
            const float w = (mr == -INFINITY) ? 0.f : expf(mr - m);
            const float4 o = *reinterpret_cast<const float4*>(Opart + ((size_t)r * N + q) * H * dv + (size_t)h * dv + c);
            num.x += w * o.x; num.y += w * o.y; num.z += w * o.z; num.w += w * o.w;
            den += w * Lpart[((size_t)r * H + h) * N + q];
        }
        *reinterpret_cast<float4*>(O + (size_t)q * ldo + (size_t)h * dv + c) =
            make_float4(num.x / den, num.y / den, num.z / den, num.w / den);
        if (USAGE && c == 0) {                       // one thread per (query, head): the slot masses, summing to 1
            for (int r = 0; r < R; ++r) {
                const float mr = Mpart[((size_t)r * H + h) * N + q];
                const float w = (mr == -INFINITY) ? 0.f : expf(mr - m);
                usage_red[r * blockDim.x + threadIdx.x] += w * Lpart[((size_t)r * H + h) * N + q] / den;
            }
        }
    }
    if (!USAGE) return;
    // per-CTA slot sums: warp w sums slots w, w + 8, ... over the block's threads in a fixed order
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int r = warp; r < R; r += nwarps) {
        double a = 0.0;
        for (int t = lane; t < (int)blockDim.x; t += 32) a += (double)usage_red[r * blockDim.x + t];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) u.partial[(size_t)blockIdx.x * R + r] = a;
    }
    __threadfence();
    __syncthreads();
    __shared__ unsigned last;
    if (threadIdx.x == 0) last = atomicAdd(u.counter, 1u) == gridDim.x - 1 ? 1u : 0u;
    __syncthreads();
    if (!last) return;
    __threadfence();
    // last CTA: the CTA sums in CTA order, then the counters; the launch counter is left at zero for the next launch
    const volatile double* pv = u.partial;
    const int live_slots = u.A ? min(*u.live / u.rows, R) : 0;
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
        double a = 0.0;
        for (int b = 0; b < (int)gridDim.x; ++b) a += pv[(size_t)b * R + r];
        u.U[r] += (float)(a * u.scale);
        if (r < live_slots) u.A[r] += 1;
    }
    if (threadIdx.x == 0) *u.counter = 0u;
}
}  // namespace aotb

// ---------------------------------------------------------------- split-KV merge over PEER memory (cfg4 row e.2)
// Same merge, but the partials of rank r are read straight from rank r's buffer: the pointers are peer mappings of a
// symmetric-memory allocation (NVLink P2P loads), so the gather of the exchange step happens inside this kernel instead of
// in three NCCL all-gathers.  Rank r's arrays are Opart_r [S][N][H*dv], Mpart_r / Lpart_r [S][H][N]; partials are visited
// in (rank, split) order on every rank, so all ranks produce bit-identical outputs.
namespace aotb {
struct MergePeers { const float* O[8]; const float* M[8]; const float* L[8]; };

__global__ void attn_merge_peers_kernel(const MergePeers p, float* __restrict__ O, int R, int S, int N, int H, int dv,
                                        int ldo) {
    pdl_sync();
    const int dv4 = dv >> 2;                       // one thread per 4 channels, as in attn_merge_kernel
    const size_t total = (size_t)N * H * dv4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (i % dv4) * 4;
        const int h = (i / dv4) % H;
        const int q = i / ((size_t)dv4 * H);
        float m = -INFINITY;
        for (int r = 0; r < R; ++r)
            for (int s = 0; s < S; ++s) m = fmaxf(m, p.M[r][((size_t)s * H + h) * N + q]);
        float4 num = make_float4(0.f, 0.f, 0.f, 0.f);
        float den = 0.f;
        for (int r = 0; r < R; ++r)
            for (int s = 0; s < S; ++s) {
                const float mr = p.M[r][((size_t)s * H + h) * N + q];
                const float w = (mr == -INFINITY) ? 0.f : expf(mr - m);
                const float4 o = *reinterpret_cast<const float4*>(p.O[r] + ((size_t)s * N + q) * H * dv + (size_t)h * dv + c);
                num.x += w * o.x; num.y += w * o.y; num.z += w * o.z; num.w += w * o.w;
                den += w * p.L[r][((size_t)s * H + h) * N + q];
            }
        *reinterpret_cast<float4*>(O + (size_t)q * ldo + (size_t)h * dv + c) =
            make_float4(num.x / den, num.y / den, num.z / den, num.w / den);
    }
}
}  // namespace aotb

using namespace aotb;

extern "C" int aotb_attn_merge_f32(const float* Opart, const float* Mpart, const float* Lpart, float* O, int R,
                                   int N, int H, int d_v, int ldo, void* stream) {
    AOTB_REQUIRE(Opart && Mpart && Lpart && O && R > 0 && N > 0 && H > 0 && d_v > 0, "aotb_attn_merge_f32: bad args");
    AOTB_REQUIRE(d_v % 4 == 0 && ldo % 4 == 0 && ((uintptr_t)Opart | (uintptr_t)O) % 16 == 0, "aotb_attn_merge_f32: d_v, ldo %% 4, 16-byte alignment");
    const size_t total = (size_t)N * H * (d_v / 4);
    int g = (int)((total + 255) / 256);
    if (g > 132 * 8) g = 132 * 8;
    launch(attn_merge_kernel<false>, dim3(g), dim3(256), 0, (cudaStream_t)stream, Opart, Mpart, Lpart, O, R, N, H, d_v, ldo,
           MergeUsage{});
    return check_launch("aotb_attn_merge_f32");
}

extern "C" size_t aotb_attn_merge_usage_workspace_bytes(int R) {
    return MERGE_USAGE_HDR + (size_t)132 * 8 * (size_t)(R > 0 ? R : 0) * sizeof(double);
}

extern "C" int aotb_attn_merge_usage_f32(const float* Opart, const float* Mpart, const float* Lpart, float* O, int R, int N,
                                         int H, int d_v, int ldo, float* U, int* A, const int* live, int rows, int layers,
                                         void* workspace, void* stream) {
    AOTB_REQUIRE(Opart && Mpart && Lpart && O && R > 0 && N > 0 && H > 0 && d_v > 0, "aotb_attn_merge_usage_f32: bad args");
    AOTB_REQUIRE(d_v % 4 == 0 && ldo % 4 == 0 && ((uintptr_t)Opart | (uintptr_t)O) % 16 == 0,
                 "aotb_attn_merge_usage_f32: d_v, ldo %% 4, 16-byte alignment");
    AOTB_REQUIRE(R <= MERGE_USAGE_MAX_SLOTS, "aotb_attn_merge_usage_f32: at most %d slots (got %d)", MERGE_USAGE_MAX_SLOTS, R);
    AOTB_REQUIRE(U && workspace && layers > 0 && (!A || (live && rows > 0)), "aotb_attn_merge_usage_f32: usage arguments");
    AOTB_REQUIRE((uintptr_t)workspace % 16 == 0, "aotb_attn_merge_usage_f32: workspace alignment");
    const size_t total = (size_t)N * H * (d_v / 4);
    int g = (int)((total + 255) / 256);
    if (g > 132 * 8) g = 132 * 8;
    MergeUsage u;
    u.U = U; u.A = A; u.live = live; u.rows = rows;
    u.scale = 1.0 / ((double)layers * H * N);
    u.counter = (unsigned*)workspace;
    u.partial = (double*)((char*)workspace + MERGE_USAGE_HDR);
    launch(attn_merge_kernel<true>, dim3(g), dim3(256), (size_t)R * 256 * sizeof(float), (cudaStream_t)stream, Opart, Mpart,
           Lpart, O, R, N, H, d_v, ldo, u);
    return check_launch("aotb_attn_merge_usage_f32");
}

extern "C" int aotb_attn_merge_peers_f32(const void* const* Oparts, const void* const* Mparts, const void* const* Lparts,
                                         int ranks, int splits, float* O, int N, int H, int d_v, int ldo, void* stream) {
    AOTB_REQUIRE(Oparts && Mparts && Lparts && O && ranks > 0 && ranks <= 8 && splits > 0 && N > 0 && H > 0 && d_v > 0,
                 "aotb_attn_merge_peers_f32: bad args (at most 8 ranks)");
    AOTB_REQUIRE(d_v % 4 == 0 && ldo % 4 == 0, "aotb_attn_merge_peers_f32: d_v and ldo must be multiples of 4");
    MergePeers p;
    for (int r = 0; r < 8; ++r) {
        p.O[r] = r < ranks ? (const float*)Oparts[r] : nullptr;
        p.M[r] = r < ranks ? (const float*)Mparts[r] : nullptr;
        p.L[r] = r < ranks ? (const float*)Lparts[r] : nullptr;
        AOTB_REQUIRE(r >= ranks || (p.O[r] && p.M[r] && p.L[r]), "aotb_attn_merge_peers_f32: null peer pointer");
    }
    const size_t total = (size_t)N * H * (d_v / 4);
    int g = (int)((total + 255) / 256);
    if (g > 132 * 8) g = 132 * 8;
    launch(attn_merge_peers_kernel, dim3(g), dim3(256), 0, (cudaStream_t)stream, p, O, ranks, splits, N, H, d_v, ldo);
    return check_launch("aotb_attn_merge_peers_f32");
}
