// Fused softmax attention on the Hopper tensor cores (wgmma + TMA + mbarrier) over split-fp16 ("fp16x2") operands: every
// fp32 value x is carried as hi = fp16(x), lo = fp16(x - hi) in 128-byte rows [hi(32) | lo(32)] (one TMA swizzle atom).
// Shared by the AOT long-term attention (lt_attn_tc.cu: H heads x d = 32) and the DeAOT one (gp_attn_tc.cu: 1 head,
// d_qk = 128, d_v = 1024), which differ only in how many 32-channel chunks make up a query / key row (QC) and how many value
// chunks one CTA accumulates (VC).
//
// One CTA = 64 NWG queries x VC value chunks x one KV split, 32 (4 NWG + 1) threads:
//   warps 0 .. 4 NWG - 1  NWG consumer warpgroups, 64 query rows each.  Per BK-key tile:
//                S = Q K^T        (wgmma m64nBKk16, Q and K from shared memory; registers hold the 64 x BK fp32 tile)
//                online softmax   (row max over the 4 lanes that share a row, p = 2^(s log2e - m log2e), fp32 row sums)
//                O' += P [Vh|Vl]  (wgmma with P from registers -- the S fragment re-packed as fp16 -- and V MN-major)
//              exact mode: S = Qh Kh + Ql Kh + Qh Kl, O' = (Ph + Pl) [Vh | Vl]; fast mode: S = Qh Kh, O' = Ph [Vh | Vl].
//              O = O'[:, :32] + O'[:, 32:] per value chunk; fp32 accumulation everywhere.
//   warp 4 NWG  TMA producer: the Q tile once, then a ring of K / V stages.
// The warpgroups run independently (each waits for the stage, each releases it), so one warpgroup's softmax overlaps the
// other's MMAs.  Layouts of the AOT kernel (all compute the same maxima and, to fp32 rounding, the same P):
//   tile    NWG = 2, BK = 64                       (default; two co-resident per SM at <= 96 registers)
//   groups  NWG = 2, BK = 128: half the tile iterations, twice the scores in registers per thread
//   ahead   NWG = 2, BK = 64, S of tile n + 1 issued before the softmax of tile n, so the tensor cores compute the next
//           scores while this warpgroup runs ex2 (a second score buffer in registers)
//   pair    NWG = 1, BK = 64: 64-query CTAs, two co-resident per SM
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace aotb {
namespace tc {

constexpr float AT_LOG2E = 1.4426950408889634f;

struct AttnTcArgs {
    int N, Tk;
    const int* Tk_dev;
    float* O;
    int ldo;
    float* Opart;     // [splits][N][gridDim.y * VC * 32]
    float* Mpart;     // [splits][QC == 1 ? H : 1][N]
    float* Lpart;
    int splits;
    int split_unit;   // KV splits are cut on multiples of this many keys
    int spin;         // 1: mbarrier waits poll without the suspend hint
    float* dbg;       // optional (QC == 1): CTA (0,0,0) dumps S of keys [0, 128) [128][128], then O'_0 [128][64]
};

template <int QC, int VC, int STAGES, int BK, int NWG>
struct AttnSmem {
    static constexpr int BM = 64 * NWG;
    static constexpr int Q_BYTES = QC * BM * 128;
    static constexpr int K_BYTES = QC * BK * 128;
    static constexpr int V_BYTES = VC * BK * 128;
    static constexpr int STAGE_BYTES = K_BYTES + V_BYTES;
    static constexpr int TOTAL = Q_BYTES + STAGES * STAGE_BYTES + (1 + 2 * STAGES) * 8 + 1024;
};

template <int N>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    if (N == 128) wgmma_ss_n128(d, a, b, scale_d);
    else wgmma_ss_n64(d, a, b, scale_d);
}

// CTAs per SM the register allocation is bounded for.  The tile layout (QC = 1, 64-key tiles, two warpgroups, no second score
// buffer) fits 96 registers without spilling, so two 9-warp CTAs share an SM and one CTA's MMAs run under the other's
// softmax; groups, ahead and the DeAOT head shape (QC = 4) spill at that bound and keep one.  pair (5-warp CTAs) takes two.
template <int QC, int BK, int NWG, bool AHEAD>
constexpr int attn_tc_min_blocks() { return NWG == 1 || (QC == 1 && BK == 64 && !AHEAD) ? 2 : 1; }

// grid (query tiles of 64 NWG, QC == 1 ? heads : value slices of VC chunks, splits).  Head / slice y reads query and key chunks
// [y, y + 1) when QC == 1, else [0, QC), and value chunks [y * VC, (y + 1) * VC).
// The body of one CTA.  A launch over n independent problems (attn_tc_batched_kernel) hands CTA (qt, y, z) of problem b:
// its query rows start at row b q_stride of Q, its keys at row b kv_stride of K / V, its live key count is Tk_dev[b], and its
// output rows are [b N, (b + 1) N) of O and of the partials (laid out over n N rows).  The one-problem kernel is b = 0, n = 1.
template <int QC, int VC, int STAGES, bool EXACT, int BK, int NWG, bool AHEAD>
__device__ __forceinline__ void attn_tc_cta(const CUtensorMap* tmQp, const CUtensorMap* tmKp, const CUtensorMap* tmVp,
                                            const AttnTcArgs& a, const int qt, const int b, const int q_stride,
                                            const int kv_stride, const int nprob) {
    const CUtensorMap& tmQ = *tmQp;
    const CUtensorMap& tmK = *tmKp;
    const CUtensorMap& tmV = *tmVp;
    using SM = AttnSmem<QC, VC, STAGES, BK, NWG>;
    constexpr int BM = SM::BM, TMA_WARP = 4 * NWG, SR = BK / 2;     // SR: score registers per thread
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sQ = smem;
    uint8_t* sKV = smem + SM::Q_BYTES;
    uint64_t* q_full = reinterpret_cast<uint64_t*>(sKV + STAGES * SM::STAGE_BYTES);
    uint64_t* kv_full = q_full + 1;
    uint64_t* kv_free = kv_full + STAGES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int y = blockIdx.y, z = blockIdx.z;
    const int qc0 = QC == 1 ? y : 0, vc0 = y * VC;
    pdl_trigger();
    if (tid == 0) {
        mbar_init(q_full, 1);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_free[s], 4 * NWG); }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();       // the packed operands and the live key count were written by earlier kernels

    const int tk = a.Tk_dev ? a.Tk_dev[b] : a.Tk;
    const int units = (tk + a.split_unit - 1) / a.split_unit;
    const int per = (units + a.splits - 1) / a.splits;
    const int k0 = min(z * per * a.split_unit, tk), k1 = min((z + 1) * per * a.split_unit, tk);
    const int ntiles = (k1 - k0 + BK - 1) / BK;

    if (warp == TMA_WARP) {
        // A CTA with an empty KV split loads nothing: its consumers never wait on q_full, and no bulk copy may still be
        // writing into this CTA's shared memory after it exits.
        if (elect_one() && ntiles > 0) {
            tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
            mbar_arrive_expect_tx(q_full, SM::Q_BYTES);
            for (int c = 0; c < QC; ++c) tma_load_3d(sQ + c * BM * 128, &tmQ, q_full, 0, b * q_stride + qt * BM, qc0 + c);
            for (int n = 0; n < ntiles; ++n) {
                const int s = n % STAGES;
                if (n >= STAGES) mbar_wait(&kv_free[s], ((n / STAGES) - 1) & 1);
                uint8_t* st = sKV + s * SM::STAGE_BYTES;
                mbar_arrive_expect_tx(&kv_full[s], SM::STAGE_BYTES);
                const int key0 = b * kv_stride + k0 + n * BK;
                for (int c = 0; c < QC; ++c) tma_load_3d(st + c * BK * 128, &tmK, &kv_full[s], 0, key0, qc0 + c);
                for (int v = 0; v < VC; ++v)
                    tma_load_3d(st + SM::K_BYTES + v * BK * 128, &tmV, &kv_full[s], 0, key0, vc0 + v);
            }
        }
        return;
    }

    // ======================= consumer warpgroups =======================
    const int wg = warp >> 2, wq = warp & 3;
    const int row0 = wg * 64 + wq * 16 + (lane >> 2);          // this thread's rows: row0, row0 + 8 (within the CTA tile)
    const int cq = (lane & 3) * 2;                             // column offset inside each 8-column group
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[VC][32];
#pragma unroll
    for (int v = 0; v < VC; ++v)
#pragma unroll
        for (int j = 0; j < 32; ++j) o[v][j] = 0.f;
    const bool dump = a.dbg && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0;
    const uint64_t dQ = smem_desc_sw128(smem_u32(sQ + wg * 64 * 128));
    const uint64_t dKV0 = smem_desc_sw128(smem_u32(sKV));
    if (ntiles > 0) mbar_wait_cp(q_full, 0, a.spin);

    // S(n) into `sc`: every stage of tile n has landed (the caller waited for kv_full)
    auto issue_s = [&](int n, float* sc) {
        const uint64_t dK = dKV0 + (uint64_t)(((n % STAGES) * SM::STAGE_BYTES) >> 4);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < QC; ++c) {
            const uint64_t q = dQ + (uint64_t)((c * BM * 128) >> 4), k = dK + (uint64_t)((c * BK * 128) >> 4);
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {            // +2 = 32 B = 16 halfs of K; hi at +0, lo at +4 (64 B)
                wgmma_ss<BK>(sc, q + 2 * ks, k + 2 * ks, (c | ks) ? 1u : 0u);
                if (EXACT) {
                    wgmma_ss<BK>(sc, q + 4 + 2 * ks, k + 2 * ks, 1u);
                    wgmma_ss<BK>(sc, q + 2 * ks, k + 4 + 2 * ks, 1u);
                }
            }
        }
        wgmma_commit();
    };
    float sbuf[AHEAD ? 2 : 1][SR];
    if (AHEAD && ntiles > 0) {
        mbar_wait_cp(&kv_full[0], 0, a.spin);
        issue_s(0, sbuf[0]);
    }

#pragma unroll 1
    for (int n = 0; n < ntiles; ++n) {
        const int s = n % STAGES;
        float* sc = sbuf[0];
        if (AHEAD) {
            if (n + 1 < ntiles) {                       // the next scores run on the tensor cores under this softmax
                mbar_wait_cp(&kv_full[(n + 1) % STAGES], ((n + 1) / STAGES) & 1, a.spin);
                issue_s(n + 1, sbuf[AHEAD ? 1 : 0]);
                wgmma_wait<1>();
            } else {
                wgmma_wait<0>();
            }
        } else {
            mbar_wait_cp(&kv_full[s], (n / STAGES) & 1, a.spin);
            issue_s(n, sc);
            wgmma_wait<0>();
        }
        reg_fence<SR>(sc);
        const uint64_t dV = dKV0 + (uint64_t)((s * SM::STAGE_BYTES + SM::K_BYTES) >> 4);
        const int key0 = k0 + n * BK;
        if (dump && key0 < 128) {
#pragma unroll
            for (int j = 0; j < SR; ++j) {
                const int key = key0 + 8 * (j >> 2) + cq + (j & 1);
                if (key < 128) a.dbg[(row0 + 8 * ((j >> 1) & 1)) * 128 + key] = sc[j];
            }
        }
        // keys of the tile beyond this split's range (or the live count) do not exist
        if (key0 + BK > k1) {
#pragma unroll
            for (int j = 0; j < SR; ++j)
                if (key0 + 8 * (j >> 2) + cq + (j & 1) >= k1) sc[j] = -INFINITY;
        }
        float mx[2] = {m[0], m[1]};
#pragma unroll
        for (int j = 0; j < SR; ++j) mx[(j >> 1) & 1] = fmaxf(mx[(j >> 1) & 1], sc[j]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        }
        float f[2], neg[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            f[h] = mx[h] > m[h] ? ex2((m[h] - mx[h]) * AT_LOG2E) : 1.f;
            m[h] = mx[h];
            l[h] *= f[h];
            neg[h] = m[h] * AT_LOG2E;
        }
#pragma unroll
        for (int v = 0; v < VC; ++v)
#pragma unroll
            for (int j = 0; j < 32; ++j) o[v][j] *= f[(j >> 1) & 1];
        uint32_t ph[SR / 2], pl[SR / 2];
#pragma unroll
        for (int j = 0; j < SR; j += 2) {
            const int h = (j >> 1) & 1;
            const float p0 = ex2(fmaf(sc[j], AT_LOG2E, -neg[h])), p1 = ex2(fmaf(sc[j + 1], AT_LOG2E, -neg[h]));
            l[h] += p0 + p1;
            const __half2 hi = __floats2half2_rn(p0, p1);
            ph[j >> 1] = *reinterpret_cast<const uint32_t*>(&hi);
            if (EXACT) pl[j >> 1] = cvt_h2(p0 - __low2float(hi), p1 - __high2float(hi));
        }
        wgmma_fence();
#pragma unroll
        for (int v = 0; v < VC; ++v) {
            const uint64_t vd = dV + (uint64_t)((v * BK * 128) >> 4);
#pragma unroll
            for (int kk = 0; kk < BK / 16; ++kk) {      // 16 keys = 16 rows of 128 B = 2048 B per k-step
                wgmma_rs_n64_tb(o[v], ph + 4 * kk, vd + (uint64_t)(kk * 128));
                if (EXACT) wgmma_rs_n64_tb(o[v], pl + 4 * kk, vd + (uint64_t)(kk * 128));
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int v = 0; v < VC; ++v) reg_fence<32>(o[v]);
        mbar_arrive_warp(&kv_free[s]);
        if (AHEAD) {                                    // S(n + 1) has completed (wait above): it becomes the current tile
            reg_fence<SR>(sbuf[AHEAD ? 1 : 0]);
#pragma unroll
            for (int j = 0; j < SR; ++j) sbuf[0][j] = sbuf[AHEAD ? 1 : 0][j];
        }
    }

    // ======================= epilogue =======================
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    }
    if (dump) {
#pragma unroll
        for (int j = 0; j < 32; ++j) a.dbg[128 * 128 + (row0 + 8 * ((j >> 1) & 1)) * 64 + 8 * (j >> 2) + cq + (j & 1)] = o[0][j];
    }
    const int cols = gridDim.y * VC * 32;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int ql = qt * BM + row0 + 8 * h;
        if (ql >= a.N) continue;
        const int q = b * a.N + ql;
        const float inv = 1.f / l[h];
#pragma unroll
        for (int v = 0; v < VC; ++v) {
#pragma unroll
            for (int g = 0; g < 4; ++g) {       // columns 8 g + cq, +1 of value chunk vc0 + v: j = 4 g + 2 h, + 1 (and + 16 for lo)
                const int j = 4 * g + 2 * h;
                float2 r = make_float2(o[v][j] + o[v][j + 16], o[v][j + 1] + o[v][j + 17]);
                const int col = (vc0 + v) * 32 + 8 * g + cq;
                if (a.splits == 1) {
                    r.x *= inv; r.y *= inv;
                    *reinterpret_cast<float2*>(a.O + (size_t)q * a.ldo + col) = r;
                } else {
                    *reinterpret_cast<float2*>(a.Opart + ((size_t)z * nprob * a.N + q) * cols + col) = r;
                }
            }
        }
        if (a.splits > 1 && (lane & 3) == 0 && (QC == 1 || y == 0)) {
            const size_t idx = ((size_t)z * (QC == 1 ? gridDim.y : 1) + (QC == 1 ? y : 0)) * nprob * a.N + q;
            a.Mpart[idx] = m[h];
            a.Lpart[idx] = l[h];
        }
    }
}

template <int QC, int VC, int STAGES, bool EXACT, int BK, int NWG, bool AHEAD>
__global__ void __launch_bounds__(32 * (4 * NWG + 1), (attn_tc_min_blocks<QC, BK, NWG, AHEAD>()))
attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const AttnTcArgs a) {
    attn_tc_cta<QC, VC, STAGES, EXACT, BK, NWG, AHEAD>(&tmQ, &tmK, &tmV, a, blockIdx.x, 0, 0, 0, 1);
}

// n independent problems in one launch: grid (n x query tiles of one problem, heads / value slices, splits).
struct AttnTcBatch {
    int n, qtiles, q_stride, kv_stride;
};

template <int QC, int VC, int STAGES, bool EXACT, int BK, int NWG, bool AHEAD>
__global__ void __launch_bounds__(32 * (4 * NWG + 1), (attn_tc_min_blocks<QC, BK, NWG, AHEAD>()))
attn_tc_batched_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, const AttnTcArgs a, const AttnTcBatch bt) {
    const int b = blockIdx.x / bt.qtiles;
    attn_tc_cta<QC, VC, STAGES, EXACT, BK, NWG, AHEAD>(&tmQ, &tmK, &tmV, a, blockIdx.x - b * bt.qtiles, b, bt.q_stride,
                                                       bt.kv_stride, bt.n);
}

// Shared-memory size and carveout of both modes' kernels, set once per process before the first launch or query.
template <int QC, int VC, int STAGES, int BK, int NWG, bool AHEAD>
int configure_attn_tc(const char* what) {
    constexpr int smem = AttnSmem<QC, VC, STAGES, BK, NWG>::TOTAL;
    auto kt = attn_tc_kernel<QC, VC, STAGES, true, BK, NWG, AHEAD>;
    auto kf = attn_tc_kernel<QC, VC, STAGES, false, BK, NWG, AHEAD>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(kt, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (attn_tc_min_blocks<QC, BK, NWG, AHEAD>() == 2) {
            // the carveout is a hint: without it the driver may keep enough L1 that only one CTA's shared memory fits
            if (e == cudaSuccess)
                e = cudaFuncSetAttribute(kt, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            if (e == cudaSuccess)
                e = cudaFuncSetAttribute(kf, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        }
        if (e != cudaSuccess) {
            set_error("%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    return AOTB_OK;
}

template <int QC, int VC, int STAGES, int BK, int NWG, bool AHEAD>
int launch_attn_tc(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnTcArgs& a, dim3 grid,
                   int exact, cudaStream_t st, const char* what) {
    const int rc = configure_attn_tc<QC, VC, STAGES, BK, NWG, AHEAD>(what);
    if (rc != AOTB_OK) return rc;
    auto kt = attn_tc_kernel<QC, VC, STAGES, true, BK, NWG, AHEAD>;
    auto kf = attn_tc_kernel<QC, VC, STAGES, false, BK, NWG, AHEAD>;
    launch(exact ? kt : kf, grid, dim3(32 * (4 * NWG + 1)), AttnSmem<QC, VC, STAGES, BK, NWG>::TOTAL, st, tq, tk, tv, a);
    return check_launch(what);
}

template <int QC, int VC, int STAGES, int BK, int NWG, bool AHEAD>
int launch_attn_tc_batched(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnTcArgs& a,
                           const AttnTcBatch& bt, dim3 grid, int exact, cudaStream_t st, const char* what) {
    constexpr int smem = AttnSmem<QC, VC, STAGES, BK, NWG>::TOTAL;
    auto kt = attn_tc_batched_kernel<QC, VC, STAGES, true, BK, NWG, AHEAD>;
    auto kf = attn_tc_batched_kernel<QC, VC, STAGES, false, BK, NWG, AHEAD>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(kt, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (attn_tc_min_blocks<QC, BK, NWG, AHEAD>() == 2) {
            if (e == cudaSuccess)
                e = cudaFuncSetAttribute(kt, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            if (e == cudaSuccess)
                e = cudaFuncSetAttribute(kf, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        }
        if (e != cudaSuccess) {
            set_error("%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    launch(exact ? kt : kf, grid, dim3(32 * (4 * NWG + 1)), smem, st, tq, tk, tv, a, bt);
    return check_launch(what);
}

// Resident CTAs per SM of one mode's kernel as launch_attn_tc configures it, with its registers per thread and local-memory
// (spill) bytes per thread.
template <int QC, int VC, int STAGES, int BK, int NWG, bool AHEAD>
int attn_tc_occupancy(int exact, int* ctas_per_sm, int* regs, int* local_bytes, const char* what) {
    const int rc = configure_attn_tc<QC, VC, STAGES, BK, NWG, AHEAD>(what);
    if (rc != AOTB_OK) return rc;
    const void* k = exact ? (const void*)attn_tc_kernel<QC, VC, STAGES, true, BK, NWG, AHEAD>
                          : (const void*)attn_tc_kernel<QC, VC, STAGES, false, BK, NWG, AHEAD>;
    cudaFuncAttributes fa;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, k, 32 * (4 * NWG + 1),
                                                                  AttnSmem<QC, VC, STAGES, BK, NWG>::TOTAL);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k);
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return AOTB_ERR_CUDA;
    }
    *regs = fa.numRegs;
    *local_bytes = (int)fa.localSizeBytes;
    return AOTB_OK;
}

}  // namespace tc
}  // namespace aotb
