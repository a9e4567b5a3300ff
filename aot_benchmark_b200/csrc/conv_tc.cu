// Implicit-GEMM convolution / linear layer on the Hopper tensor cores (wgmma + TMA + mbarrier), NHWC fp32 in / fp32 out,
// through the split-fp16 ("fp16x2") scheme of lt_attn_tc.cu.
//
//   out[m][n] = act( wscale[n] * sum_k A(m,k) * W'[k][n] + bias[n] + res[m][n] )      m -> (b, oy, ox), k -> (ky, kx, ci)
//
// The weights arrive normalised per output channel (ops.split_fp16_scaled): column n holds w * 2^e_n and the finish
// multiplies the accumulator by wscale[n] = 2^-e_n, an exact operation, so the split keeps its relative precision for
// channels of any magnitude.
//
// Same reference sites as conv_igemm.cu (resnet.py:34-54,140-157 with FrozenBatchNorm2d folded,
// aot.py:19-21,83, fpn.py:34-58, every nn.Linear of transformer.py:321-367,582-665).  Eligibility:
// Cin % 4 == 0, Cout % 64 == 0, dilation 1 (everything on the R50-AOTL path except the 11-channel conv_out;
// the 7x7 stem runs on a 4-channel zero-padded copy of the image).
//
// One CTA = 128 output pixels x BN (64 | 128 | 256) output channels, 384 threads in three warpgroups, warp-specialised:
//   warps 0-7   two consumer warpgroups (64 pixel rows each).  Per K chunk they wait for the stage's "A full" and "B full"
//               barriers, issue 4 k-steps x (Ah Wh + Al Wh + Ah Wl) as wgmma m64nBNk16 and release the stage of the
//               previous chunk on "empty" once its MMAs have completed.  Afterwards the accumulators go through a fp32
//               staging tile in shared memory and the same warps run the finish (bias / residual / activation -> fp32 NHWC).
//   warps 8-11  producer warpgroup.  It gathers the fp32 activations of all 128 rows of a chunk straight from NHWC global
//               memory (im2col is never materialised), splits them into hi = fp16(x), lo = fp16(x - hi), stores both
//               128 x 64 half tiles 128B-swizzled and K-major, and arrives on "A full" after fence.proxy.async.  Thread 256
//               streams the pre-split weights (Wh, Wl as [Cout][K] fp16, K-major) into the same stage by TMA.
// The loads go through registers, not cp.async: the split needs the values in registers anyway, and an fp32 staging area
// (32 KB per chunk in flight) does not fit beside two BN = 256 stages.  The producer keeps two half-chunks (one chunk, 32 KB
// per CTA) of loads in flight while it splits and stores the third, which is 96 registers per thread.
// The N tile sets how often the activations are gathered: a layer with Cout = 256 reads its input once at BN = 256 and four
// times at BN = 64.  STAGES: 4 at BN = 64, 3 at 128, 2 at 256 (a stage is 32 KB of A plus BN * 256 bytes of B).
//
// Single-pass mode (SPLIT = false, selected by wl == NULL): the producer stores hi = fp16(x) only, the TMA thread streams Wh
// only and the consumers issue Ah Wh once per k-step.  Products are then fp16 x fp16 with fp32 accumulation: each operand
// carries 2^-11 relative rounding (the weights keep their per-channel normalisation, so any scale gets it).  A stage is
// 16 KB of A plus BN * 128 bytes of B, so the same budget holds twice the chunks: STAGES 8 at BN = 64, 6 at 128, 4 at 256.
#include <type_traits>

#include "common.cuh"
#include "tc_common.cuh"

namespace aotb {
namespace tc {

constexpr int CONV_A_BYTES = 128 * 128;        // one 128 x 64 half tile (both consumer warpgroups' rows)

template <int BN>
__device__ __forceinline__ void wgmma_conv(float* acc, uint64_t a, uint64_t b) {
    if (BN == 256) wgmma_ss_n256(acc, a, b, 1u);
    else if (BN == 128) wgmma_ss_n128(acc, a, b, 1u);
    else wgmma_ss_n64(acc, a, b, 1u);
}

// Accumulator fragment -> row-major fp32 staging tile [128][ld] (row = pixel of the tile, column = channel of the tile).
template <int BN>
__device__ __forceinline__ void conv_acc_to_staging(const float* acc, float* stg, int ld) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row0 = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2), cq = (lane & 3) * 2;
#pragma unroll
    for (int j = 0; j < BN / 2; j += 2)
        *reinterpret_cast<float2*>(stg + (row0 + 8 * ((j >> 1) & 1)) * ld + 8 * (j >> 2) + cq) = make_float2(acc[j], acc[j + 1]);
}

struct ConvTcArgs {
    const float* in;
    const float* bias;
    const float* wscale;   // per output channel, null = 1
    const float* res;
    float* out;
    int B, H, W, Cin, ldin;
    int Ho, Wo, Cout, ldout, ldres;
    int KH, KW, stride, pad;
    int M, nchunks;
    int act;
    int splits;          // split-K: the `splits` CTAs (blockIdx.z) of one output tile form a thread-block cluster; CTA z
                         // handles chunks [z*per, (z+1)*per) and the partial tiles are summed over distributed smem
    int spin;            // 1: mbarrier waits without the suspend hint
    long long* prof;     // diagnostic: 12 clock64 stamps per CTA (see aotb_set_conv_tiling), or null
};

static int g_conv_tiling = 0;      // aotb_set_conv_tiling

struct RowInfo { int pix_base, iy0, ix0, valid; };

// Finish of one output tile by the 256 epilogue threads.  The staging tile is [128][BN + 4] fp32; with split-K the S
// CTAs of the cluster each own 128 / S rows and sum that slice of every peer's staging buffer in rank order.  A thread
// keeps one 4-channel column (its bias is loaded once) and walks rows; NB rows are processed per batch with every load
// of the batch (S remote tiles + residual) issued before the first use -- a load-use-load chain costs one DSMEM / L2
// round trip per row and was 6 us per tile.
template <int BN, int S, int NB>
__device__ __forceinline__ void conv_finish_tile(const ConvTcArgs& a, const uint8_t* smem, int tid, int m0, int n0, int zrank) {
    constexpr int LD = BN + 4, C4 = BN / 4, RSTEP = 256 / C4, ROWS = 128 / S, ITERS = ROWS / RSTEP;
    constexpr int B = NB < ITERS ? NB : ITERS;
    static_assert(ITERS >= 1 && ITERS % B == 0, "finish tiling");
    const int c = (tid % C4) * 4, n = n0 + c;
    const int r0 = zrank * ROWS + tid / C4;
    const float4 b4 = a.bias ? __ldg(reinterpret_cast<const float4*>(a.bias + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 s4 = a.wscale ? __ldg(reinterpret_cast<const float4*>(a.wscale + n)) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float* lbase = reinterpret_cast<const float*>(smem) + r0 * LD + c;
    const uint32_t sbase = smem_u32(lbase);
#pragma unroll 1
    for (int i0 = 0; i0 < ITERS; i0 += B) {
        float4 v[B][S], rs[B];
#pragma unroll
        for (int b = 0; b < B; ++b) {
            const int ro = (i0 + b) * RSTEP;
            if (S == 1) {
                v[b][0] = *reinterpret_cast<const float4*>(lbase + ro * LD);
            } else {
#pragma unroll
                for (int z = 0; z < S; ++z) v[b][z] = dsmem_ld_f4(dsmem_addr(sbase + (uint32_t)(ro * LD) * 4u, (uint32_t)z));
            }
            const int m = m0 + r0 + ro;
            rs[b] = (a.res && m < a.M) ? *reinterpret_cast<const float4*>(a.res + (size_t)m * a.ldres + n)
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int b = 0; b < B; ++b) {
            float4 o = v[b][0];
#pragma unroll
            for (int z = 1; z < S; ++z) { o.x += v[b][z].x; o.y += v[b][z].y; o.z += v[b][z].z; o.w += v[b][z].w; }
            // o * s is exact (s is a power of two), so the fma rounds like o * s + b
            o.x = fmaf(o.x, s4.x, b4.x); o.y = fmaf(o.y, s4.y, b4.y); o.z = fmaf(o.z, s4.z, b4.z); o.w = fmaf(o.w, s4.w, b4.w);
            o.x += rs[b].x; o.y += rs[b].y; o.z += rs[b].z; o.w += rs[b].w;
            o.x = apply_act(o.x, a.act); o.y = apply_act(o.y, a.act);
            o.z = apply_act(o.z, a.act); o.w = apply_act(o.w, a.act);
            const int m = m0 + r0 + (i0 + b) * RSTEP;
            if (m < a.M) *reinterpret_cast<float4*>(a.out + (size_t)m * a.ldout + n) = o;
        }
    }
}

// Finish without split-K with the global loads taken off its critical path: the bias and the residual rows of the FIRST batch are
// already in registers (`pre`, loaded by finish_prefetch before the thread waited for the accumulator, i.e. under the tail of the
// K loop), and inside the loop the residual rows of batch k+1 are requested before batch k is computed and stored.  The staging
// tile is read with ld.shared so that the compiler does not have to order those reads behind the global stores.
// Rows per batch: 4 at BN = 256, where the prefetched rows sit beside 128 accumulator registers.
template <int BN>
struct FinishPre { static constexpr int B = BN == 256 ? 4 : 8; float4 b4, s4; float4 rs[B]; };

template <int BN>
__device__ __forceinline__ void finish_prefetch(const ConvTcArgs& a, int tid, int m0, int n0, FinishPre<BN>& pre) {
    constexpr int C4 = BN / 4, RSTEP = 256 / C4;
    const int n = n0 + (tid % C4) * 4, r0 = tid / C4;
    pre.b4 = a.bias ? __ldg(reinterpret_cast<const float4*>(a.bias + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
    pre.s4 = a.wscale ? __ldg(reinterpret_cast<const float4*>(a.wscale + n)) : make_float4(1.f, 1.f, 1.f, 1.f);
#pragma unroll
    for (int b = 0; b < FinishPre<BN>::B; ++b) {
        const int m = m0 + r0 + b * RSTEP;
        pre.rs[b] = (a.res && m < a.M) ? *reinterpret_cast<const float4*>(a.res + (size_t)m * a.ldres + n)
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

template <int BN>
__device__ __forceinline__ void conv_finish_tile_pre(const ConvTcArgs& a, const uint8_t* smem, int tid, int m0, int n0,
                                                     const FinishPre<BN>& pre) {
    constexpr int LD = BN + 4, C4 = BN / 4, RSTEP = 256 / C4, ITERS = 128 / RSTEP, B = FinishPre<BN>::B;
    static_assert(ITERS % B == 0, "finish tiling");
    const int c = (tid % C4) * 4, n = n0 + c, r0 = tid / C4;
    const uint32_t sbase = smem_u32(reinterpret_cast<const float*>(smem) + r0 * LD + c);
    float4 rs[B];
#pragma unroll
    for (int b = 0; b < B; ++b) rs[b] = pre.rs[b];
#pragma unroll 1
    for (int i0 = 0; i0 < ITERS; i0 += B) {
        float4 v[B], nx[B];
#pragma unroll
        for (int b = 0; b < B; ++b)
            asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[b].x), "=f"(v[b].y), "=f"(v[b].z), "=f"(v[b].w)
                         : "r"(sbase + (uint32_t)((i0 + b) * RSTEP * LD) * 4u));
        if (i0 + B < ITERS) {                      // residual rows of the next batch, in flight while this one is stored
#pragma unroll
            for (int b = 0; b < B; ++b) {
                const int m = m0 + r0 + (i0 + B + b) * RSTEP;
                nx[b] = (a.res && m < a.M) ? *reinterpret_cast<const float4*>(a.res + (size_t)m * a.ldres + n)
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
#pragma unroll
        for (int b = 0; b < B; ++b) {
            float4 o = v[b];
            o.x = fmaf(o.x, pre.s4.x, pre.b4.x); o.y = fmaf(o.y, pre.s4.y, pre.b4.y);
            o.z = fmaf(o.z, pre.s4.z, pre.b4.z); o.w = fmaf(o.w, pre.s4.w, pre.b4.w);
            o.x += rs[b].x; o.y += rs[b].y; o.z += rs[b].z; o.w += rs[b].w;
            o.x = apply_act(o.x, a.act); o.y = apply_act(o.y, a.act);
            o.z = apply_act(o.z, a.act); o.w = apply_act(o.w, a.act);
            const int m = m0 + r0 + (i0 + b) * RSTEP;
            if (m < a.M) *reinterpret_cast<float4*>(a.out + (size_t)m * a.ldout + n) = o;
        }
        if (i0 + B < ITERS) {
#pragma unroll
            for (int b = 0; b < B; ++b) rs[b] = nx[b];
        }
    }
}

template <int BN, int STAGES, bool SPLIT>
struct ConvSmem {
    static constexpr int A_BYTES = CONV_A_BYTES;
    static constexpr int B_BYTES = BN * 128;
    static constexpr int PARTS = SPLIT ? 2 : 1;        // hi and lo tiles, or hi only
    static constexpr int STAGE_BYTES = PARTS * A_BYTES + PARTS * B_BYTES;
    static constexpr int STG_LD = BN + 4;              // staging tile [128][BN + 4] fp32, aliases the stages
    static_assert(128 * STG_LD * 4 <= STAGES * STAGE_BYTES, "staging tile must fit in the operand stages");
    static constexpr int TOTAL = STAGES * STAGE_BYTES + 128 * (int)sizeof(RowInfo) + 3 * STAGES * 8 + 1024;
    static_assert(TOTAL <= 227 * 1024, "shared memory of one CTA");
};

template <int BN, int STAGES, bool SPLIT>
__global__ void __launch_bounds__(384, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const ConvTcArgs a) {
    using SM = ConvSmem<BN, STAGES, SPLIT>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    RowInfo* rinfo = reinterpret_cast<RowInfo*>(smem + STAGES * SM::STAGE_BYTES);
    uint64_t* a_full = reinterpret_cast<uint64_t*>(rinfo + 128);    // 128 producer-thread arrivals
    uint64_t* b_full = a_full + STAGES;                               // TMA transaction bytes
    uint64_t* s_free = b_full + STAGES;                               // 8 consumer-warp arrivals

    const int tid = threadIdx.x, warp = tid >> 5;
    const int m0 = blockIdx.x * 128, n0 = blockIdx.y * BN;
    long long* prof = a.prof ? a.prof + 12 * ((size_t)(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) : nullptr;
    auto stamp = [&](int slot) { if (prof) prof[slot] = clock64(); };
    if (tid == 0) stamp(0);
    pdl_trigger();      // the next kernel may start its prologue; it waits for this grid before reading our output

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&a_full[s], 128); mbar_init(&b_full[s], 1); mbar_init(&s_free[s], 8); }
        fence_mbar_init();
    }
    if (tid < 128) {
        const int m = m0 + tid;
        RowInfo ri;
        if (m < a.M) {
            const int HoWo = a.Ho * a.Wo;
            const int b = m / HoWo, r = m - b * HoWo;
            const int oy = r / a.Wo, ox = r - oy * a.Wo;
            ri.pix_base = b * a.H * a.W;
            ri.iy0 = oy * a.stride - a.pad;
            ri.ix0 = ox * a.stride - a.pad;
            ri.valid = 1;
        } else {
            ri.pix_base = 0; ri.iy0 = 0; ri.ix0 = 0; ri.valid = 0;
        }
        rinfo[tid] = ri;
    }
    __syncthreads();
    if (tid == 0) stamp(1);
    pdl_wait();         // activations / residual below were written by earlier kernels
    const int cpt = (a.Cin % 64 == 0) ? (a.Cin >> 6) : 0;  // 64-wide chunks per filter tap (0: general Cin % 4 path)
    const int per = (a.nchunks + a.splits - 1) / a.splits;
    const int kbeg = blockIdx.z * per;
    const int nloc = max(0, min(per, a.nchunks - kbeg));     // chunks of this CTA (local index it <-> chunk kbeg + it)

    FinishPre<BN> pre;
    // warpgroup index made warp-uniform for the compiler: wgmma in a branch it cannot prove uniform is serialised
    const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
    if (wg < 2) {
        // ======================= consumers: wgmma only =======================
        const uint64_t dA0 = smem_desc_sw128(smem_u32(smem + wg * 64 * 128));
        const uint64_t dB0 = smem_desc_sw128(smem_u32(smem + SM::PARTS * SM::A_BYTES));
        float acc[BN / 2];
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
#pragma unroll 1
        for (int it = 0; it < nloc; ++it) {
            const int s = it % STAGES;
            const uint32_t ph = (it / STAGES) & 1;
            mbar_wait_cp(&a_full[s], ph, a.spin);
            mbar_wait_cp(&b_full[s], ph, a.spin);
            if (it == 0 && tid == 0) stamp(3);
            const uint64_t so = (uint64_t)((s * SM::STAGE_BYTES) >> 4);
            const uint64_t ah = dA0 + so, al = ah + (SM::A_BYTES >> 4), bh = dB0 + so, bl = bh + (uint64_t)(SM::B_BYTES >> 4);
            reg_fence<BN / 2>(acc);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                wgmma_conv<BN>(acc, ah + 2 * ks, bh + 2 * ks);
                if constexpr (SPLIT) {
                    wgmma_conv<BN>(acc, al + 2 * ks, bh + 2 * ks);
                    wgmma_conv<BN>(acc, ah + 2 * ks, bl + 2 * ks);
                }
            }
            wgmma_commit();
            reg_fence<BN / 2>(acc);
            wgmma_wait<1>();                              // the MMAs of the previous chunk have completed: release its stage
            if (it > 0) mbar_arrive_warp(&s_free[(it - 1) % STAGES]);
        }
        wgmma_wait<0>();
        reg_fence<BN / 2>(acc);
        if (tid == 0) stamp(4);
        if (a.splits == 1) finish_prefetch<BN>(a, tid, m0, n0, pre);      // bias + first residual rows
        // every MMA of both warpgroups has completed before the staging tile overwrites the operand stages (the producer
        // wrote nothing after the last chunk, whose stage the consumers have waited for)
        asm volatile("bar.sync 1, 256;" ::: "memory");
        conv_acc_to_staging<BN>(acc, reinterpret_cast<float*>(smem), SM::STG_LD);
        if (tid == 0) stamp(6);
    } else {
        // ======================= producer: activation gather + weight TMA =======================
        // Thread p gathers the 16-byte segment q of rows rsub + 8 i (i = 0..15) of every chunk, in two half chunks (rows
        // [0, 64) then [64, 128)) of 8 float4.  A ring of three half-chunk buffers keeps the next two in flight.
        const int p = tid - 256, q = p & 15, rsub = p >> 4;
        // byte offset of this thread's 8-byte slot in the 128 x 64 half tile (128B swizzle; row & 7 == rsub)
        const uint32_t soff = rsub * 128 + (((q >> 1) ^ rsub) << 4) + ((q & 1) << 3);
        const float4* in4 = reinterpret_cast<const float4*>(a.in);
        // source of row rsub + 8 i for the current filter tap, in float4 units (~0u = zero padding / out of range);
        // recomputed only when the tap changes (never for 1x1 convs and linears, every Cin/64 chunks for 3x3)
        uint32_t off[16];
        int cur_tap = -1, c4 = 0;
        if (p == 0) { tma_prefetch_desc(&tmWh); if constexpr (SPLIT) tma_prefetch_desc(&tmWl); }
        auto load_half = [&](int h, auto part_c, float4* v) {
            constexpr int part = decltype(part_c)::value;
            if (part == 0) {
                const int kc = kbeg + (h >> 1);
                int tap, c0;
                if (cpt > 0) { tap = kc / cpt; c0 = ((kc - tap * cpt) << 6) + q * 4; }       // Cin % 64 == 0
                else { const int k = kc * 64 + q * 4; tap = k / a.Cin; c0 = k - tap * a.Cin; }  // Cin % 4 == 0 (stem)
                c4 = c0 >> 2;
                if (tap != cur_tap) {
                    cur_tap = tap;
                    const bool kvalid = tap < a.KH * a.KW;                                     // zero padding of K
                    const int ky = tap / a.KW, kx = tap - ky * a.KW;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const RowInfo ri = rinfo[rsub + i * 8];
                        const int iy = ri.iy0 + ky, ix = ri.ix0 + kx;
                        off[i] = (kvalid && ri.valid && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W)
                                     ? (uint32_t)(((size_t)(ri.pix_base + iy * a.W + ix) * a.ldin) >> 2)
                                     : ~0u;
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const uint32_t o = off[part * 8 + i];
                v[i] = o != ~0u ? __ldg(in4 + ((size_t)o + c4)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        };
        auto store_half = [&](int h, auto part_c, const float4* v) {
            constexpr int part = decltype(part_c)::value;
            const int it = h >> 1, s = it % STAGES;
            uint8_t* stage = smem + s * SM::STAGE_BYTES;
            if (part == 0) {
                if (it >= STAGES) mbar_wait_cp(&s_free[s], ((it / STAGES) - 1) & 1, a.spin);
                if (p == 0) {
                    uint8_t* Bh = stage + SM::PARTS * SM::A_BYTES;
                    mbar_arrive_expect_tx(&b_full[s], SM::PARTS * SM::B_BYTES);
                    tma_load_2d(Bh, &tmWh, &b_full[s], (kbeg + it) * 64, n0);
                    if constexpr (SPLIT) tma_load_2d(Bh + SM::B_BYTES, &tmWl, &b_full[s], (kbeg + it) * 64, n0);
                }
            }
            uint8_t* Ah = stage + part * 64 * 128 + soff;
            uint8_t* Al = Ah + SM::A_BYTES;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const __half2 h0 = __floats2half2_rn(v[i].x, v[i].y), h1 = __floats2half2_rn(v[i].z, v[i].w);
                if constexpr (!SPLIT) {
                    uint2 ph;
                    ph.x = *reinterpret_cast<const uint32_t*>(&h0); ph.y = *reinterpret_cast<const uint32_t*>(&h1);
                    *reinterpret_cast<uint2*>(Ah + i * 1024) = ph;
                    continue;
                }
                const __half2 l0 = __floats2half2_rn(v[i].x - __low2float(h0), v[i].y - __high2float(h0));
                const __half2 l1 = __floats2half2_rn(v[i].z - __low2float(h1), v[i].w - __high2float(h1));
                uint2 ph, pl;
                ph.x = *reinterpret_cast<const uint32_t*>(&h0); ph.y = *reinterpret_cast<const uint32_t*>(&h1);
                pl.x = *reinterpret_cast<const uint32_t*>(&l0); pl.y = *reinterpret_cast<const uint32_t*>(&l1);
                *reinterpret_cast<uint2*>(Ah + i * 1024) = ph;      // row part*64 + i*8 + rsub
                *reinterpret_cast<uint2*>(Al + i * 1024) = pl;
            }
            if (part == 1) {
                fence_proxy_async();      // generic-proxy smem writes -> visible to the tensor core (async proxy)
                mbar_arrive(&a_full[s]);
                if (it == 0 && p == 0) stamp(2);
            }
        };
        using P0 = std::integral_constant<int, 0>;
        using P1 = std::integral_constant<int, 1>;
        const int nh = 2 * nloc;      // half chunks; h -> buffer h % 3, part h % 2
        float4 v0[8], v1[8], v2[8];
        if (nh > 0) { load_half(0, P0{}, v0); load_half(1, P1{}, v1); }
#pragma unroll 1
        for (int h = 0; h < nh; h += 6) {
            if (h + 2 < nh) load_half(h + 2, P0{}, v2);
            store_half(h, P0{}, v0);
            if (h + 3 < nh) load_half(h + 3, P1{}, v0);
            store_half(h + 1, P1{}, v1);
            if (h + 2 < nh) {
                if (h + 4 < nh) load_half(h + 4, P0{}, v1);
                store_half(h + 2, P0{}, v2);
                if (h + 5 < nh) load_half(h + 5, P1{}, v2);
                store_half(h + 3, P1{}, v0);
            }
            if (h + 4 < nh) {
                if (h + 6 < nh) load_half(h + 6, P0{}, v0);
                store_half(h + 4, P0{}, v1);
                if (h + 7 < nh) load_half(h + 7, P1{}, v1);
                store_half(h + 5, P1{}, v2);
            }
        }
        if (p == 0) stamp(5);
    }
    // Finish: CTA z of a split-K cluster owns rows [z*128/S, (z+1)*128/S) of the tile and reads that slice of every
    // peer's staging buffer through distributed shared memory, summing in rank order (deterministic); without split-K
    // (S = 1) it is the CTA's own buffer.  Then bias / residual / activation and coalesced row stores.  No global
    // partials, no second kernel.
    __syncwarp();
    if (a.splits > 1) cluster_sync_all(); else __syncthreads();
    if (tid == 0) stamp(8);
    if (warp < 8) {
        const int zr = a.splits > 1 ? (int)blockIdx.z : 0;
        if (a.splits == 1) conv_finish_tile_pre<BN>(a, smem, tid, m0, n0, pre);
        else if (a.splits == 2) conv_finish_tile<BN, 2, 4>(a, smem, tid, m0, n0, zr);
        else if (a.splits == 4) conv_finish_tile<BN, 4, 2>(a, smem, tid, m0, n0, zr);
        else conv_finish_tile<BN, 8, 2>(a, smem, tid, m0, n0, zr);
    }
    if (tid == 0) stamp(9);
    if (a.splits > 1) {
        __syncwarp();
        cluster_sync_all();      // nobody leaves (and frees its shared memory) while a peer may still read it
    }
    if (tid == 0) stamp(7);
}

static int make_tmap_weights(CUtensorMap* out, const void* base, int Kpad, int Cout, int BN) {
    PFN_encodeTiled fn = tensor_map_encoder();
    if (!fn) return AOTB_ERR_CUDA;
    cuuint64_t dims[2] = {(cuuint64_t)Kpad, (cuuint64_t)Cout};
    cuuint64_t strides[1] = {(cuuint64_t)Kpad * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)BN};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(weights) failed (%d)", (int)r);
        return AOTB_ERR_CUDA;
    }
    return AOTB_OK;
}

template <int BN, int STAGES, bool SPLIT>
static int launch_conv_tc(const CUtensorMap& th, const CUtensorMap& tl, const ConvTcArgs& a, cudaStream_t st) {
    constexpr int smem = ConvSmem<BN, STAGES, SPLIT>::TOTAL;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BN, STAGES, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             smem);
        if (e != cudaSuccess) {
            set_error("aotb_conv2d_nhwc_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    dim3 grid(cdiv(a.M, 128), a.Cout / BN, a.splits);
    launch_cluster(conv_tc_kernel<BN, STAGES, SPLIT>, dim3(grid), dim3(384), smem, st, a.splits, th, tl, a);
    return check_launch("aotb_conv2d_nhwc_tc");
}

}  // namespace tc
}  // namespace aotb

using namespace aotb;

extern "C" int aotb_set_conv_tiling(int mode) {
    AOTB_REQUIRE(mode >= 0 && mode < (1 << 12), "aotb_set_conv_tiling: mode is a 12-bit mask");
    tc::g_conv_tiling = mode;
    return AOTB_OK;
}

// wh / wl: pre-split weights [Cout][Kpad] fp16 (K = KH*KW*Cin ordered (ky,kx,ci), zero-padded to a multiple of 64);
// wl == null selects the single-pass kernel (hi operands only); wscale [Cout]: per-channel factor of the accumulator (null = 1).
extern "C" int aotb_conv2d_nhwc_tc(const float* in, const void* wh, const void* wl, const float* bias, const float* wscale,
                                   const float* res, float* out, int B, int H, int W, int Cin, int ldin, int Cout, int ldout, int ldres,
                                   int KH, int KW, int stride, int pad, int act, void* workspace, size_t workspace_bytes,
                                   void* stream) {
    AOTB_REQUIRE(in && wh && out, "aotb_conv2d_nhwc_tc: null pointer");
    const bool split = wl != nullptr;
    AOTB_REQUIRE(Cin % 4 == 0 && Cout % 64 == 0, "aotb_conv2d_nhwc_tc: Cin must be a multiple of 4, Cout of 64");
    AOTB_REQUIRE(act >= aotb::ACT_NONE && act <= aotb::ACT_RELU6, "aotb_conv2d_nhwc_tc: activation %d not supported (0-4)", act);
    AOTB_REQUIRE(ldin % 4 == 0 && ldout % 4 == 0 && (!res || ldres % 4 == 0) && ((uintptr_t)in % 16 == 0) &&
                     ((uintptr_t)out % 16 == 0) && (!res || (uintptr_t)res % 16 == 0) && (!bias || (uintptr_t)bias % 16 == 0) &&
                     (!wscale || (uintptr_t)wscale % 16 == 0),
                 "aotb_conv2d_nhwc_tc: 16-byte alignment required");
    // the producer addresses the input in 32-bit float4 offsets (~0u marks padding)
    AOTB_REQUIRE((size_t)B * H * W * ldin / 4 < 0xFFFFFFFFull, "aotb_conv2d_nhwc_tc: input larger than 2^32 float4");
    tc::ConvTcArgs a;
    a.in = in; a.bias = bias; a.wscale = wscale; a.res = res; a.out = out;
    a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.ldin = ldin;
    a.Ho = (H + 2 * pad - KH) / stride + 1;
    a.Wo = (W + 2 * pad - KW) / stride + 1;
    AOTB_REQUIRE(a.Ho > 0 && a.Wo > 0, "aotb_conv2d_nhwc_tc: empty output");
    a.Cout = Cout; a.ldout = ldout; a.ldres = ldres; a.KH = KH; a.KW = KW; a.stride = stride; a.pad = pad;
    a.M = B * a.Ho * a.Wo;
    const int K = ((KH * KW * Cin + 63) / 64) * 64;   // weights are zero-padded to a multiple of 64 along K
    a.nchunks = K / 64;
    a.act = act;
    // Tile policy: pick the N tile (64 / 128 / 256 dividing Cout) and the split-K cluster size (1 / 2 / 4 / 8) that minimise
    //     T = waves * (ramp + chunks_per_cta * t_chunk[BN] + t_finish[BN]),   t_chunk[BN] = max(kGather, BN / 64)
    // over the 132 SMs of an H100 (one CTA per SM).  Costs are in units of the MMAs of one BN = 64 chunk.  The producer's
    // gather of a chunk (32 KB of fp32 activations) overlaps the MMAs and takes kGather units whatever BN is, so narrow
    // tiles are gather-bound and BN = 256 is MMA-bound.  Split-K is only used to fill a partial wave.  kGather was fitted
    // with scripts/conv_sweep.py on an H100 (80GB HBM3, 700 W): over the 20 conv / linear shapes of an R50-AOTL 480p frame
    // the policy's tiles take 632 us in total against 632 us for the best measured tiling of each shape.  Bit 0 of the
    // tuning mask ("narrow") selects the simpler heuristic instead.
    // The single-pass kernel has its own row: one MMA per k-step (a third of the units) and its own gather constant
    // kGather1 (half the shared-memory stores, no lo split), so every tile is gather-bound and the choice turns on waves
    // and finish cost.  Checked with scripts/conv_sweep.py --single-pass on the same card and shapes: the policy's tiles
    // take 478 us against 473 us for the best measured tiling of each shape (the split kernel's policy: 633 us).
    const int mt = cdiv(a.M, 128);
    int BN = 64, best_s = 1;
    const float kGather = 2.5f, kGather1 = 2.0f;
    if ((tc::g_conv_tiling & 1) == 0) {
        float best = 1e30f;
        const int bns[3] = {256, 128, 64};
        const float t_chunk[3] = {fmaxf(kGather, 4.0f), fmaxf(kGather, 2.0f), fmaxf(kGather, 1.0f)};
        const float t_chunk1[3] = {fmaxf(kGather1, 4.0f / 3), fmaxf(kGather1, 2.0f / 3), fmaxf(kGather1, 1.0f / 3)};
        const float t_fin[3] = {8.0f, 4.0f, 2.0f};
        for (int bi = 0; bi < 3; ++bi) {
            if (Cout % bns[bi]) continue;
            for (int sp = 1; sp <= 8; sp <<= 1) {
                if (sp > a.nchunks) break;
                const int ctas = mt * (Cout / bns[bi]) * sp;
                const int slots = sp == 8 ? 128 : 132;                        // co-resident CTAs with clusters of sp
                if (sp > 1 && ctas > slots) continue;                         // split-K only to fill a partial wave
                const int waves = cdiv(ctas, slots);
                const float t = waves * (3.0f + cdiv(a.nchunks, sp) * (split ? t_chunk[bi] : t_chunk1[bi]) + t_fin[bi]);
                if (t < best) { best = t; BN = bns[bi]; best_s = sp; }
            }
        }
    } else {          // "narrow": BN = 128 when that still fills ~a wave on its own, else 64; split-K to ~one wave
        if (Cout % 128 == 0 && mt * (Cout / 128) >= 120) BN = 128;
        const int ctas = mt * (Cout / BN);
        if (ctas < 100 && a.nchunks >= 4) {
            best_s = 8;
            while (best_s > 1 && (ctas * best_s > 160 || a.nchunks / best_s < 2)) best_s >>= 1;
        }
    }
    const int force_bn = (tc::g_conv_tiling >> 4) & 15, force_s = (tc::g_conv_tiling >> 8) & 15;
    if (force_bn) {
        BN = 32 << force_bn;
        AOTB_REQUIRE((BN == 64 || BN == 128 || BN == 256) && Cout % BN == 0, "aotb_conv2d_nhwc_tc: forced tile %d invalid", BN);
    }
    a.splits = force_bn ? 1 : best_s;
    const int ctas = mt * (Cout / BN);
    if (force_s) {
        AOTB_REQUIRE((force_s == 1 || force_s == 2 || force_s == 4 || force_s == 8) && force_s <= a.nchunks,
                     "aotb_conv2d_nhwc_tc: forced split %d invalid", force_s);
        a.splits = force_s;
    }
    a.spin = (tc::g_conv_tiling & 2) ? 1 : 0;
    a.prof = nullptr;
    if (tc::g_conv_tiling & 4) {      // diagnostic stamps go to the caller's workspace
        const size_t need = (size_t)ctas * a.splits * 12 * sizeof(long long);
        AOTB_REQUIRE(workspace && workspace_bytes >= need, "aotb_conv2d_nhwc_tc: profile mode needs %zu workspace bytes", need);
        a.prof = (long long*)workspace;
    }
    CUtensorMap th, tl;
    int rc;
    if ((rc = tc::make_tmap_weights(&th, wh, K, Cout, BN)) != AOTB_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (!split) {             // the kernel never reads tmWl
        if (BN == 256) return tc::launch_conv_tc<256, 4, false>(th, th, a, st);
        if (BN == 128) return tc::launch_conv_tc<128, 6, false>(th, th, a, st);
        return tc::launch_conv_tc<64, 8, false>(th, th, a, st);
    }
    if ((rc = tc::make_tmap_weights(&tl, wl, K, Cout, BN)) != AOTB_OK) return rc;
    if (BN == 256) return tc::launch_conv_tc<256, 2, true>(th, tl, a, st);
    if (BN == 128) return tc::launch_conv_tc<128, 3, true>(th, tl, a, st);
    return tc::launch_conv_tc<64, 4, true>(th, tl, a, st);
}
