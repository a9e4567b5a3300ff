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
// One tile = 128 output pixels x BN (64 | 128 | 256) output channels; 384 threads in three warpgroups, warp-specialised.
// Without split-K the launch is persistent: min(tiles, SMs) CTAs, CTA b computing tiles b, b + grid, ... in a static order,
// with one stage ring whose chunk counter and phases run on across tiles.
//   warps 0-7   two consumer warpgroups (64 pixel rows each).  Per K chunk they wait for the stage's "A full" and "B full"
//               barriers, issue 4 k-steps x (Ah Wh + Al Wh + Ah Wl) as wgmma m64nBNk16 and release the stage of the
//               previous chunk on "empty" once its MMAs have completed (and the tile's last stage after its final wait).
//               Then the same warps run the finish (bias / residual / activation -> fp32 NHWC) from the accumulator
//               registers while the producer already gathers the next tile; split-K goes through a staging tile instead.
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
    int M, mtiles, nchunks;
    int act;
    int splits;          // split-K: the `splits` CTAs (blockIdx.z) of one output tile form a thread-block cluster; CTA z
                         // handles chunks [z*per, (z+1)*per) and the partial tiles are summed over distributed smem
    int spin;            // 1: mbarrier waits without the suspend hint
    int const_w;         // 1: no earlier kernel of the stream writes the weights (their first TMA loads precede pdl_wait)
    long long* prof;     // diagnostic: 12 clock64 stamps per CTA (see aotb_set_conv_tiling), or null
    int htx, hti;        // halo path: 16-column tiles per map row, 8 x 16 tiles per image
};

constexpr int AOTB_CONV_CONST_WEIGHTS = 256;       // flag in the act argument (include/aotb200.h)
static int g_conv_tiling = 0;      // aotb_set_conv_tiling
static int g_conv_grid_cap = 0;    // aotb_set_conv_grid_cap (0: one CTA per SM)
static int g_conv_halo = 1;        // aotb_set_conv_halo (0: never, 1: tile model, 2: every eligible launch)

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

__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }

// Finish without split-K, straight from the accumulator fragments (persistent launches: no staging tile, so the operand
// stages stay free for the next tile's loads).  Thread (warp w, lane l) holds rows r and r + 8 (r = 64 (w / 4) + 16 (w % 4)
// + l / 4) at columns 8 k + 2 (l % 4) + {0, 1}: one float2 per row and column group, so the four lanes of a row write a full
// 32-byte sector.  The residual is read in the same layout, by the thread that then writes the element (an in-place
// residual, res == out, is read before it is overwritten).  Same arithmetic per element as conv_finish_tile: bitwise equal.
// bs: the tile's bias and scale columns in shared memory ([2][BN]).  The activation is a template argument: a runtime
// switch per element, unrolled over BN / 2 elements, would not fit the instruction cache.  For the same reason GELU and
// SiLU run a rolled loop over the column groups (the accumulators shift down one group per step), so their erf / exp code
// appears once.  G column groups per batch: every residual load of a batch is issued before its first use.  With one
// group per batch (BN = 256, where 128 accumulators leave no room for more, and the rolled loop) each step would wait a
// full L2 round trip for its residual; prefetch.global.L1 requests the groups PF steps ahead without registers.
// r: output pixel of the thread's first row; its second row is pixel r + 8 (ok0 / ok1: the rows lie in the map).
template <int BN, int ACT>
__device__ __forceinline__ void conv_finish_frag(const ConvTcArgs& a, float* acc, const float* bs, int r, bool ok0, bool ok1,
                                                 int n0) {
    constexpr bool ROLL = ACT == ACT_GELU || ACT == ACT_SILU;
    constexpr int G = (ROLL || BN == 256) ? 1 : 8, NG = BN / 8, PF = 8;
    const int lane = threadIdx.x & 31;
    const int c = (lane & 3) * 2;
    const bool ok[2] = {ok0, ok1};
    auto res_at = [&](int h, int k) { return a.res + (size_t)(r + 8 * h) * a.ldres + n0 + c + 8 * k; };
    auto prefetch = [&](int k) {
        if (G == 1 && a.res && k < NG) {
            if (ok[0]) prefetch_l1(res_at(0, k));
            if (ok[1]) prefetch_l1(res_at(1, k));
        }
    };
    // one column group: o = act(fmaf(acc, scale, bias) + res), acc[j], acc[j + 1] at row r + 8 h
    auto group = [&](int k, int h, float a0, float a1, float2 rs) {
        const int n = c + 8 * k;
        const float2 b2 = *reinterpret_cast<const float2*>(bs + n), s2 = *reinterpret_cast<const float2*>(bs + BN + n);
        // o * s is exact (s is a power of two), so the fma rounds like o * s + b
        float ox = fmaf(a0, s2.x, b2.x), oy = fmaf(a1, s2.y, b2.y);
        ox += rs.x; oy += rs.y;
        ox = apply_act(ox, ACT); oy = apply_act(oy, ACT);
        if (ok[h]) *reinterpret_cast<float2*>(a.out + (size_t)(r + 8 * h) * a.ldout + n0 + n) = make_float2(ox, oy);
    };
#pragma unroll
    for (int k = 0; k < PF; ++k) prefetch(k);
    if constexpr (ROLL) {
#pragma unroll 1
        for (int k = 0; k < NG; ++k) {
            prefetch(k + PF);
            float2 rs[2];
#pragma unroll
            for (int h = 0; h < 2; ++h)
                rs[h] = (a.res && ok[h]) ? *reinterpret_cast<const float2*>(res_at(h, k)) : make_float2(0.f, 0.f);
#pragma unroll
            for (int h = 0; h < 2; ++h) group(k, h, acc[2 * h], acc[2 * h + 1], rs[h]);
#pragma unroll
            for (int i = 0; i < BN / 2 - 4; ++i) acc[i] = acc[i + 4];
        }
    } else {
#pragma unroll
        for (int k0 = 0; k0 < NG; k0 += G) {
            prefetch(k0 + PF);
            float2 rs[G][2];
#pragma unroll
            for (int k = 0; k < G; ++k)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    rs[k][h] = (a.res && ok[h]) ? *reinterpret_cast<const float2*>(res_at(h, k0 + k)) : make_float2(0.f, 0.f);
#pragma unroll
            for (int k = 0; k < G; ++k)
#pragma unroll
                for (int h = 0; h < 2; ++h) group(k0 + k, h, acc[4 * (k0 + k) + 2 * h], acc[4 * (k0 + k) + 2 * h + 1], rs[k][h]);
        }
    }
}

template <int BN>
__device__ __forceinline__ void conv_finish_act(const ConvTcArgs& a, float* acc, const float* bs, int r, bool ok0, bool ok1,
                                                int n0) {
    switch (a.act) {
        case ACT_RELU: conv_finish_frag<BN, ACT_RELU>(a, acc, bs, r, ok0, ok1, n0); break;
        case ACT_GELU: conv_finish_frag<BN, ACT_GELU>(a, acc, bs, r, ok0, ok1, n0); break;
        case ACT_SILU: conv_finish_frag<BN, ACT_SILU>(a, acc, bs, r, ok0, ok1, n0); break;
        case ACT_RELU6: conv_finish_frag<BN, ACT_RELU6>(a, acc, bs, r, ok0, ok1, n0); break;
        default: conv_finish_frag<BN, ACT_NONE>(a, acc, bs, r, ok0, ok1, n0); break;
    }
}

template <int BN, int STAGES, bool SPLIT, bool PERSIST>
struct ConvSmem {
    static constexpr int A_BYTES = CONV_A_BYTES;
    static constexpr int B_BYTES = BN * 128;
    static constexpr int PARTS = SPLIT ? 2 : 1;        // hi and lo tiles, or hi only
    static constexpr int STAGE_BYTES = PARTS * A_BYTES + PARTS * B_BYTES;
    static constexpr int STG_LD = BN + 4;              // split-K staging tile [128][BN + 4] fp32, aliases the stages
    static_assert(128 * STG_LD * 4 <= STAGES * STAGE_BYTES, "staging tile must fit in the operand stages");
    // persistent: row tables of two tiles and the bias / scale columns of two tiles; split-K: one row table
    static constexpr int RTABLES = PERSIST ? 2 : 1, BS_FLOATS = PERSIST ? 2 * 2 * BN : 0;
    static constexpr int TOTAL = STAGES * STAGE_BYTES + RTABLES * 128 * (int)sizeof(RowInfo) + BS_FLOATS * 4 + 3 * STAGES * 8 + 1024;
    static_assert(TOTAL <= 227 * 1024, "shared memory of one CTA");
};

// PERSIST (launches without split-K): grid.x <= tiles CTAs, CTA b computing tiles b, b + grid.x, ... with t = mb * ntn + nb
// (the N tiles of one M block are adjacent), the finish straight from the accumulators.  !PERSIST (split-K): grid
// (M tiles, N tiles, splits), one tile per CTA, the cluster's partial tiles summed through staging tiles.  Separate
// instantiations, so the split-K launches run a one-tile body without the tile loop and the per-activation finishes.
template <int BN, int STAGES, bool SPLIT, bool PERSIST>
__global__ void __launch_bounds__(384, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const ConvTcArgs a) {
    using SM = ConvSmem<BN, STAGES, SPLIT, PERSIST>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    RowInfo* rinfo = reinterpret_cast<RowInfo*>(smem + STAGES * SM::STAGE_BYTES);   // [RTABLES][128]: tiles j, j + 1
    float* bsm = reinterpret_cast<float*>(rinfo + SM::RTABLES * 128);  // [2][2][BN]: bias, scale of tiles j, j + 1
    uint64_t* a_full = reinterpret_cast<uint64_t*>(bsm + SM::BS_FLOATS);  // 128 producer-thread arrivals
    uint64_t* b_full = a_full + STAGES;                               // TMA transaction bytes
    uint64_t* s_free = b_full + STAGES;                               // 8 consumer-warp arrivals

    const int tid = threadIdx.x, warp = tid >> 5;
    const int ntn = a.Cout / BN, ntiles = a.mtiles * ntn;
    // tiles of this CTA
    const int ntc = !PERSIST ? 1 : (int)blockIdx.x < ntiles ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    auto tile_m0 = [&](int j) {
        if constexpr (PERSIST) return ((int)(blockIdx.x + j * gridDim.x) / ntn) * 128;
        else return (int)blockIdx.x * 128;
    };
    auto tile_n0 = [&](int j) {
        if constexpr (PERSIST) return ((int)(blockIdx.x + j * gridDim.x) % ntn) * BN;
        else return (int)blockIdx.y * BN;
    };
    long long* prof = a.prof ? a.prof + 12 * ((size_t)(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) : nullptr;
    auto stamp = [&](int slot) { if (prof) prof[slot] = clock64(); };
    if (tid == 0) stamp(0);
    pdl_trigger();      // the next kernel may start its prologue; it waits for this grid before reading our output

    const int per = PERSIST ? a.nchunks : (a.nchunks + a.splits - 1) / a.splits;
    const int kbeg = PERSIST ? 0 : blockIdx.z * per;
    const int nloc = max(0, min(per, a.nchunks - kbeg));     // chunks per tile of this CTA (local it <-> chunk kbeg + it)
    // Global chunk g = j * nloc + it runs on across the CTA's tiles: stage g % STAGES, phase (g / STAGES) & 1.
    const int nchk = ntc * nloc;
    // constant weights (a.const_w): the B tiles of the first STAGES chunks are requested before the grid dependency wait
    const int npre = a.const_w ? min(STAGES, nchk) : 0;
    auto issue_b = [&](int g) {
        const int j = PERSIST ? g / nloc : 0, it = g - j * nloc, s = g % STAGES;
        uint8_t* Bh = smem + s * SM::STAGE_BYTES + SM::PARTS * SM::A_BYTES;
        mbar_arrive_expect_tx(&b_full[s], SM::PARTS * SM::B_BYTES);
        tma_load_2d(Bh, &tmWh, &b_full[s], (kbeg + it) * 64, tile_n0(j));
        if constexpr (SPLIT) tma_load_2d(Bh + SM::B_BYTES, &tmWl, &b_full[s], (kbeg + it) * 64, tile_n0(j));
    };
    // row table of tile j -> rinfo[j & 1], one row per producer thread
    auto write_rows = [&](int j, int p) {
        const int m = tile_m0(j) + p;
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
        rinfo[(j & 1) * 128 + p] = ri;
    };

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&a_full[s], 128); mbar_init(&b_full[s], 1); mbar_init(&s_free[s], 8); }
        fence_mbar_init();
    }
    if (tid >= 256) {
        for (int j = 0; j < min(ntc, 2); ++j) write_rows(j, tid - 256);
    }
    __syncthreads();
    if (tid == 0) stamp(1);
    if (tid == 256) {
        tma_prefetch_desc(&tmWh);
        if constexpr (SPLIT) tma_prefetch_desc(&tmWl);
        for (int g = 0; g < npre; ++g) issue_b(g);
    }
    pdl_wait();         // activations / residual below were written by earlier kernels
    const int cpt = (a.Cin % 64 == 0) ? (a.Cin >> 6) : 0;  // 64-wide chunks per filter tap (0: general Cin % 4 path)

    // warpgroup index made warp-uniform for the compiler: wgmma in a branch it cannot prove uniform is serialised
    const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
    if (wg < 2) {
        // ======================= consumers: wgmma, then the finish of each tile =======================
        const uint64_t dA0 = smem_desc_sw128(smem_u32(smem + wg * 64 * 128));
        const uint64_t dB0 = smem_desc_sw128(smem_u32(smem + SM::PARTS * SM::A_BYTES));
        int g = 0;
#pragma unroll 1
        for (int j = 0; j < ntc; ++j) {
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            float* bs = bsm + (j & 1) * 2 * BN;
            if (PERSIST && tid < BN) {            // read by the finish after the K loop, behind the barrier below
                const int n = tile_n0(j) + tid;
                bs[tid] = a.bias ? __ldg(a.bias + n) : 0.f;
                bs[BN + tid] = a.wscale ? __ldg(a.wscale + n) : 1.f;
            }
#pragma unroll 1
            for (int it = 0; it < nloc; ++it, ++g) {
                const int s = g % STAGES;
                const uint32_t ph = (g / STAGES) & 1;
                mbar_wait_cp(&a_full[s], ph, a.spin);
                mbar_wait_cp(&b_full[s], ph, a.spin);
                if (g == 0 && tid == 0) stamp(3);
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
                if (it > 0) mbar_arrive_warp(&s_free[(g - 1) % STAGES]);
            }
            wgmma_wait<0>();
            reg_fence<BN / 2>(acc);
            if (tid == 0) { if (PERSIST && j == 0) stamp(10); stamp(4); }
            if constexpr (PERSIST) {
                if (nloc > 0) mbar_arrive_warp(&s_free[(g - 1) % STAGES]);   // the producer may refill it for the next tile
                // the bias / scale columns of tile j are visible; every consumer has finished tile j - 1, whose buffer
                // tile j + 1 rewrites
                asm volatile("bar.sync 1, 256;" ::: "memory");
                const int r = tile_m0(j) + warp * 16 + ((tid & 31) >> 2);
                conv_finish_act<BN>(a, acc, bs, r, r < a.M, r + 8 < a.M, tile_n0(j));
                if (tid == 0) { if (j == 0) stamp(8); stamp(9); }
            } else {
                // every MMA of both warpgroups has completed before the staging tile overwrites the operand stages (a split-K
                // CTA has one tile, so the producer writes nothing after its last chunk)
                asm volatile("bar.sync 1, 256;" ::: "memory");
                conv_acc_to_staging<BN>(acc, reinterpret_cast<float*>(smem), SM::STG_LD);
                if (tid == 0) stamp(6);
            }
        }
    } else {
        // ======================= producer: activation gather + weight TMA =======================
        // Thread p gathers the 16-byte segment q of rows rsub + 8 i (i = 0..15) of every chunk, in two half chunks (rows
        // [0, 64) then [64, 128)) of 8 float4.  A ring of three half-chunk buffers keeps the next two in flight, across tile
        // boundaries: the next tile's chunks are gathered while the consumers finish this one.
        const int p = tid - 256, q = p & 15, rsub = p >> 4;
        // byte offset of this thread's 8-byte slot in the 128 x 64 half tile (128B swizzle; row & 7 == rsub)
        const uint32_t soff = rsub * 128 + (((q >> 1) ^ rsub) << 4) + ((q & 1) << 3);
        const float4* in4 = reinterpret_cast<const float4*>(a.in);
        // source of row rsub + 8 i for the current filter tap, in float4 units (~0u = zero padding / out of range);
        // recomputed only when the tap or the tile changes (once per tile for 1x1 convs and linears)
        uint32_t off[16];
        int cur_tap = -1, c4 = 0;
        const RowInfo* rows = rinfo;
        auto load_half = [&](int h, auto part_c, float4* v) {
            constexpr int part = decltype(part_c)::value;
            if (part == 0) {
                const int g = h >> 1, j = PERSIST ? g / nloc : 0, it = g - j * nloc;
                if (PERSIST && it == 0) {   // first chunk of tile j: its row table is rinfo[j & 1]
                    cur_tap = -1;
                    rows = rinfo + (j & 1) * 128;
                    if (j > 0) {
                        // every producer thread has finished reading the table of tile j - 1, and the table of tile j
                        // (written at the start of tile j - 1) is visible: tile j + 1 reuses the buffer of tile j - 1
                        asm volatile("bar.sync 2, 128;" ::: "memory");
                        if (j + 1 < ntc) write_rows(j + 1, p);
                    }
                }
                const int kc = kbeg + it;
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
                        const RowInfo ri = rows[rsub + i * 8];
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
            const int g = h >> 1, s = g % STAGES;
            uint8_t* stage = smem + s * SM::STAGE_BYTES;
            if (part == 0) {
                if (g >= STAGES) mbar_wait_cp(&s_free[s], ((g / STAGES) - 1) & 1, a.spin);
                if (p == 0 && g >= npre) issue_b(g);
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
                if (g == 0 && p == 0) stamp(2);
            }
        };
        using P0 = std::integral_constant<int, 0>;
        using P1 = std::integral_constant<int, 1>;
        const int nh = 2 * nchk;      // half chunks of all tiles; h -> buffer h % 3, part h % 2
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
    if constexpr (!PERSIST) {
        // Split-K finish: CTA z of the cluster owns rows [z*128/S, (z+1)*128/S) of the tile and reads that slice of every
        // peer's staging buffer through distributed shared memory, summing in rank order (deterministic).  Then bias /
        // residual / activation and coalesced row stores.  No global partials, no second kernel.
        __syncwarp();
        cluster_sync_all();
        if (tid == 0) stamp(8);
        if (warp < 8) {
            const int zr = (int)blockIdx.z, m0 = tile_m0(0), n0 = tile_n0(0);
            if (a.splits == 2) conv_finish_tile<BN, 2, 4>(a, smem, tid, m0, n0, zr);
            else if (a.splits == 4) conv_finish_tile<BN, 4, 2>(a, smem, tid, m0, n0, zr);
            else conv_finish_tile<BN, 8, 2>(a, smem, tid, m0, n0, zr);
        }
        if (tid == 0) stamp(9);
        __syncwarp();
        cluster_sync_all();      // nobody leaves (and frees its shared memory) while a peer may still read it
    } else if (tid == 0 && prof) {
        prof[11] = ntc;
    }
    if (tid == 0) stamp(7);
}

// ======================= stride-1 3x3 convolutions from one staged halo per 64-channel slice =======================
// One tile = 8 x 16 output pixels of one image x BN channels; pixel row m of the tile (the accumulator row) is
// (ty, tx) = (m / 16, m % 16), so consumer warp w (0-7) holds map row y0 + w.  For each 64-channel slice of Cin the
// producer stages the tile's 10 x 18 input halo once, split into hi / lo fp16 (180 rows of 128 bytes per part, 16-byte
// column c of halo pixel h at h * 128 + ((c ^ (h % 8)) << 4), so the eight rows an ldmatrix phase reads hit eight
// different bank groups); pixels outside the image are stored as zeros, which is the padding.  The nine taps then read
// their A fragments out of the halo with ldmatrix, each lane addressing the halo pixel of its output pixel shifted by
// (ky, kx), and issue register-A wgmma: per chunk 4 k-steps x (Ah Wh + Al Wh + Ah Wl) as in conv_tc_kernel.
// K runs slice-major, chunk (slice, tap) = K columns [tap * Cin + 64 slice, + 64) of the (ky, kx, ci) weight packing; with
// Cin = 64 that is the order of conv_tc_kernel, whose outputs this kernel then reproduces bit for bit.
//   warps 0-7   consumers.  Per chunk: ldmatrix of KG k-steps, wgmma_fence, their MMAs, wait (the A registers are reused),
//               release the weight stage after the chunk and the halo after the slice's last ldmatrix; the finish as in
//               the persistent conv_tc_kernel.
//   warp 8      one lane streams the weight chunks by TMA into a STAGES ring (b_full / b_free).
//   warps 9-11  halo producers (96 threads), two halo buffers (h_full / h_free): slice u + 1 -- of this or the next
//               tile -- is staged while the taps of slice u run.
constexpr int HALO_PIX = 10 * 18, HALO_PART_BYTES = HALO_PIX * 128;

template <int BN, int STAGES, bool SPLIT>
struct HaloSmem {
    static constexpr int PARTS = SPLIT ? 2 : 1;
    static constexpr int B_BYTES = BN * 128;
    static constexpr int STAGE_BYTES = PARTS * B_BYTES;
    static constexpr int HALO_BYTES = PARTS * HALO_PART_BYTES;
    static constexpr int TOTAL = STAGES * STAGE_BYTES + 2 * HALO_BYTES + 2 * 2 * BN * 4 + (2 * STAGES + 4) * 8 + 1024;
    static_assert(TOTAL <= 227 * 1024, "shared memory of one CTA");
};

template <int BN>
__device__ __forceinline__ void wgmma_rs_conv(float* acc, const uint32_t* a, uint64_t b) {
    if (BN == 256) wgmma_rs_n256(acc, a, b);
    else if (BN == 128) wgmma_rs_n128(acc, a, b);
    else wgmma_rs_n64(acc, a, b);
}

template <int BN, int STAGES, bool SPLIT>
__global__ void __launch_bounds__(384, 1)
conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const ConvTcArgs a) {
    using SM = HaloSmem<BN, STAGES, SPLIT>;
    // k-steps per wgmma group: their A fragments are live until the group's wait (8 registers per k-step when split),
    // beside BN / 2 accumulators
    constexpr int KG = BN < 256 ? 4 : SPLIT ? 1 : 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* halo = smem + STAGES * SM::STAGE_BYTES;                       // [2][PARTS][180][128 B]
    float* bsm = reinterpret_cast<float*>(halo + 2 * SM::HALO_BYTES);     // [2][2][BN]: bias, scale of tiles j, j + 1
    uint64_t* b_full = reinterpret_cast<uint64_t*>(bsm + 4 * BN);          // TMA transaction bytes
    uint64_t* b_free = b_full + STAGES;                                   // 8 consumer-warp arrivals
    uint64_t* h_full = b_free + STAGES;                                   // 96 producer-thread arrivals
    uint64_t* h_free = h_full + 2;                                        // 8 consumer-warp arrivals

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ntn = a.Cout / BN, ntiles = a.mtiles * ntn;
    const int ntc = (int)blockIdx.x < ntiles ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int ns = a.Cin >> 6, nloc = 9 * ns, nchk = ntc * nloc;
    // tile j of this CTA: image b, top-left output pixel (y0, x0), first channel n0; the N tiles of one pixel tile are
    // adjacent and every image has its own tile range
    auto tile_of = [&](int j, int& b, int& y0, int& x0, int& n0) {
        const int t = (int)blockIdx.x + j * (int)gridDim.x, mb = t / ntn;
        n0 = (t - mb * ntn) * BN;
        b = mb / a.hti;
        const int r = mb - b * a.hti, ty = r / a.htx;
        y0 = ty * 8;
        x0 = (r - ty * a.htx) * 16;
    };
    pdl_trigger();
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_free[s], 8); }
        for (int s = 0; s < 2; ++s) { mbar_init(&h_full[s], 96); mbar_init(&h_free[s], 8); }
        fence_mbar_init();
    }
    __syncthreads();
    const int npre = a.const_w ? min(STAGES, nchk) : 0;
    auto issue_b = [&](int g) {
        const int j = g / nloc, it = g - j * nloc, sl = it / 9, tap = it - sl * 9, s = g % STAGES;
        int b, y0, x0, n0;
        tile_of(j, b, y0, x0, n0);
        uint8_t* Bh = smem + s * SM::STAGE_BYTES;
        const int k0 = tap * a.Cin + sl * 64;
        mbar_arrive_expect_tx(&b_full[s], SM::STAGE_BYTES);
        tma_load_2d(Bh, &tmWh, &b_full[s], k0, n0);
        if constexpr (SPLIT) tma_load_2d(Bh + SM::B_BYTES, &tmWl, &b_full[s], k0, n0);
    };
    if (tid == 256) {
        tma_prefetch_desc(&tmWh);
        if constexpr (SPLIT) tma_prefetch_desc(&tmWl);
        for (int g = 0; g < npre; ++g) issue_b(g);
    }
    pdl_wait();         // activations / residual below were written by earlier kernels

    const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
    if (wg < 2) {
        // ======================= consumers =======================
        const uint64_t dB0 = smem_desc_sw128(smem_u32(smem));
        // ldmatrix row of this lane: tile column (lane & 7) + 8 ((lane >> 3) & 1), 16-byte column half lane >> 4
        const int lx = (lane & 7) + ((lane >> 3) & 1) * 8, lc = lane >> 4;
        const uint32_t halo_s = smem_u32(halo);
        int g = 0, u = 0;
#pragma unroll 1
        for (int j = 0; j < ntc; ++j) {
            int b, y0, x0, n0;
            tile_of(j, b, y0, x0, n0);
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            float* bs = bsm + (j & 1) * 2 * BN;
            if (tid < BN) {            // read by the finish after the K loop, behind the barrier below
                bs[tid] = a.bias ? __ldg(a.bias + n0 + tid) : 0.f;
                bs[BN + tid] = a.wscale ? __ldg(a.wscale + n0 + tid) : 1.f;
            }
#pragma unroll 1
            for (int sl = 0; sl < ns; ++sl, ++u) {
                const int hb = u & 1;
                mbar_wait_cp(&h_full[hb], (u >> 1) & 1, a.spin);
                const uint32_t hbase = halo_s + hb * SM::HALO_BYTES;
#pragma unroll 1
                for (int tap = 0; tap < 9; ++tap, ++g) {
                    const int ky = tap / 3, kx = tap - ky * 3;
                    const int hp = (warp + ky) * 18 + lx + kx;
                    const uint32_t rowa = hbase + hp * 128, sw = hp & 7;
                    const int s = g % STAGES;
                    mbar_wait_cp(&b_full[s], (g / STAGES) & 1, a.spin);
                    const uint64_t bh = dB0 + (uint64_t)((s * SM::STAGE_BYTES) >> 4), bl = bh + (uint64_t)(SM::B_BYTES >> 4);
#pragma unroll
                    for (int k0 = 0; k0 < 4; k0 += KG) {
                        uint32_t ah[KG][4], al[KG][4];
#pragma unroll
                        for (int k = 0; k < KG; ++k) {
                            const uint32_t ad = rowa + (((2 * (k0 + k) + lc) ^ sw) << 4);
                            ldmatrix_x4(ah[k], ad);
                            if constexpr (SPLIT) ldmatrix_x4(al[k], ad + HALO_PART_BYTES);
                        }
                        // the slice's last reads of the halo are in registers: the producer may restage it
                        if (tap == 8 && k0 + KG == 4) mbar_arrive_warp(&h_free[hb]);
                        reg_fence<BN / 2>(acc);
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < KG; ++k) {
                            const int ks = k0 + k;
                            wgmma_rs_conv<BN>(acc, ah[k], bh + 2 * ks);
                            if constexpr (SPLIT) {
                                wgmma_rs_conv<BN>(acc, al[k], bh + 2 * ks);
                                wgmma_rs_conv<BN>(acc, ah[k], bl + 2 * ks);
                            }
                        }
                        wgmma_commit();
                        wgmma_wait<0>();
                        reg_fence<BN / 2>(acc);
#pragma unroll
                        for (int k = 0; k < KG; ++k)       // the fragments stay allocated until the wait above
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                asm volatile("" : "+r"(ah[k][i])::"memory");
                                if constexpr (SPLIT) asm volatile("" : "+r"(al[k][i])::"memory");
                            }
                    }
                    mbar_arrive_warp(&b_free[s]);
                }
            }
            // the bias / scale columns of tile j are visible; every consumer has finished tile j - 1, whose buffer
            // tile j + 1 rewrites
            asm volatile("bar.sync 1, 256;" ::: "memory");
            const int oy = y0 + warp, ox = x0 + (lane >> 2);
            const int r = (b * a.H + oy) * a.W + ox;
            conv_finish_act<BN>(a, acc, bs, r, oy < a.H && ox < a.W, oy < a.H && ox + 8 < a.W, n0);
        }
    } else if (warp == 8) {
        // ======================= weight TMA =======================
        if (lane == 0) {
#pragma unroll 1
            for (int g = npre; g < nchk; ++g) {
                const int s = g % STAGES;
                if (g >= STAGES) mbar_wait_cp(&b_free[s], ((g / STAGES) - 1) & 1, a.spin);
                issue_b(g);
            }
        }
    } else {
        // ======================= halo producers =======================
        // Thread p loads the 16-byte segment q = p % 16 (channels 4 q .. 4 q + 3 of the slice) of halo pixels p / 16 + 6 i,
        // i = 0..29, in batches of NB loads in flight (two round trips to memory per slice; three at BN = 256, whose 128
        // accumulators leave fewer registers).
        const int p = tid - 288, q = p & 15, h0 = p >> 4;
        const float4* in4 = reinterpret_cast<const float4*>(a.in);
        int u = 0;
#pragma unroll 1
        for (int j = 0; j < ntc; ++j) {
            int b, y0, x0, n0;
            tile_of(j, b, y0, x0, n0);
#pragma unroll 1
            for (int sl = 0; sl < ns; ++sl, ++u) {
                const int hb = u & 1;
                if (u >= 2) mbar_wait_cp(&h_free[hb], ((u >> 1) - 1) & 1, a.spin);
                uint8_t* hh = halo + hb * SM::HALO_BYTES;
                const int c4 = sl * 16 + q;
                constexpr int NB = BN == 256 ? 10 : 15;
#pragma unroll 1
                for (int i0 = 0; i0 < 30; i0 += NB) {
                    float4 v[NB];
#pragma unroll
                    for (int i = 0; i < NB; ++i) {
                        const int h = h0 + 6 * (i0 + i), hy = h / 18, hx = h - hy * 18;
                        const int iy = y0 - 1 + hy, ix = x0 - 1 + hx;
                        v[i] = (iy >= 0 && iy < a.H && ix >= 0 && ix < a.W)
                                   ? __ldg(in4 + (((size_t)(b * a.H + iy) * a.W + ix) * a.ldin >> 2) + c4)
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
#pragma unroll
                    for (int i = 0; i < NB; ++i) {
                        const int h = h0 + 6 * (i0 + i);
                        uint8_t* dst = hh + h * 128 + ((((q >> 1) ^ (h & 7))) << 4) + ((q & 1) << 3);
                        const __half2 x0h = __floats2half2_rn(v[i].x, v[i].y), x1h = __floats2half2_rn(v[i].z, v[i].w);
                        uint2 ph;
                        ph.x = *reinterpret_cast<const uint32_t*>(&x0h); ph.y = *reinterpret_cast<const uint32_t*>(&x1h);
                        *reinterpret_cast<uint2*>(dst) = ph;
                        if constexpr (SPLIT) {
                            const __half2 l0 = __floats2half2_rn(v[i].x - __low2float(x0h), v[i].y - __high2float(x0h));
                            const __half2 l1 = __floats2half2_rn(v[i].z - __low2float(x1h), v[i].w - __high2float(x1h));
                            uint2 pl;
                            pl.x = *reinterpret_cast<const uint32_t*>(&l0); pl.y = *reinterpret_cast<const uint32_t*>(&l1);
                            *reinterpret_cast<uint2*>(dst + HALO_PART_BYTES) = pl;
                        }
                    }
                }
                mbar_arrive(&h_full[hb]);
            }
        }
    }
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

static int sm_count() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
            n = 132;
    }
    return n;
}

// Without split-K one persistent CTA per SM (at most one per tile, at most the grid cap); split-K: one CTA per tile and K slice.
static dim3 conv_grid(const ConvTcArgs& a, int BN) {
    if (a.splits > 1) return dim3(a.mtiles, a.Cout / BN, a.splits);
    const int cap = g_conv_grid_cap > 0 ? g_conv_grid_cap : sm_count();
    return dim3(min(a.mtiles * (a.Cout / BN), cap), 1, 1);
}

template <int BN, int STAGES, bool SPLIT, bool PERSIST>
static int launch_conv_tc_as(const CUtensorMap& th, const CUtensorMap& tl, const ConvTcArgs& a, cudaStream_t st) {
    constexpr int smem = ConvSmem<BN, STAGES, SPLIT, PERSIST>::TOTAL;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BN, STAGES, SPLIT, PERSIST>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) {
            set_error("aotb_conv2d_nhwc_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    launch_cluster(conv_tc_kernel<BN, STAGES, SPLIT, PERSIST>, conv_grid(a, BN), dim3(384), smem, st, a.splits, th, tl, a);
    return check_launch("aotb_conv2d_nhwc_tc");
}

template <int BN, int STAGES, bool SPLIT>
static int launch_conv_tc(const CUtensorMap& th, const CUtensorMap& tl, const ConvTcArgs& a, cudaStream_t st) {
    return a.splits > 1 ? launch_conv_tc_as<BN, STAGES, SPLIT, false>(th, tl, a, st)
                        : launch_conv_tc_as<BN, STAGES, SPLIT, true>(th, tl, a, st);
}

template <int BN, int STAGES, bool SPLIT>
static int launch_halo(const CUtensorMap& th, const CUtensorMap& tl, const ConvTcArgs& a, cudaStream_t st) {
    constexpr int smem = HaloSmem<BN, STAGES, SPLIT>::TOTAL;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(conv3x3_halo_kernel<BN, STAGES, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) {
            set_error("aotb_conv2d_nhwc_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    launch_cluster(conv3x3_halo_kernel<BN, STAGES, SPLIT>, conv_grid(a, BN), dim3(384), smem, st, 1, th, tl, a);
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

extern "C" int aotb_set_conv_grid_cap(int ctas) {
    AOTB_REQUIRE(ctas >= 0, "aotb_set_conv_grid_cap: negative cap");
    tc::g_conv_grid_cap = ctas;
    return AOTB_OK;
}

extern "C" int aotb_set_conv_halo(int mode) {
    AOTB_REQUIRE(mode >= 0 && mode <= 2, "aotb_set_conv_halo: mode is 0, 1 or 2");
    tc::g_conv_halo = mode;
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
    const int const_w = (act & tc::AOTB_CONV_CONST_WEIGHTS) ? 1 : 0;
    act &= ~tc::AOTB_CONV_CONST_WEIGHTS;
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
    a.mtiles = cdiv(a.M, 128);
    const int K = ((KH * KW * Cin + 63) / 64) * 64;   // weights are zero-padded to a multiple of 64 along K
    a.nchunks = K / 64;
    a.act = act;
    a.const_w = const_w;
    // Tile policy: pick the N tile (64 / 128 / 256 dividing Cout) and the split-K cluster size (1 / 2 / 4 / 8) that minimise
    //     split-K (S > 1, one tile per CTA):  T = waves * (ramp + chunks_per_cta * t_chunk[BN] + t_finish[BN])
    //     persistent (S = 1, tpc = ceil(tiles / 132) tiles per CTA):
    //         T = ramp + tpc * chunks * t_chunk[BN] + t_finish[BN] + (tpc - 1) * max(0, chunks * t_mma[BN] + t_finish[BN] - chunks * t_chunk[BN])
    //     t_chunk[BN] = max(kGather, t_mma[BN]),  t_mma[BN] = BN / 64
    // over the 132 SMs of an H100 (one CTA per SM).  Costs are in units of the MMAs of one BN = 64 chunk.  The producer's
    // gather of a chunk (32 KB of fp32 activations) overlaps the MMAs and takes kGather units whatever BN is, so narrow
    // tiles are gather-bound and BN = 256 is MMA-bound.  A persistent CTA pays the ramp once, and the finish of a tile runs
    // while the producer gathers the next tile, so only the part of the consumers' MMAs + finish that exceeds the gather of a
    // tile is added per further tile (the last tile's finish is never hidden).  Split-K is only used to fill a partial wave.
    // kGather was fitted
    // with scripts/conv_sweep.py on an H100 (80GB HBM3, 700 W): over the 20 conv / linear shapes of an R50-AOTL 480p frame
    // the policy's tiles take 632 us in total against 632 us for the best measured tiling of each shape.  Bit 0 of the
    // tuning mask ("narrow") selects the simpler heuristic instead.
    // The single-pass kernel has its own row: one MMA per k-step (a third of the units) and its own gather constant
    // kGather1 (half the shared-memory stores, no lo split), so every tile is gather-bound and the choice turns on waves
    // and finish cost.  Checked with scripts/conv_sweep.py --single-pass on the same card and shapes: the policy's tiles
    // take 478 us against 473 us for the best measured tiling of each shape (the split kernel's policy: 633 us).
    // After the persistent schedule, over the 22 shapes of the sweep (the stem and layer 2's first 1x1 added), the policy's
    // tiles take 664 us (fp32) and 509 us (fp16) against 753 / 582 us before; the split-K picks were left as they were.
    const int mt = cdiv(a.M, 128);
    int BN = 64, best_s = 1;
    const float kGather = 2.5f, kGather1 = 2.0f;
    float best = 1e30f;
    if ((tc::g_conv_tiling & 1) == 0) {
        const int bns[3] = {256, 128, 64};
        const float t_mma[3] = {4.0f, 2.0f, 1.0f}, t_mma1[3] = {4.0f / 3, 2.0f / 3, 1.0f / 3};
        const float t_fin[3] = {8.0f, 4.0f, 2.0f};
        for (int bi = 0; bi < 3; ++bi) {
            // beside 128 accumulator registers the BN = 256 finish reads the residual one column group at a time
            const float tf = t_fin[bi] * (bi == 0 && res ? 2.0f : 1.0f);
            if (Cout % bns[bi]) continue;
            const float tm = split ? t_mma[bi] : t_mma1[bi], tc = fmaxf(split ? kGather : kGather1, tm);
            for (int sp = 1; sp <= 8; sp <<= 1) {
                if (sp > a.nchunks) break;
                const int ctas = mt * (Cout / bns[bi]) * sp;
                const int slots = sp == 8 ? 128 : 132;                        // co-resident CTAs with clusters of sp
                if (sp > 1 && ctas > slots) continue;                         // split-K only to fill a partial wave
                float t;
                if (sp == 1) {
                    const int tpc = cdiv(ctas, 132);
                    t = 3.0f + tpc * a.nchunks * tc + tf + (tpc - 1) * fmaxf(0.f, a.nchunks * (tm - tc) + tf);
                } else {
                    t = cdiv(ctas, slots) * (3.0f + cdiv(a.nchunks, sp) * tc + t_fin[bi]);
                }
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
    if (force_s) {
        AOTB_REQUIRE((force_s == 1 || force_s == 2 || force_s == 4 || force_s == 8) && force_s <= a.nchunks,
                     "aotb_conv2d_nhwc_tc: forced split %d invalid", force_s);
        a.splits = force_s;
    }
    a.spin = (tc::g_conv_tiling & 2) ? 1 : 0;
    a.prof = nullptr;
    a.htx = a.hti = 0;
    // Halo path (conv3x3_halo_kernel) for stride-1 3x3 pad-1 convolutions: 8 x 16 pixel tiles, each input element
    // gathered and split once per 64-channel slice instead of once per tap, never split-K.  Its row of the model, in the
    // same units: the consumers' MMAs bound a tile (the halo of a slice, 46 KB of fp32, is staged under the nine taps of
    // the previous one), and the finish is not hidden, since both consumer warpgroups reach it together:
    //     T = ramp + tpc * (nchunks * t_mma[BN] + t_finish[BN]),   tpc = ceil(pixel tiles * Cout / BN / 132)
    // (single pass: t_mma at least 1).  Fitted with scripts/conv3x3_halo_sweep.py on an H100 80GB HBM3 (700 W), DESIGN 8.
    // The policy takes it when it beats the best tiling of the chunked kernel above, split-K included.  A forced tiling
    // keeps the chunked kernel unless aotb_set_conv_halo(2) forces the halo path (with the forced N tile).
    const bool halo_ok = tc::g_conv_halo && KH == 3 && KW == 3 && stride == 1 && pad == 1 && Cin % 64 == 0 && force_s <= 1 &&
                         (tc::g_conv_tiling & 4) == 0;
    int hBN = BN;
    bool use_halo = false;
    if (halo_ok) {
        a.htx = cdiv(W, 16);
        a.hti = a.htx * cdiv(H, 8);
        float best_h = 1e30f;
        const int bns[3] = {256, 128, 64};
        for (int bi = 0; bi < 3; ++bi) {
            const int bn = bns[bi];
            if (Cout % bn || (force_bn && bn != BN)) continue;
            // single pass: a chunk costs at least one unit whatever its MMAs (the per-chunk waits and the A fragment loads)
            const float tm = split ? bn / 64 : fmaxf(bn / 192.0f, 1.0f), tf = 2.0f * (bn / 64) * (bn == 256 && res ? 2.0f : 1.0f);
            const float th = 3.0f + cdiv(B * a.hti * (Cout / bn), 132) * (a.nchunks * tm + tf);
            if (th < best_h) { best_h = th; hBN = bn; }
        }
        use_halo = tc::g_conv_halo == 2 ||
                   (!force_bn && !force_s && (tc::g_conv_tiling & 1) == 0 && best_h < best);
    }
    if (use_halo) {
        BN = hBN;
        a.splits = 1;
        a.mtiles = B * a.hti;
    }
    if (tc::g_conv_tiling & 4) {      // diagnostic stamps go to the caller's workspace
        const dim3 grid = tc::conv_grid(a, BN);
        const size_t need = (size_t)grid.x * grid.y * grid.z * 12 * sizeof(long long);
        AOTB_REQUIRE(workspace && workspace_bytes >= need, "aotb_conv2d_nhwc_tc: profile mode needs %zu workspace bytes", need);
        a.prof = (long long*)workspace;
    }
    CUtensorMap th, tl;
    int rc;
    if ((rc = tc::make_tmap_weights(&th, wh, K, Cout, BN)) != AOTB_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (use_halo) {
        if (!split) {
            if (BN == 256) return tc::launch_halo<256, 4, false>(th, th, a, st);
            if (BN == 128) return tc::launch_halo<128, 6, false>(th, th, a, st);
            return tc::launch_halo<64, 8, false>(th, th, a, st);
        }
        if ((rc = tc::make_tmap_weights(&tl, wl, K, Cout, BN)) != AOTB_OK) return rc;
        if (BN == 256) return tc::launch_halo<256, 2, true>(th, tl, a, st);
        if (BN == 128) return tc::launch_halo<128, 3, true>(th, tl, a, st);
        return tc::launch_halo<64, 4, true>(th, tl, a, st);
    }
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
