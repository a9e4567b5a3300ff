// A whole chain of convolutions / linears as ONE persistent kernel with tile-level dataflow.
//
// conv_tc.cu launches one kernel per layer: at the sizes of a 480p frame a layer is one or two waves of 128-pixel tiles, so
// every launch pays prologue (barrier init) -> first operand chunk -> K loop -> finish in lockstep on all
// SMs and the next layer cannot start before the last CTA has drained.  The ResNet-50 stages (networks/encoders/resnet.py:34-54,140-157, FrozenBN
// folded) are 52 such launches per frame.  Here the whole chain is a PROGRAM of tiles executed by one CTA per SM:
//
//   program     tiles (layer, m-tile of 128 output pixels, n-tile of BN channels) in layer order, dealt round-robin to the
//               CTAs; every CTA walks its tiles in program order.  A tile names the m-tiles of its input (and residual) layer
//               it reads; `done[layer][m-tile]` counts the finished n-tiles of an m-tile (release / acquire at gpu scope).
//               A tile starts as soon as ITS inputs are complete -- no grid barrier, no launch boundary: layers overlap at
//               tile granularity (a 1x1 conv needs the same m-tile of its input, a 3x3 the neighbouring image rows).
//               Dependencies always point backwards in program order and every CTA executes in program order, so the
//               earliest unfinished tile can always run: no deadlock.
//   roles       288 threads.  warps 0-7: two warpgroups running the K loop of conv_tc.cuh (fp32 NHWC gather -> fp16 hi / lo
//               split -> 128B-swizzled smem -> wgmma into register accumulators, exactly the per-layer kernel's K loop), then
//               the epilogue of the tile; warp 8: TMA producer of the pre-split weights (never waits for a dependency: the
//               weights of the next tile stream in while the activations are still being produced elsewhere).  The operand
//               ring and its mbarrier phases run on across tiles.
//   epilogue    straight from the accumulator fragments (each group of 4 lanes holds 8 consecutive channels of a row: full
//               32-byte sectors): bias + residual + activation, stores -> CTA barrier -> one release-add on done[layer][m-tile].
//   arithmetic  identical to conv_tc.cu: per 64-deep K chunk 4 x (Ah Wh + Al Wh + Ah Wl), fp32 accumulation, same chunk
//               order => bit-identical outputs to the per-layer kernel without split-K.
#include "conv_tc.cuh"
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace aotb {
namespace tc {

struct ChainLayer {                 // device copy of one layer (64-byte aligned array)
    const float* in;
    const float* bias;
    const float* wscale;            // per output channel, null = 1
    const float* res;
    float* out;
    int H, W, Cin, ldin;
    int Ho, Wo, Cout, ldout, ldres;
    int KH, KW, stride, pad;
    int M, nchunks, act, BN;
    int in_done, res_done;          // offset of the producing layer's counters in `done`, -1 = ready before the launch
    int in_need, res_need;          // n-tiles per m-tile of the producing layer
    int done_off;                   // this layer's counters
    int splits;                     // split-K factor S of this layer (1 = none)
    float* scratch;                 // S > 1: raw fp32 partial tiles [S - 1][M][Cout] of splits 0 .. S-2
    int part_off;                   // S > 1: counters [m-tiles * n-tiles] of published partials
    int ntn;                        // n-tiles per m-tile
};
// k0 / k1: chunk range of this work item; split s of S (s == S - 1 finishes the tile: it adds the partials of the others in
// split order, so the result does not depend on which CTA finishes first)
struct ChainTile { int layer, mt, nt, dep_lo, dep_hi, k0, k1, split; };

struct ChainArgs {
    const ChainLayer* layers;
    const ChainTile* tiles;
    const CUtensorMap* tmaps;       // [2 * nlayers]: Wh, Wl
    int* done;
    int ntiles;
    unsigned long long* prof;       // diagnostic (AOTB_CHAIN_PROF=1): 4 globaltimer stamps per work item, or null
    int knock;                      // diagnostic (AOTB_CHAIN_KNOCK, timing only, results wrong): 1 no output stores,
                                    // 4 relaxed instead of release publish, 8 no bias / residual / partial loads
};

constexpr int CH_STAGES = 3, CH_THREADS = 288;
constexpr int CH_B_BYTES = 128 * 128;                      // BN <= 128 rows of 128 B
constexpr int CH_STAGE_BYTES = 2 * CONV_A_BYTES + 2 * CH_B_BYTES;

struct ChRowInfo { int pix_base, iy0, ix0, valid; };

// Dependency counters.  Publishing: the 256 epilogue threads meet at a CTA barrier after their stores, then ONE thread does a
// gpu-scope release-add (the release is cumulative over the writes it has observed through the barrier).  Waiting: ONE thread
// polls with relaxed loads and issues a single gpu-scope acquire fence once the counters are there, then a CTA barrier hands
// the data to the other threads.  (Fencing in every thread, or polling with ld.acquire, would invalidate the SM's L1 at gpu
// scope once per thread.)
__device__ __forceinline__ int ld_relaxed_gpu(const int* p) {
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
    asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// wait until done[lo..hi] >= need (bounded: a protocol bug traps instead of hanging the GPU)
__device__ __forceinline__ void wait_done(const int* done, int lo, int hi, int need) {
    for (int m = lo; m <= hi; ++m) {
        uint32_t spins = 0;
        while (ld_relaxed_gpu(done + m) < need) {
            __nanosleep(64);
            if (++spins > (1u << 23)) __trap();
        }
    }
    fence_acq_rel_gpu();
}
__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// Epilogue of one work item straight from the accumulator fragment: a raw partial (split-K, not the last split) or the
// finished tile (partials of the other splits in split order + own sum, times wscale, bias, residual, activation).  The
// scale is applied to the finished sum only: the raw partials are unscaled.
template <int BN>
__device__ __forceinline__ void chain_epilogue(const ChainArgs& a, const ChainLayer& L, const ChainTile& t, const float* acc) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row0 = t.mt * 128 + (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2), cq = (lane & 3) * 2;
    const int n0 = t.nt * BN, M = L.M, Cout = L.Cout, S = L.splits;
    const bool last = t.split == S - 1, noload = a.knock & 8, nostore = a.knock & 1;
    const size_t plane = (size_t)M * Cout;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = row0 + 8 * h;
        if (m >= M) continue;
#pragma unroll
        for (int g = 0; g < BN / 8; ++g) {
            const int n = n0 + 8 * g + cq, j = 4 * g + 2 * h;
            float2 o = make_float2(acc[j], acc[j + 1]);
            if (!last) {          // raw partial accumulator -> scratch[split][m][n], no bias / residual / activation
                if (!nostore) *reinterpret_cast<float2*>(L.scratch + (size_t)t.split * plane + (size_t)m * Cout + n) = o;
                continue;
            }
            if (S > 1 && !noload) {      // partials of splits 0 .. S-2 first, in split order, then this split's own sum
                float2 p = *reinterpret_cast<const float2*>(L.scratch + (size_t)m * Cout + n);
                for (int s = 1; s < S - 1; ++s) {
                    const float2 q = *reinterpret_cast<const float2*>(L.scratch + (size_t)s * plane + (size_t)m * Cout + n);
                    p.x += q.x; p.y += q.y;
                }
                o.x = p.x + o.x; o.y = p.y + o.y;
            }
            const float2 b2 = (L.bias && !noload) ? *reinterpret_cast<const float2*>(L.bias + n) : make_float2(0.f, 0.f);
            const float2 s2 = (L.wscale && !noload) ? *reinterpret_cast<const float2*>(L.wscale + n) : make_float2(1.f, 1.f);
            const float2 r2 = (L.res && !noload) ? *reinterpret_cast<const float2*>(L.res + (size_t)m * L.ldres + n)
                                                 : make_float2(0.f, 0.f);
            o.x = fmaf(o.x, s2.x, b2.x); o.y = fmaf(o.y, s2.y, b2.y);      // exact product: rounds like o * s + b
            o.x += r2.x; o.y += r2.y;
            o.x = apply_act(o.x, L.act); o.y = apply_act(o.y, L.act);
            if (!nostore) *reinterpret_cast<float2*>(L.out + (size_t)m * L.ldout + n) = o;
        }
    }
}

__global__ void __launch_bounds__(CH_THREADS, 1) conv_chain_kernel(const ChainArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    ChRowInfo* rinfo = reinterpret_cast<ChRowInfo*>(smem + CH_STAGES * CH_STAGE_BYTES);      // [2][128]
    uint64_t* b_full = reinterpret_cast<uint64_t*>(rinfo + 256);
    uint64_t* s_free = b_full + CH_STAGES;

    const int tid = threadIdx.x, warp = tid >> 5;
    pdl_trigger();
    if (tid == 0) {
        for (int s = 0; s < CH_STAGES; ++s) { mbar_init(&b_full[s], 1); mbar_init(&s_free[s], 8); }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();                     // the chain's first input was written by the kernel before this one

    if (warp < 8) {
        // ======================= K loop + epilogue (two warpgroups) =======================
        const int q = tid & 15, rbase = (tid >> 7) * 64 + ((tid & 127) >> 4);   // rows rbase + i*8, i = 0..7
        int g0 = 0, seq = 0;
        for (int ti = blockIdx.x; ti < a.ntiles; ti += gridDim.x, ++seq) {
            const ChainTile t = a.tiles[ti];
            const ChainLayer& L = a.layers[t.layer];
            const float* in = L.in;
            const int H = L.H, W = L.W, Cin = L.Cin, ldin = L.ldin, KW = L.KW, taps = L.KH * L.KW;
            const int kbeg = t.k0, nchunks = t.k1 - t.k0;
            ChRowInfo* ri = rinfo + (seq & 1) * 128;
            if (tid < 128) {
                const int m = t.mt * 128 + tid;
                ChRowInfo r;
                if (m < L.M) {
                    const int oy = m / L.Wo, ox = m - oy * L.Wo;           // batch 1
                    r.pix_base = 0; r.iy0 = oy * L.stride - L.pad; r.ix0 = ox * L.stride - L.pad; r.valid = 1;
                } else {
                    r.pix_base = 0; r.iy0 = 0; r.ix0 = 0; r.valid = 0;
                }
                ri[tid] = r;
            }
            if (tid == 0 && a.prof) a.prof[4 * (size_t)ti] = gtime();
            if (tid == 0 && L.in_done >= 0) wait_done(a.done + L.in_done, t.dep_lo, t.dep_hi, L.in_need);
            if (tid == 0 && a.prof) a.prof[4 * (size_t)ti + 1] = gtime();
            asm volatile("bar.sync 1, 256;" ::: "memory");
            const int cpt = Cin >> 6;                                          // 64-wide chunks per filter tap
            int rowoff[8];                                                     // element offset of the row's pixel, -1 = zero padding
            int cur_tap = -1;
            auto load_chunk = [&](int kc, float4* v) {
                const int tap = kc / cpt, c0 = ((kc - tap * cpt) << 6) + q * 4;
                if (tap != cur_tap) {
                    cur_tap = tap;
                    const bool kvalid = tap < taps;
                    const int ky = tap / KW, kx = tap - ky * KW;
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const ChRowInfo r = ri[rbase + i * 8];
                        const int iy = r.iy0 + ky, ix = r.ix0 + kx;
                        rowoff[i] = (kvalid && r.valid && iy >= 0 && iy < H && ix >= 0 && ix < W) ? (iy * W + ix) * ldin : -1;
                    }
                }
#pragma unroll
                for (int i = 0; i < 8; ++i)        // plain (coherent) loads: the rows were written earlier in THIS launch
                    v[i] = rowoff[i] >= 0 ? *reinterpret_cast<const float4*>(in + rowoff[i] + c0) : make_float4(0.f, 0.f, 0.f, 0.f);
            };
            float acc[64];
#pragma unroll
            for (int j = 0; j < 64; ++j) acc[j] = 0.f;
            if (L.BN == 128) conv_kloop<128, CH_STAGES>(acc, smem, CH_STAGE_BYTES, CH_B_BYTES, b_full, s_free, g0, nchunks, kbeg, load_chunk, 0, nullptr);
            else conv_kloop<64, CH_STAGES>(acc, smem, CH_STAGE_BYTES, CH_B_BYTES, b_full, s_free, g0, nchunks, kbeg, load_chunk, 0, nullptr);
            g0 += nchunks;
            if (tid == 0 && a.prof) a.prof[4 * (size_t)ti + 2] = gtime();
            const bool last = t.split == L.splits - 1;
            int* pcount = a.done + L.part_off + t.mt * L.ntn + t.nt;
            if (last && ((L.res && L.res_done >= 0) || L.splits > 1)) {       // uniform over the 256 threads
                if (tid == 0 && L.res && L.res_done >= 0) wait_done(a.done + L.res_done, t.mt, t.mt, L.res_need);
                if (tid == 0 && L.splits > 1) wait_done(pcount, 0, 0, L.splits - 1);   // the other splits' partial tiles
                asm volatile("bar.sync 1, 256;" ::: "memory");
            }
            if (L.BN == 128) chain_epilogue<128>(a, L, t, acc);
            else chain_epilogue<64>(a, L, t, acc);
            asm volatile("bar.sync 1, 256;" ::: "memory");       // every epilogue thread's stores happen before ...
            if (tid == 0) {                                                                    // ... the gpu-scope release
                int* cnt = last ? a.done + L.done_off + t.mt : pcount;
                if (a.knock & 4) asm volatile("red.relaxed.gpu.global.add.s32 [%0], %1;" ::"l"(cnt), "r"(1) : "memory");
                else red_release_gpu_add(cnt, 1);
            }
            if (tid == 0 && a.prof) a.prof[4 * (size_t)ti + 3] = gtime();
        }
    } else if (warp == 8) {
        // ======================= weight TMA producer =======================
        if (elect_one()) {
            int g0 = 0;
            for (int ti = blockIdx.x; ti < a.ntiles; ti += gridDim.x) {
                const ChainTile t = a.tiles[ti];
                const ChainLayer& L = a.layers[t.layer];
                const CUtensorMap* th = a.tmaps + 2 * t.layer;
                const int nchunks = t.k1 - t.k0, BN = L.BN, n0 = t.nt * BN;
                for (int kc = 0; kc < nchunks; ++kc) {
                    const int g = g0 + kc, s = g % CH_STAGES;
                    if (g >= CH_STAGES) mbar_wait(&s_free[s], ((g / CH_STAGES) - 1) & 1);
                    uint8_t* Bh = smem + s * CH_STAGE_BYTES + 2 * CONV_A_BYTES;
                    mbar_arrive_expect_tx(&b_full[s], 2 * BN * 128);
                    tma_load_2d(Bh, th, &b_full[s], (t.k0 + kc) * 64, n0);
                    tma_load_2d(Bh + CH_B_BYTES, th + 1, &b_full[s], (t.k0 + kc) * 64, n0);
                }
                g0 += nchunks;
            }
        }
    }
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace tc
}  // namespace aotb

using namespace aotb;

// Host-side description of one layer of a chain (caller-owned device pointers, same conventions as aotb_conv2d_nhwc_tc).
// in_layer / res_layer: index (in this array) of the layer that PRODUCES `in` / `res` inside the chain, or -1 when the
// tensor is complete before the chain starts.
struct aotb_chain_layer {
    const float* in;
    const void* wh;
    const void* wl;
    const float* bias;
    const float* wscale;
    const float* res;
    float* out;
    int H, W, Cin, ldin, Cout, ldout, ldres, KH, KW, stride, pad, act, in_layer, res_layer;
};

namespace {
struct ChainPlan {
    std::vector<tc::ChainLayer> layers;
    std::vector<tc::ChainTile> tiles;
    int ndone = 0;
    std::vector<size_t> scratch_floats;          // per layer: floats of its split-K scratch (0 = none)
    size_t off_tiles = 0, off_tmaps = 0, off_done = 0, off_prof = 0, off_scratch = 0, bytes = 0;
};

int plan_chain(const aotb_chain_layer* ls, int n, ChainPlan& P) {
    std::vector<int> mtiles(n), ntn(n);
    for (int i = 0; i < n; ++i) {
        const aotb_chain_layer& l = ls[i];
        AOTB_REQUIRE(l.in && l.wh && l.wl && l.out, "aotb_conv_chain: layer %d: null pointer", i);
        AOTB_REQUIRE(l.Cin % 64 == 0 && l.Cout % 64 == 0, "aotb_conv_chain: layer %d: Cin and Cout must be multiples of 64", i);
        AOTB_REQUIRE(l.ldin % 4 == 0 && l.ldout % 4 == 0 && (!l.res || l.ldres % 4 == 0), "aotb_conv_chain: layer %d: strides", i);
        AOTB_REQUIRE(l.act >= ACT_NONE && l.act <= ACT_RELU6, "aotb_conv_chain: layer %d: activation %d not supported (0-4)", i,
                     l.act);
        AOTB_REQUIRE(l.in_layer < i && l.res_layer < i, "aotb_conv_chain: layer %d: producers must come earlier in the chain", i);
        tc::ChainLayer d{};
        d.in = l.in; d.bias = l.bias; d.wscale = l.wscale; d.res = l.res; d.out = l.out;
        d.H = l.H; d.W = l.W; d.Cin = l.Cin; d.ldin = l.ldin;
        d.Ho = (l.H + 2 * l.pad - l.KH) / l.stride + 1;
        d.Wo = (l.W + 2 * l.pad - l.KW) / l.stride + 1;
        AOTB_REQUIRE(d.Ho > 0 && d.Wo > 0, "aotb_conv_chain: layer %d: empty output", i);
        d.Cout = l.Cout; d.ldout = l.ldout; d.ldres = l.ldres;
        d.KH = l.KH; d.KW = l.KW; d.stride = l.stride; d.pad = l.pad;
        d.M = d.Ho * d.Wo;
        d.nchunks = l.KH * l.KW * l.Cin / 64;
        d.act = l.act;
        d.BN = (l.Cout % 128 == 0) ? 128 : 64;
        mtiles[i] = cdiv(d.M, 128);
        ntn[i] = l.Cout / d.BN;
        d.done_off = P.ndone;
        P.ndone += mtiles[i];
        // split-K: layers with few tiles and a long K loop (the 31x54 maps of ResNet layer3) would leave most SMs idle and put
        // 20+ us of chunks on the dependency chain of every block: cut K into S work items of >= 8 chunks while the layer has
        // fewer than ~one work item per SM
        d.ntn = ntn[i];
        d.splits = 1;
        static int min_chunks = -1, max_split = -1, want_items = -1;
        if (min_chunks < 0) {
            const char* e1 = getenv("AOTB_CHAIN_MINCHUNKS"); min_chunks = e1 ? atoi(e1) : 8;
            const char* e2 = getenv("AOTB_CHAIN_MAXSPLIT"); max_split = e2 ? atoi(e2) : 4;
            const char* e3 = getenv("AOTB_CHAIN_ITEMS"); want_items = e3 ? atoi(e3) : 120;
        }
        while (d.splits < max_split && mtiles[i] * ntn[i] * d.splits < want_items && d.nchunks / (d.splits + 1) >= min_chunks) ++d.splits;
        d.part_off = -1;
        d.scratch = nullptr;
        if (d.splits > 1) {
            d.part_off = P.ndone;
            P.ndone += mtiles[i] * ntn[i];
        }
        P.scratch_floats.push_back(d.splits > 1 ? (size_t)(d.splits - 1) * d.M * d.Cout : 0);
        d.in_done = d.res_done = -1;
        d.in_need = d.res_need = 0;
        if (l.in_layer >= 0) {
            AOTB_REQUIRE(P.layers[l.in_layer].M == l.H * l.W, "aotb_conv_chain: layer %d: input geometry does not match its producer", i);
            d.in_done = P.layers[l.in_layer].done_off; d.in_need = ntn[l.in_layer];
        }
        if (l.res && l.res_layer >= 0) {
            AOTB_REQUIRE(P.layers[l.res_layer].M == d.M, "aotb_conv_chain: layer %d: residual geometry does not match its producer", i);
            d.res_done = P.layers[l.res_layer].done_off; d.res_need = ntn[l.res_layer];
        }
        P.layers.push_back(d);
    }
    for (int i = 0; i < n; ++i) {
        const tc::ChainLayer& d = P.layers[i];
        for (int mt = 0; mt < mtiles[i]; ++mt) {
            const int m0 = mt * 128, m1 = std::min(m0 + 127, d.M - 1);
            int lo, hi;
            if (d.KH == 1 && d.KW == 1 && d.stride == 1 && d.pad == 0) {
                lo = mt; hi = m1 / 128;                                   // the same pixels of the input
            } else {                                                      // every input image row the tile's output rows touch
                const int oy0 = m0 / d.Wo, oy1 = m1 / d.Wo;
                const int iy0 = std::max(0, oy0 * d.stride - d.pad), iy1 = std::min(d.H - 1, oy1 * d.stride - d.pad + d.KH - 1);
                lo = (iy0 * d.W) / 128; hi = (iy1 * d.W + d.W - 1) / 128;
            }
            for (int nt = 0; nt < ntn[i]; ++nt)
                for (int sp = 0; sp < d.splits; ++sp) {             // split sp covers chunks [k0, k1); the last one finishes the tile
                    const int per = cdiv(d.nchunks, d.splits);
                    const int k0 = sp * per, k1 = std::min(d.nchunks, k0 + per);
                    P.tiles.push_back(tc::ChainTile{i, mt, nt, lo, hi, k0, k1, sp});
                }
        }
    }
    P.off_tiles = tc::align_up(P.layers.size() * sizeof(tc::ChainLayer), 256);
    P.off_tmaps = tc::align_up(P.off_tiles + P.tiles.size() * sizeof(tc::ChainTile), 256);
    P.off_done = tc::align_up(P.off_tmaps + 2 * (size_t)n * sizeof(CUtensorMap), 256);
    P.off_prof = P.off_done + tc::align_up((size_t)P.ndone * sizeof(int), 256);
    P.off_scratch = P.off_prof + tc::align_up(P.tiles.size() * 4 * sizeof(unsigned long long), 256);
    size_t fl = 0;
    for (size_t v : P.scratch_floats) fl += tc::align_up(v, 64);
    P.bytes = P.off_scratch + fl * sizeof(float);
    return AOTB_OK;
}

int make_tmap_w(CUtensorMap* out, const void* base, int K, int Cout, int BN) {
    tc::PFN_encodeTiled fn = tc::tensor_map_encoder();
    if (!fn) return AOTB_ERR_CUDA;
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)Cout};
    cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)BN};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(chain weights) failed (%d)", (int)r);
        return AOTB_ERR_CUDA;
    }
    return AOTB_OK;
}
}  // namespace

// Size of the device-resident program of a chain (layer table, tile list, tensor maps, dependency counters).
extern "C" int aotb_conv_chain_plan(const void* layers, int nlayers, size_t* program_bytes, int* ntiles, int* ncounters) {
    AOTB_REQUIRE(layers && nlayers > 0 && program_bytes && ntiles && ncounters, "aotb_conv_chain_plan: bad args");
    ChainPlan P;
    int rc = plan_chain((const aotb_chain_layer*)layers, nlayers, P);
    if (rc != AOTB_OK) return rc;
    *program_bytes = P.bytes; *ntiles = (int)P.tiles.size(); *ncounters = P.ndone;
    return AOTB_OK;
}

// Host-only view of the tile program (tests / diagnostics): 8 ints per work item (layer, m-tile, n-tile, dep_lo, dep_hi, k0, k1,
// split) and 10 per layer (M, BN, counters offset, producer counters offset or -1, residual counters offset or -1, in_need,
// res_need, splits, partial counters offset or -1, chunks).
extern "C" int aotb_conv_chain_dump(const void* layers, int nlayers, int* tiles8, int max_tiles, int* layers10) {
    AOTB_REQUIRE(layers && nlayers > 0 && tiles8 && layers10, "aotb_conv_chain_dump: bad args");
    ChainPlan P;
    int rc = plan_chain((const aotb_chain_layer*)layers, nlayers, P);
    if (rc != AOTB_OK) return rc;
    AOTB_REQUIRE((int)P.tiles.size() <= max_tiles, "aotb_conv_chain_dump: %zu tiles exceed the buffer", P.tiles.size());
    for (size_t i = 0; i < P.tiles.size(); ++i) {
        const tc::ChainTile& t = P.tiles[i];
        int* o = tiles8 + 8 * i;
        o[0] = t.layer; o[1] = t.mt; o[2] = t.nt; o[3] = t.dep_lo; o[4] = t.dep_hi; o[5] = t.k0; o[6] = t.k1; o[7] = t.split;
    }
    for (int i = 0; i < nlayers; ++i) {
        const tc::ChainLayer& d = P.layers[i];
        int* o = layers10 + 10 * i;
        o[0] = d.M; o[1] = d.BN; o[2] = d.done_off; o[3] = d.in_done; o[4] = d.res_done; o[5] = d.in_need; o[6] = d.res_need;
        o[7] = d.splits; o[8] = d.part_off; o[9] = d.nchunks;
    }
    return AOTB_OK;
}

// Write the program into `program` (device memory, >= program_bytes, 256-byte aligned).  Call once per geometry, outside any
// stream capture (it copies from host memory and synchronises the stream).
extern "C" int aotb_conv_chain_build(const void* layers, int nlayers, void* program, size_t program_bytes, void* stream) {
    AOTB_REQUIRE(layers && nlayers > 0 && program && ((uintptr_t)program % 256) == 0, "aotb_conv_chain_build: bad args");
    const aotb_chain_layer* ls = (const aotb_chain_layer*)layers;
    ChainPlan P;
    int rc = plan_chain(ls, nlayers, P);
    if (rc != AOTB_OK) return rc;
    AOTB_REQUIRE(program_bytes >= P.bytes, "aotb_conv_chain_build: program buffer too small (%zu < %zu)", program_bytes, P.bytes);
    {
        size_t fl = 0;
        for (int i = 0; i < nlayers; ++i) {
            if (P.scratch_floats[i]) P.layers[i].scratch = (float*)((uint8_t*)program + P.off_scratch) + fl;
            fl += tc::align_up(P.scratch_floats[i], 64);
        }
    }
    std::vector<uint8_t> host(P.off_scratch, 0);               // the scratch region itself is never initialised
    memcpy(host.data(), P.layers.data(), P.layers.size() * sizeof(tc::ChainLayer));
    memcpy(host.data() + P.off_tiles, P.tiles.data(), P.tiles.size() * sizeof(tc::ChainTile));
    for (int i = 0; i < nlayers; ++i) {
        const int K = ls[i].KH * ls[i].KW * ls[i].Cin;
        CUtensorMap th, tl;
        if ((rc = make_tmap_w(&th, ls[i].wh, K, ls[i].Cout, P.layers[i].BN)) != AOTB_OK) return rc;
        if ((rc = make_tmap_w(&tl, ls[i].wl, K, ls[i].Cout, P.layers[i].BN)) != AOTB_OK) return rc;
        memcpy(host.data() + P.off_tmaps + (2 * (size_t)i) * sizeof(CUtensorMap), &th, sizeof(CUtensorMap));
        memcpy(host.data() + P.off_tmaps + (2 * (size_t)i + 1) * sizeof(CUtensorMap), &tl, sizeof(CUtensorMap));
    }
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemcpyAsync(program, host.data(), P.off_scratch, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
        set_error("aotb_conv_chain_build: %s", cudaGetErrorString(e));
        return AOTB_ERR_CUDA;
    }
    return AOTB_OK;
}

// Byte offset of the diagnostic time stamps (4 x uint64 per work item, written when AOTB_CHAIN_PROF=1) inside a program buffer.
extern "C" size_t aotb_conv_chain_prof_offset(int nlayers, int ntiles, int ncounters) {
    const size_t off_tiles = tc::align_up((size_t)nlayers * sizeof(tc::ChainLayer), 256);
    const size_t off_tmaps = tc::align_up(off_tiles + (size_t)ntiles * sizeof(tc::ChainTile), 256);
    const size_t off_done = tc::align_up(off_tmaps + 2 * (size_t)nlayers * sizeof(CUtensorMap), 256);
    return off_done + tc::align_up((size_t)ncounters * sizeof(int), 256);
}

// Run a built program: clears the dependency counters and launches the persistent kernel (graph-capturable).
extern "C" int aotb_conv_chain_run(void* program, int nlayers, int ntiles, int ncounters, void* stream) {
    AOTB_REQUIRE(program && nlayers > 0 && ntiles > 0 && ncounters > 0, "aotb_conv_chain_run: bad args");
    const size_t off_tiles = tc::align_up((size_t)nlayers * sizeof(tc::ChainLayer), 256);
    const size_t off_tmaps = tc::align_up(off_tiles + (size_t)ntiles * sizeof(tc::ChainTile), 256);
    const size_t off_done = tc::align_up(off_tmaps + 2 * (size_t)nlayers * sizeof(CUtensorMap), 256);
    uint8_t* base = (uint8_t*)program;
    tc::ChainArgs a;
    a.layers = (const tc::ChainLayer*)base;
    a.tiles = (const tc::ChainTile*)(base + off_tiles);
    a.tmaps = (const CUtensorMap*)(base + off_tmaps);
    a.done = (int*)(base + off_done);
    a.ntiles = ntiles;
    static int prof = -1;
    if (prof < 0) { const char* e = getenv("AOTB_CHAIN_PROF"); prof = (e && atoi(e)) ? 1 : 0; }
    a.prof = prof ? (unsigned long long*)(base + off_done + tc::align_up((size_t)ncounters * sizeof(int), 256)) : nullptr;
    static int knock = -1;
    if (knock < 0) { const char* e = getenv("AOTB_CHAIN_KNOCK"); knock = e ? atoi(e) : 0; }
    a.knock = knock;
    cudaStream_t st = (cudaStream_t)stream;
    constexpr int smem = tc::CH_STAGES * tc::CH_STAGE_BYTES + 256 * (int)sizeof(tc::ChRowInfo) + 2 * tc::CH_STAGES * 8 + 1024;
    static bool configured = false;
    static int sms = 0;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(tc::conv_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        int dev = 0;
        if (e == cudaSuccess) e = cudaGetDevice(&dev);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) {
            set_error("aotb_conv_chain_run: %s", cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    cudaError_t e = cudaMemsetAsync(a.done, 0, (size_t)ncounters * sizeof(int), st);
    if (e != cudaSuccess) {
        set_error("aotb_conv_chain_run: memset: %s", cudaGetErrorString(e));
        return AOTB_ERR_CUDA;
    }
    const int grid = ntiles < sms ? ntiles : sms;            // one CTA per SM: all CTAs are co-resident (the dataflow needs it)
    launch(tc::conv_chain_kernel, dim3(grid), dim3(tc::CH_THREADS), smem, st, a);
    return check_launch("aotb_conv_chain_run");
}
