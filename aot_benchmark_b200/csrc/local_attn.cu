// Short-term local-window attention (K2 / K2'), fp32, one warp per (query pixel, head).
//
// Restates MultiheadLocalAttentionV2.forward (networks/layers/attention.py:308-376) and
// LocalGatedPropagation.forward (:789-861) in the form of SURVEY Appendix C -- i.e. the
// reference's own `unfold` definition (:343-348 / :830-835) of what the absent third-party
// spatial_correlation_sampler computes -- without the [1,H,225,N] score tensor, the boolean
// scatter of local2global (:378-417) or the dense N x N matmul (:366-368):
//
//   r[wi]  = relative_emb_k(q)[g*225+wi]            (grouped 1x1 conv + bias on UNSCALED q, :327)
//   s[wi]  = (q/T).k[y+dy,x+dx] + r[wi]             in frame;   r[wi] - 1e8 outside (:355-357)
//   p      = softmax_wi(s)                          225 taps, wi = (dy+7)*15 + (dx+7)
//   o[c]   = sum_wi p[wi] * ( v[y+dy,x+dx][c] + relative_emb_v[g][c][wi] )   (:363-371; no emb_v in DeAOT)
//
// Layout: q,k [HW][ldq/ldk] (head g at columns g*D), v [HW][ldv] (head g at g*DV), out [HW][ldo].
// Phase 1 puts window taps on lanes (each lane owns <= 8 taps and walks the D channels with
// 128-bit loads); phase 2 puts channels on lanes so every tap is one coalesced row read.
#include "common.cuh"
#include "tc_common.cuh"

namespace aotb {

constexpr int LW = 15, LR = 7, LTAPS = 225;

// 16-byte asynchronous global -> shared copy (LDGSTS); bytes = 0 zero-fills the destination (out-of-frame halo positions).  All
// copies of a halo are issued back to back and completed by one wait: the register-staged loop they replace paid one L2 round
// trip per iteration (7 per halo and thread).
__device__ __forceinline__ void cp_async16(float* dst_smem, const float* src, int bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src),
                 "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory"); }

struct LocalArgs {
    const float* q; int ldq;
    const float* k; int ldk;
    const float* v; int ldv;
    const float* relk_w;   // [H*225][D]
    const float* relk_b;   // [H*225]
    const float* relv;     // [H][DV][225] or null
    float* out; int ldo;
    int h, w, H;
    float T;
};

template <int D, int DV, bool HAS_RELV, bool STAGE_WK>
__global__ void __launch_bounds__(256) local_attn_kernel(const LocalArgs p) {
    pdl_sync();
    constexpr int WARPS = 8;
    constexpr int WKS = D + 4;                 // padded row stride of the staged rel-k weights
    extern __shared__ __align__(16) float smem[];
    float* q_raw = smem;                       // [WARPS][D]
    float* q_scl = q_raw + WARPS * D;          // [WARPS][D]
    float* prob = q_scl + WARPS * D;           // [WARPS][232]
    float* wk_s = prob + WARPS * 232;          // [225][WKS]           (STAGE_WK)
    float* relv_s = wk_s + (STAGE_WK ? LTAPS * WKS : 0);  // [DV][225] (HAS_RELV, DV == 32)

    const int g = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int N = p.h * p.w;
    const int qi = blockIdx.x * WARPS + warp;

    if constexpr (STAGE_WK) {
        const float* src = p.relk_w + (size_t)g * LTAPS * D;
        for (int f = threadIdx.x; f < LTAPS * (D / 4); f += blockDim.x) {
            const int r = f / (D / 4), c = (f % (D / 4)) * 4;
            *reinterpret_cast<float4*>(wk_s + r * WKS + c) = __ldg(reinterpret_cast<const float4*>(src + r * D + c));
        }
    }
    if constexpr (HAS_RELV) {
        const float* src = p.relv + (size_t)g * DV * LTAPS;
        for (int f = threadIdx.x; f < DV * LTAPS; f += blockDim.x) relv_s[f] = __ldg(src + f);
    }
    if (qi < N) {
        for (int c = lane; c < D; c += 32) {
            const float x = __ldg(p.q + (size_t)qi * p.ldq + g * D + c);
            q_raw[warp * D + c] = x;
            q_scl[warp * D + c] = x / p.T;   // true division (attention.py:330)
        }
    }
    __syncthreads();
    if (qi >= N) return;

    const int y = qi / p.w, x = qi - y * p.w;
    const float* qr = q_raw + warp * D;
    const float* qs = q_scl + warp * D;

    // ---- phase 1: scores, taps on lanes
    float s[8];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int wi = lane + 32 * j;
        float sc = -INFINITY;
        if (wi < LTAPS) {
            const int dy = wi / LW - LR, dx = wi % LW - LR;
            const int yy = y + dy, xx = x + dx;
            const bool inside = (yy >= 0 && yy < p.h && xx >= 0 && xx < p.w);
            float rel = __ldg(p.relk_b + g * LTAPS + wi);
            float dot = 0.f;
            const float* wrow = STAGE_WK ? (wk_s + wi * WKS) : (p.relk_w + ((size_t)g * LTAPS + wi) * D);
            const float* krow = p.k + (size_t)(inside ? (yy * p.w + xx) : 0) * p.ldk + g * D;
#pragma unroll 4
            for (int c = 0; c < D; c += 4) {
                const float4 qa = *reinterpret_cast<const float4*>(qr + c);
                float4 wv;
                if constexpr (STAGE_WK) wv = *reinterpret_cast<const float4*>(wrow + c);
                else wv = __ldg(reinterpret_cast<const float4*>(wrow + c));
                rel = fmaf(wv.x, qa.x, rel); rel = fmaf(wv.y, qa.y, rel);
                rel = fmaf(wv.z, qa.z, rel); rel = fmaf(wv.w, qa.w, rel);
                if (inside) {
                    const float4 qb = *reinterpret_cast<const float4*>(qs + c);
                    const float4 kv = __ldg(reinterpret_cast<const float4*>(krow + c));
                    dot = fmaf(qb.x, kv.x, dot); dot = fmaf(qb.y, kv.y, dot);
                    dot = fmaf(qb.z, kv.z, dot); dot = fmaf(qb.w, kv.w, dot);
                }
            }
            sc = inside ? (dot + rel) : (rel - 1e8f);
        }
        s[j] = sc;
        mx = fmaxf(mx, sc);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        s[j] = (lane + 32 * j < LTAPS) ? expf(s[j] - mx) : 0.f;
        sum += s[j];
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    float* pw = prob + warp * 232;
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (lane + 32 * j < LTAPS) pw[lane + 32 * j] = s[j] * inv;
    __syncwarp();

    // ---- phase 2: aggregate, channels on lanes
    constexpr int NV = DV / 128 > 0 ? DV / 128 : 1;  // float4 groups per lane when DV >= 128
    if constexpr (DV == 32) {
        float acc = 0.f;
        for (int wi = 0; wi < LTAPS; ++wi) {
            const int dy = wi / LW - LR, dx = wi % LW - LR;
            const int yy = y + dy, xx = x + dx;
            const float pv = pw[wi];
            if (yy >= 0 && yy < p.h && xx >= 0 && xx < p.w)
                acc = fmaf(pv, __ldg(p.v + (size_t)(yy * p.w + xx) * p.ldv + g * DV + lane), acc);
            if constexpr (HAS_RELV) acc = fmaf(pv, relv_s[lane * LTAPS + wi], acc);
        }
        p.out[(size_t)qi * p.ldo + g * DV + lane] = acc;
    } else {
        static_assert(DV == 32 || DV % 128 == 0, "DV");
        static_assert(!HAS_RELV || DV == 32, "relative_emb_v only exists in the AOT head shape");
        float4 acc[NV];
#pragma unroll
        for (int i = 0; i < NV; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int wi = 0; wi < LTAPS; ++wi) {
            const int dy = wi / LW - LR, dx = wi % LW - LR;
            const int yy = y + dy, xx = x + dx;
            if (yy < 0 || yy >= p.h || xx < 0 || xx >= p.w) continue;
            const float pv = pw[wi];
            const float* vrow = p.v + (size_t)(yy * p.w + xx) * p.ldv + g * DV;
#pragma unroll
            for (int i = 0; i < NV; ++i) {
                const float4 vv = __ldg(reinterpret_cast<const float4*>(vrow + i * 128 + lane * 4));
                acc[i].x = fmaf(pv, vv.x, acc[i].x); acc[i].y = fmaf(pv, vv.y, acc[i].y);
                acc[i].z = fmaf(pv, vv.z, acc[i].z); acc[i].w = fmaf(pv, vv.w, acc[i].w);
            }
        }
#pragma unroll
        for (int i = 0; i < NV; ++i)
            *reinterpret_cast<float4*>(p.out + (size_t)qi * p.ldo + g * DV + i * 128 + lane * 4) = acc[i];
    }
}

template <int D, int DV, bool HAS_RELV, bool STAGE_WK>
static int launch_local(const LocalArgs& a, cudaStream_t st) {
    const size_t smem = sizeof(float) * (size_t)(8 * D * 2 + 8 * 232 + (STAGE_WK ? LTAPS * (D + 4) : 0) +
                                                 (HAS_RELV ? DV * LTAPS : 0));
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(local_attn_kernel<D, DV, HAS_RELV, STAGE_WK>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) {
            set_error("aotb_local_attention_f32: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    dim3 grid(cdiv(a.h * a.w, 8), a.H);
    launch(local_attn_kernel<D, DV, HAS_RELV, STAGE_WK>, dim3(grid), dim3(256), smem, st, a);
    return check_launch("aotb_local_attention_f32");
}


// Tiled kernel for the AOT head shape (d_att = d_v = 32): one CTA per (TY x TX query tile, head), 16 warps.
// The per-warp kernel above is bound by shared-memory bandwidth (one LDS per FMA).  Here every operand that is
// reused sits in registers and the other one is a broadcast read:
//   R pass    thread <-> (tap, half of the queries): its relative_emb_k row stays in 32 registers, q comes from
//             shared memory as broadcast float4 reads; writes r[tap] into the score tile.
//   dot pass  thread <-> key position of the 15 x (TX+14) strip under one query row: the key row is read once into
//             32 registers and dotted with the TX queries of the row (position p is tap p-x of query x), then
//             added onto r in the score tile ( -1e8 outside the frame, attention.py:355-357).
//   softmax   warp per query over the padded [15][16] score rows.
//   aggregate warp <-> 3 neighbouring queries, channels on lanes: the 17 value positions and 15 relative_emb_v
//             rows of a window row are loaded once and shared by the 3 queries; probabilities come in as float4.
// The K halo buffer is refilled with V after the dot pass.  relv_t is relative_emb_v transposed to [H][225][32].
template <int TY, int TX>
__global__ void __launch_bounds__(512, 1) local_attn_tile_kernel(const LocalArgs p, const float* __restrict__ relv_t) {
    pdl_sync();
    constexpr int D = 32, HH = TY + 2 * LR, HWD = TX + 2 * LR, NPOS = HH * HWD, LD = 36;
    constexpr int NT = 512, NQ = TY * TX, PLD = LW * 16;
    static_assert(TX % 3 == 0 && TY * (TX / 3) == NT / 32, "aggregate pass: one warp per 3 queries");
    static_assert(LW * HWD <= NT && 2 * LTAPS <= NT && NQ % 2 == 0, "pass mappings");
    extern __shared__ __align__(16) float smem[];
    float* halo = smem;                   // [NPOS][LD]   K, then V
    float* qs = halo + NPOS * LD;         // [NQ][D]
    float* prob = qs + NQ * D;            // [NQ][15][16] scores, then probabilities (slot 15 of each row is padding)
    float* rvs = prob + NQ * PLD;         // [225][D]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tiles_x = (p.w + TX - 1) / TX;
    const int ty0 = (blockIdx.x / tiles_x) * TY, tx0 = (blockIdx.x % tiles_x) * TX;
    const int g = blockIdx.y;

    auto load_halo = [&](const float* src, int ld) {          // asynchronous: complete after cp_async_wait_all() + barrier
        for (int f = tid; f < NPOS * 8; f += NT) {
            const int pos = f >> 3, c4 = (f & 7) * 4;
            const int hy = pos / HWD, hx = pos - hy * HWD;
            const int yy = ty0 - LR + hy, xx = tx0 - LR + hx;
            const bool in = yy >= 0 && yy < p.h && xx >= 0 && xx < p.w;
            cp_async16(halo + pos * LD + c4, in ? src + (size_t)(yy * p.w + xx) * ld + g * D + c4 : src, in ? 16 : 0);
        }
    };
    for (int f = tid; f < NQ * 8; f += NT) {
        const int ql = f >> 3, c4 = (f & 7) * 4;
        const int ly = ql / TX, lx = ql - ly * TX;
        const int y = ty0 + ly, x = tx0 + lx;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (y < p.h && x < p.w) v = __ldg(reinterpret_cast<const float4*>(p.q + (size_t)(y * p.w + x) * p.ldq + g * D + c4));
        *reinterpret_cast<float4*>(qs + ql * D + c4) = v;
    }
    {
        const float* src = relv_t + (size_t)g * LTAPS * D;
        for (int f = tid; f < LTAPS * 8; f += NT) cp_async16(rvs + 4 * f, src + 4 * f, 16);
    }
    load_halo(p.k, p.ldk);
    cp_async_wait_all();
    __syncthreads();

    // ---- R pass: r[tap] = relative_emb_k(q)[tap] on the unscaled q (attention.py:327)
    if (tid < 2 * LTAPS) {
        const int half = tid / LTAPS, tap = tid - half * LTAPS;
        float wk[D];
        const float4* wp = reinterpret_cast<const float4*>(p.relk_w + ((size_t)g * LTAPS + tap) * D);
#pragma unroll
        for (int c = 0; c < D / 4; ++c) {
            const float4 t = __ldg(wp + c);
            wk[4 * c] = t.x; wk[4 * c + 1] = t.y; wk[4 * c + 2] = t.z; wk[4 * c + 3] = t.w;
        }
        const float bias = __ldg(p.relk_b + g * LTAPS + tap);
        const int slot = (tap / LW) * 16 + tap % LW;
#pragma unroll 2
        for (int qi = 0; qi < NQ / 2; ++qi) {
            const int ql = half * (NQ / 2) + qi;
            const float4* q4 = reinterpret_cast<const float4*>(qs + ql * D);
            float r0 = bias, r1 = 0.f;
#pragma unroll
            for (int c = 0; c < D / 4; ++c) {
                const float4 t = q4[c];
                r0 = fmaf(wk[4 * c], t.x, r0); r1 = fmaf(wk[4 * c + 1], t.y, r1);
                r0 = fmaf(wk[4 * c + 2], t.z, r0); r1 = fmaf(wk[4 * c + 3], t.w, r1);
            }
            prob[ql * PLD + slot] = r0 + r1;
        }
    }
    __syncthreads();

    // ---- dot pass: s[tap] = (q . k[pos]) / T + r[tap]  in frame,  r[tap] - 1e8 outside
    if (tid < LW * HWD) {
        const int dy = tid / HWD, hx = tid - dy * HWD;
        const float invT = 1.f / p.T;
        const int xx = tx0 + hx - LR;
        const bool xin = (xx >= 0 && xx < p.w);
#pragma unroll 1
        for (int ly = 0; ly < TY; ++ly) {
            const int yy = ty0 + ly + dy - LR;
            const bool inside = xin && yy >= 0 && yy < p.h;
            float kv[D];
            const float4* kp = reinterpret_cast<const float4*>(halo + ((ly + dy) * HWD + hx) * LD);
#pragma unroll
            for (int c = 0; c < D / 4; ++c) {
                const float4 t = kp[c];
                kv[4 * c] = t.x; kv[4 * c + 1] = t.y; kv[4 * c + 2] = t.z; kv[4 * c + 3] = t.w;
            }
#pragma unroll
            for (int lx = 0; lx < TX; ++lx) {
                const int dx = hx - lx;
                const float4* q4 = reinterpret_cast<const float4*>(qs + (ly * TX + lx) * D);
                float d0 = 0.f, d1 = 0.f;
#pragma unroll
                for (int c = 0; c < D / 4; ++c) {
                    const float4 t = q4[c];
                    d0 = fmaf(kv[4 * c], t.x, d0); d1 = fmaf(kv[4 * c + 1], t.y, d1);
                    d0 = fmaf(kv[4 * c + 2], t.z, d0); d1 = fmaf(kv[4 * c + 3], t.w, d1);
                }
                if (dx >= 0 && dx < LW) {
                    float* sp = prob + (ly * TX + lx) * PLD + dy * 16 + dx;
                    *sp += inside ? (d0 + d1) * invT : -1e8f;
                }
            }
        }
    }
    __syncthreads();          // scores complete; the K halo is dead
    load_halo(p.v, p.ldv);

    // ---- softmax over the 225 taps of each query (padding slots excluded)
    for (int ql = warp; ql < NQ; ql += NT / 32) {
        float* pq = prob + ql * PLD;
        float sc[8];
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i = lane + 32 * j;
            const bool valid = i < PLD && (i & 15) != 15;
            sc[j] = valid ? pq[i] : -INFINITY;
            mx = fmaxf(mx, sc[j]);
        }
        mx = warp_max(mx);
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            sc[j] = expf(sc[j] - mx);         // exp(-inf) = 0 for the padding slots
            sum += sc[j];
        }
        sum = warp_sum(sum);
        const float inv = 1.f / sum;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i = lane + 32 * j;
            if (i < PLD) pq[i] = sc[j] * inv;
        }
    }
    cp_async_wait_all();      // the V halo, requested before the softmax
    __syncthreads();

    // ---- aggregate: o[c] = sum_tap p[tap] * (v[pos][c] + relative_emb_v[tap][c]), channels on lanes
    {
        const int ly = warp / (TX / 3), lx0 = (warp % (TX / 3)) * 3;
        float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
        for (int dy = 0; dy < LW; ++dy) {
            const float* vrow = halo + ((ly + dy) * HWD + lx0) * LD + lane;   // zero outside the frame
            float vv[LW + 2], rr[LW];
#pragma unroll
            for (int j = 0; j < LW + 2; ++j) vv[j] = vrow[j * LD];
#pragma unroll
            for (int dx = 0; dx < LW; ++dx) rr[dx] = rvs[(dy * LW + dx) * D + lane];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const float4* pp = reinterpret_cast<const float4*>(prob + (ly * TX + lx0 + i) * PLD + dy * 16);
                const float4 p0 = pp[0], p1 = pp[1], p2 = pp[2], p3 = pp[3];
                const float pa[16] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w,
                                      p2.x, p2.y, p2.z, p2.w, p3.x, p3.y, p3.z, p3.w};
#pragma unroll
                for (int dx = 0; dx < LW; ++dx) acc[i] = fmaf(pa[dx], vv[i + dx] + rr[dx], acc[i]);
            }
        }
        const int y = ty0 + ly;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const int x = tx0 + lx0 + i;
            if (y < p.h && x < p.w) p.out[(size_t)(y * p.w + x) * p.ldo + g * D + lane] = acc[i];
        }
    }
}

static int launch_local_tile(const LocalArgs& a, const float* relv_t, cudaStream_t st) {
    // 8 x 6 query tiles: 36 tiles x 8 heads = 288 CTAs on the 31 x 54 map = 2.2 waves of 132 SMs
    constexpr int TY = 8, TX = 6;
    const size_t smem = sizeof(float) * (size_t)((TY + 14) * (TX + 14) * 36 + TY * TX * 32 + TY * TX * LW * 16 + LTAPS * 32);
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(local_attn_tile_kernel<TY, TX>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem);
        if (e != cudaSuccess) {
            set_error("aotb_local_attention_tile_f32: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    dim3 grid(cdiv(a.h, TY) * cdiv(a.w, TX), a.H);
    launch(local_attn_tile_kernel<TY, TX>, dim3(grid), dim3(512), smem, st, a, relv_t);
    return check_launch("aotb_local_attention_tile_f32");
}


// Tensor-core kernel for the AOT head shape (d_att = d_v = 32): one CTA per (8 x 16 query tile, head), one warp per query row
// of 16 (the M = 16 of mma.sync.m16n8k16).  The K and V halos (22 x 32 positions, fp32) are staged once by cp.async; then every
// warp walks the 15 window rows dy with an online softmax:
//   R       [16 q] x [32 c] x [16 dx]      dense: unscaled q . relative_emb_k[dy*15 + dx] + bias (dx = 15 is padding)
//   S band  [16 q] x [32 c] x [32 hx]      (q/T) . k over the halo row ly + dy; tap dx = hx - lx, the rest of the band is unused
//   the band goes to the warp's scratch at [lx][dx] and comes back in the accumulator layout of R: s = r + dot (r - 1e8 outside
//   the frame, attention.py:355-357); p = exp(s - m) with the running row max m
//   P relv  [16 q] x [16 dx] x [32 c]      dense: the probabilities straight from the score accumulators
//   P V     [16 q] x [32 hx] x [32 c]      band: P scattered back to [lx][hx] through the scratch (zero off the band)
// Every product is split fp16x2 (hi.hi + lo.hi + hi.lo into fp32, DESIGN 3.1).  The 32-channel contractions assign thread
// (g, j) the channels 8j .. 8j+7 (two float4) as its k slots; the 32 output channels are n = 4 g + n-tile, so the V and relv
// operands are float4 reads and every output row is two float4 stores.  Halo rows use 36 floats: both reads are conflict-free.
constexpr int LTC_TY = 8, LTC_TX = 16, LTC_HH = LTC_TY + 2 * LR, LTC_HW = 32, LTC_LD = 36, LTC_SS = 17;
constexpr size_t LTC_SMEM = sizeof(float) * (size_t)(2 * LTC_HH * LTC_HW * LTC_LD + LTC_TY * 16 * LTC_SS);

__device__ __forceinline__ void split2(float x, float y, uint32_t& hi, uint32_t& lo) {
    hi = tc::cvt_h2(x, y);
    const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    lo = tc::cvt_h2(x - h.x, y - h.y);
}
__device__ __forceinline__ void mma16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// d += A.B in split fp16x2: Ah.Bh + Al.Bh + Ah.Bl
__device__ __forceinline__ void mma_x3(float* d, const uint32_t* ah, const uint32_t* al, const uint32_t* bh, const uint32_t* bl) {
    mma16816(d, ah, bh[0], bh[1]);
    mma16816(d, al, bh[0], bh[1]);
    mma16816(d, ah, bl[0], bl[1]);
}

// One CTA of the tensor-core local attention over the map whose q / k / v / out rows `p` points at.
__device__ __forceinline__ void local_attn_mma_cta(const LocalArgs& p, const float* __restrict__ relv_t) {
    pdl_sync();
    constexpr int TX = LTC_TX, HW = LTC_HW, LD = LTC_LD, SS = LTC_SS, NPOS = LTC_HH * LTC_HW;
    extern __shared__ __align__(16) float smem[];
    float* ks = smem;                     // [22][32][LD]  K halo (zero outside the frame)
    float* vs = ks + NPOS * LD;           // [22][32][LD]  V halo
    const int tid = threadIdx.x, ly = tid >> 5, lane = tid & 31, g4 = lane >> 2, j = lane & 3;
    float* scr = vs + NPOS * LD + ly * 16 * SS;   // [16][SS] this warp's scores / probabilities at [lx][dx]
    const int tiles_x = (p.w + TX - 1) / TX;
    const int ty0 = (blockIdx.x / tiles_x) * LTC_TY, tx0 = (blockIdx.x % tiles_x) * TX;
    const int g = blockIdx.y;

    for (int f = tid; f < NPOS * 8; f += 256) {
        const int pos = f >> 3, c4 = (f & 7) * 4;
        const int yy = ty0 - LR + pos / HW, xx = tx0 - LR + pos % HW;
        const bool in = yy >= 0 && yy < p.h && xx >= 0 && xx < p.w;
        const size_t off = (size_t)(yy * p.w + xx);
        cp_async16(ks + pos * LD + c4, in ? p.k + off * p.ldk + g * 32 + c4 : p.k, in ? 16 : 0);
        cp_async16(vs + pos * LD + c4, in ? p.v + off * p.ldv + g * 32 + c4 : p.v, in ? 16 : 0);
    }

    // q fragments of rows lx = g4 and g4 + 8: unscaled for R, divided by T before the split for the dot (attention.py:330)
    uint32_t qh[2][4], ql[2][4], sh[2][4], sl[2][4];
    {
        const int y = ty0 + ly;
        const float T = p.T;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int x = tx0 + g4 + 8 * r;
            float4 f[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
            if (y < p.h && x < p.w) {
                const float4* src = reinterpret_cast<const float4*>(p.q + (size_t)(y * p.w + x) * p.ldq + g * 32 + 8 * j);
                f[0] = __ldg(src);
                f[1] = __ldg(src + 1);
            }
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                split2(f[kk].x, f[kk].y, qh[kk][r], ql[kk][r]);
                split2(f[kk].z, f[kk].w, qh[kk][r + 2], ql[kk][r + 2]);
                split2(f[kk].x / T, f[kk].y / T, sh[kk][r], sl[kk][r]);
                split2(f[kk].z / T, f[kk].w / T, sh[kk][r + 2], sl[kk][r + 2]);
            }
        }
    }
    cp_async_wait_all();
    __syncthreads();

    const float* wk = p.relk_w + (size_t)g * LTAPS * 32 + 8 * j;
    const float* bk = p.relk_b + g * LTAPS;
    const float* rv = relv_t + (size_t)g * LTAPS * 32 + 4 * g4;
    // this thread's relative_emb_k rows (taps dx = 8 nt + g4), biases (dx = 8 nt + 2 j + e) and relv_t rows (dx = 2 j + (t & 1) +
    // 8 (t >> 1)) of one window row; zero at the padding tap dx = 15.  Loaded one window row ahead, so their L2 latency hides
    // under the MMAs of the current row.
    struct RowOps { float4 wf[2][2]; float b[2][2]; float4 rf[4]; };
    auto load_row = [&](int dy, RowOps& r) {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
            const int dxb = 8 * nt + g4;
            const float4* src = reinterpret_cast<const float4*>(wk + (dy * LW + dxb) * 32);
            r.wf[nt][0] = dxb < LW ? __ldg(src) : z;
            r.wf[nt][1] = dxb < LW ? __ldg(src + 1) : z;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int dx = 8 * nt + 2 * j + e;
                r.b[nt][e] = dx < LW ? __ldg(bk + dy * LW + dx) : 0.f;
            }
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int dx = 2 * j + (t & 1) + 8 * (t >> 1);
            r.rf[t] = dx < LW ? __ldg(reinterpret_cast<const float4*>(rv + (dy * LW + dx) * 32)) : z;
        }
    };
    RowOps nxt;
    load_row(0, nxt);
    float o[4][4] = {};
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll 1
    for (int dy = 0; dy < LW; ++dy) {
        const RowOps cur = nxt;
        if (dy + 1 < LW) load_row(dy + 1, nxt);
        const int hr = ly + dy;
        const int yy = ty0 - LR + hr;
        const bool yin = yy >= 0 && yy < p.h;
        // ---- R: bias + q . relative_emb_k over the taps dx = 8 nt + g4 of this window row
        float s[2][4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                s[nt][e] = cur.b[nt][e];
                s[nt][e + 2] = cur.b[nt][e];
            }
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                const float4 f = cur.wf[nt][kk];
                uint32_t bh[2], bl[2];
                split2(f.x, f.y, bh[0], bl[0]);
                split2(f.z, f.w, bh[1], bl[1]);
                mma_x3(s[nt], qh[kk], ql[kk], bh, bl);
            }
        }
        // ---- S band: (q/T) . k[hx] for the 32 halo positions hx = 8 nt + g4 of halo row hr
        float sb[4][4] = {};
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const float4* kp = reinterpret_cast<const float4*>(ks + (hr * HW + 8 * nt + g4) * LD + 8 * j);
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                const float4 f = kp[kk];
                uint32_t bh[2], bl[2];
                split2(f.x, f.y, bh[0], bl[0]);
                split2(f.z, f.w, bh[1], bl[1]);
                mma_x3(sb[nt], sh[kk], sl[kk], bh, bl);
            }
        }
        // tap dx = hx - lx of row lx: the dot in frame, -1e8 outside
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int lx = g4 + 8 * (i >> 1), hx = 8 * nt + 2 * j + (i & 1), dx = hx - lx;
                const int xx = tx0 - LR + hx;
                if (dx >= 0 && dx < LW) scr[lx * SS + dx] = (yin && xx >= 0 && xx < p.w) ? sb[nt][i] : -1e8f;
            }
        __syncwarp();
        float mx[2] = {m[0], m[1]};
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int lx = g4 + 8 * (i >> 1), dx = 8 * nt + 2 * j + (i & 1);
                s[nt][i] = dx < LW ? s[nt][i] + scr[lx * SS + dx] : -INFINITY;
                mx[i >> 1] = fmaxf(mx[i >> 1], s[nt][i]);
            }
        __syncwarp();
        // ---- online softmax over the taps seen so far (row max and sum shared by the 4 lanes of a row)
        float sc[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            sc[r] = expf(m[r] - mx[r]);
            m[r] = mx[r];
            l[r] *= sc[r];
        }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) o[nt][i] *= sc[i >> 1];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                s[nt][i] = expf(s[nt][i] - m[i >> 1]);          // exp(-inf) = 0 for the padding slot dx = 15
                l[i >> 1] += s[nt][i];
                scr[(g4 + 8 * (i >> 1)) * SS + 8 * nt + 2 * j + (i & 1)] = s[nt][i];
            }
        // ---- P relv: A = P straight from the score accumulators, B = relv_t rows dy*15 + dx, channels 4 g4 .. 4 g4 + 3
        {
            uint32_t ah[4], al[4];
            split2(s[0][0], s[0][1], ah[0], al[0]);
            split2(s[0][2], s[0][3], ah[1], al[1]);
            split2(s[1][0], s[1][1], ah[2], al[2]);
            split2(s[1][2], s[1][3], ah[3], al[3]);
            const float* f0 = &cur.rf[0].x; const float* f1 = &cur.rf[1].x; const float* f2 = &cur.rf[2].x; const float* f3 = &cur.rf[3].x;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                uint32_t bh[2], bl[2];
                split2(f0[nt], f1[nt], bh[0], bl[0]);
                split2(f2[nt], f3[nt], bh[1], bl[1]);
                mma_x3(o[nt], ah, al, bh, bl);
            }
        }
        __syncwarp();
        // ---- P V over the band: A[lx][hx] = P[lx][hx - lx] (zero off the band), B = V halo row hr
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
            uint32_t ah[4], al[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int lx = g4 + 8 * (t & 1), hx = 16 * kk + 2 * j + 8 * (t >> 1);
                const float p0 = (hx - lx >= 0 && hx - lx < 16) ? scr[lx * SS + hx - lx] : 0.f;
                const float p1 = (hx + 1 - lx >= 0 && hx + 1 - lx < 16) ? scr[lx * SS + hx + 1 - lx] : 0.f;
                split2(p0, p1, ah[t], al[t]);
            }
            float4 f[4];
#pragma unroll
            for (int t = 0; t < 4; ++t)
                f[t] = *reinterpret_cast<const float4*>(vs + (hr * HW + 16 * kk + 2 * j + (t & 1) + 8 * (t >> 1)) * LD + 4 * g4);
            const float* f0 = &f[0].x; const float* f1 = &f[1].x; const float* f2 = &f[2].x; const float* f3 = &f[3].x;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                uint32_t bh[2], bl[2];
                split2(f0[nt], f1[nt], bh[0], bl[0]);
                split2(f2[nt], f3[nt], bh[1], bl[1]);
                mma_x3(o[nt], ah, al, bh, bl);
            }
        }
        __syncwarp();
    }
    // ---- normalise and store: row g4 + 8 r holds channels 8 j + 4 e + nt in o[nt][2 r + e]
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
        const int y = ty0 + ly, x = tx0 + g4 + 8 * r;
        if (y < p.h && x < p.w) {
            const float inv = 1.f / l[r];
            float4* dst = reinterpret_cast<float4*>(p.out + (size_t)(y * p.w + x) * p.ldo + g * 32 + 8 * j);
            dst[0] = make_float4(o[0][2 * r] * inv, o[1][2 * r] * inv, o[2][2 * r] * inv, o[3][2 * r] * inv);
            dst[1] = make_float4(o[0][2 * r + 1] * inv, o[1][2 * r + 1] * inv, o[2][2 * r + 1] * inv, o[3][2 * r + 1] * inv);
        }
    }
}

__global__ void __launch_bounds__(256, 1) local_attn_mma_kernel(const LocalArgs p, const float* __restrict__ relv_t) {
    local_attn_mma_cta(p, relv_t);
}

// n maps of h x w pixels stacked along the rows: map b = blockIdx.z is rows [b h w, (b + 1) h w) of q, k, v and out.
__global__ void __launch_bounds__(256, 1) local_attn_mma_batched_kernel(const LocalArgs p, const float* __restrict__ relv_t) {
    const size_t r0 = (size_t)blockIdx.z * p.h * p.w;
    LocalArgs pb = p;
    pb.q += r0 * p.ldq;
    pb.k += r0 * p.ldk;
    pb.v += r0 * p.ldv;
    pb.out += r0 * p.ldo;
    local_attn_mma_cta(pb, relv_t);
}

static int launch_local_tc_batched(const LocalArgs& a, const float* relv_t, int n, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(local_attn_mma_batched_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)LTC_SMEM);
        if (e != cudaSuccess) {
            set_error("aotb_local_attention_tc_batched_f32: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    dim3 grid(cdiv(a.h, LTC_TY) * cdiv(a.w, LTC_TX), a.H, n);
    launch(local_attn_mma_batched_kernel, grid, dim3(256), LTC_SMEM, st, a, relv_t);
    return check_launch("aotb_local_attention_tc_batched_f32");
}

static int launch_local_tc(const LocalArgs& a, const float* relv_t, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(local_attn_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LTC_SMEM);
        if (e != cudaSuccess) {
            set_error("aotb_local_attention_tc_f32: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured = true;
    }
    dim3 grid(cdiv(a.h, LTC_TY) * cdiv(a.w, LTC_TX), a.H);
    launch(local_attn_mma_kernel, grid, dim3(256), LTC_SMEM, st, a, relv_t);
    return check_launch("aotb_local_attention_tc_f32");
}


// Tiled kernel for the DeAOT head shape (1 head, d_att = 128, d_v = 1024, no relative_emb_v; attention.py:789-861): the same
// four passes as local_attn_tile_kernel, with the channel dimensions walked in chunks of 32 through the SAME shared-memory
// halo buffer:
//   scores    for every 32-channel chunk of q / k: the R pass adds q_chunk . relative_emb_k[tap]_chunk (bias with chunk 0) and
//             the dot pass adds q_chunk . k_chunk[pos] / T (the -1e8 of out-of-frame taps with chunk 0) into the score tile;
//   softmax   once;
//   aggregate blockIdx.y selects a group of VC x 32 value channels; for each 32-channel chunk the V halo is staged and every
//             warp accumulates its 3 queries with the channels on lanes.
// The generic per-warp kernel (local_attn_kernel<128, 1024>) re-reads K / V rows from L1 / L2 for every query: 226 us per launch
// at 31 x 54 (19.6 % of the R50-DeAOTL frame).  Here a CTA re-computes the scores of its query tile for its channel group
// (VC = 8: 4 groups of 256 channels -> 144 CTAs, one wave) and reads every halo row once per chunk.
// One CTA of the tiled DeAOT local attention over the map whose q / k / v / out rows `p` points at (taken by value: passed by
// reference, the one-map kernel schedules differently).
template <int TY, int TX, int KC, int VC>
__device__ __forceinline__ void local_gated_tile_cta(const LocalArgs p) {
    pdl_sync();
    constexpr int C = 32, HH = TY + 2 * LR, HWD = TX + 2 * LR, NPOS = HH * HWD, LD = 36;
    constexpr int NT = 512, NQ = TY * TX, PLD = LW * 16, DQ = KC * C;
    static_assert(TX % 3 == 0 && TY * (TX / 3) == NT / 32, "aggregate pass: one warp per 3 queries");
    static_assert(LW * HWD <= NT && 2 * LTAPS <= NT && NQ % 2 == 0, "pass mappings");
    extern __shared__ __align__(16) float smem[];
    float* halo = smem;                   // [NPOS][LD]   one 32-channel chunk of K, later of V
    float* qs = halo + NPOS * LD;         // [NQ][DQ]
    float* prob = qs + NQ * DQ;           // [NQ][15][16] scores, then probabilities (slot 15 of each row is padding)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tiles_x = (p.w + TX - 1) / TX;
    const int ty0 = (blockIdx.x / tiles_x) * TY, tx0 = (blockIdx.x % tiles_x) * TX;
    const int cg = blockIdx.y;            // value-channel group

    auto load_halo = [&](const float* src, int ld, int c0) {   // asynchronous: complete after cp_async_wait_all() + barrier
        for (int f = tid; f < NPOS * 8; f += NT) {
            const int pos = f >> 3, c4 = (f & 7) * 4;
            const int hy = pos / HWD, hx = pos - hy * HWD;
            const int yy = ty0 - LR + hy, xx = tx0 - LR + hx;
            const bool in = yy >= 0 && yy < p.h && xx >= 0 && xx < p.w;
            cp_async16(halo + pos * LD + c4, in ? src + (size_t)(yy * p.w + xx) * ld + c0 + c4 : src, in ? 16 : 0);
        }
    };
    for (int f = tid; f < NQ * (DQ / 4); f += NT) {
        const int ql = f / (DQ / 4), c4 = (f % (DQ / 4)) * 4;
        const int ly = ql / TX, lx = ql - ly * TX;
        const int y = ty0 + ly, x = tx0 + lx;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (y < p.h && x < p.w) v = __ldg(reinterpret_cast<const float4*>(p.q + (size_t)(y * p.w + x) * p.ldq + c4));
        *reinterpret_cast<float4*>(qs + ql * DQ + c4) = v;
    }
    load_halo(p.k, p.ldk, 0);
    cp_async_wait_all();
    __syncthreads();

    // ---- R pass: r[tap] = relative_emb_k(q)[tap] on the unscaled q (attention.py:814-816), all chunks
    if (tid < 2 * LTAPS) {
        const int half = tid / LTAPS, tap = tid - half * LTAPS;
        const float bias = __ldg(p.relk_b + tap);
        const int slot = (tap / LW) * 16 + tap % LW;
#pragma unroll 1
        for (int kc = 0; kc < KC; ++kc) {
            float wk[C];
            const float4* wp = reinterpret_cast<const float4*>(p.relk_w + (size_t)tap * DQ + kc * C);
#pragma unroll
            for (int c = 0; c < C / 4; ++c) {
                const float4 t = __ldg(wp + c);
                wk[4 * c] = t.x; wk[4 * c + 1] = t.y; wk[4 * c + 2] = t.z; wk[4 * c + 3] = t.w;
            }
#pragma unroll 2
            for (int qi = 0; qi < NQ / 2; ++qi) {
                const int ql = half * (NQ / 2) + qi;
                const float4* q4 = reinterpret_cast<const float4*>(qs + ql * DQ + kc * C);
                float r0 = kc == 0 ? bias : prob[ql * PLD + slot], r1 = 0.f;
#pragma unroll
                for (int c = 0; c < C / 4; ++c) {
                    const float4 t = q4[c];
                    r0 = fmaf(wk[4 * c], t.x, r0); r1 = fmaf(wk[4 * c + 1], t.y, r1);
                    r0 = fmaf(wk[4 * c + 2], t.z, r0); r1 = fmaf(wk[4 * c + 3], t.w, r1);
                }
                prob[ql * PLD + slot] = r0 + r1;
            }
        }
    }
    __syncthreads();

    // ---- dot pass per 32-channel chunk: s[tap] += (q_chunk . k_chunk[pos]) / T in frame;  r[tap] - 1e8 outside (:844)
#pragma unroll 1
    for (int kc = 0; kc < KC; ++kc) {
        if (kc > 0) {
            load_halo(p.k, p.ldk, kc * C);
            cp_async_wait_all();
            __syncthreads();
        }
        if (tid < LW * HWD) {
            const int dy = tid / HWD, hx = tid - dy * HWD;
            const float invT = 1.f / p.T;
            const int xx = tx0 + hx - LR;
            const bool xin = (xx >= 0 && xx < p.w);
#pragma unroll 1
            for (int ly = 0; ly < TY; ++ly) {
                const int yy = ty0 + ly + dy - LR;
                const bool inside = xin && yy >= 0 && yy < p.h;
                float kv[C];
                const float4* kp = reinterpret_cast<const float4*>(halo + ((ly + dy) * HWD + hx) * LD);
#pragma unroll
                for (int c = 0; c < C / 4; ++c) {
                    const float4 t = kp[c];
                    kv[4 * c] = t.x; kv[4 * c + 1] = t.y; kv[4 * c + 2] = t.z; kv[4 * c + 3] = t.w;
                }
#pragma unroll
                for (int lx = 0; lx < TX; ++lx) {
                    const int dx = hx - lx;
                    const float4* q4 = reinterpret_cast<const float4*>(qs + (ly * TX + lx) * DQ + kc * C);
                    float d0 = 0.f, d1 = 0.f;
#pragma unroll
                    for (int c = 0; c < C / 4; ++c) {
                        const float4 t = q4[c];
                        d0 = fmaf(kv[4 * c], t.x, d0); d1 = fmaf(kv[4 * c + 1], t.y, d1);
                        d0 = fmaf(kv[4 * c + 2], t.z, d0); d1 = fmaf(kv[4 * c + 3], t.w, d1);
                    }
                    if (dx >= 0 && dx < LW) {
                        float* sp = prob + (ly * TX + lx) * PLD + dy * 16 + dx;
                        if (inside) *sp += (d0 + d1) * invT;
                        else if (kc == 0) *sp += -1e8f;
                    }
                }
            }
        }
        __syncthreads();      // this chunk of the K halo is dead
    }
    load_halo(p.v, p.ldv, (cg * VC) * C);      // first V chunk, overlapped with the softmax below

    // ---- softmax over the 225 taps of each query (padding slots excluded)
    for (int ql = warp; ql < NQ; ql += NT / 32) {
        float* pq = prob + ql * PLD;
        float sc[8];
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i = lane + 32 * j;
            const bool valid = i < PLD && (i & 15) != 15;
            sc[j] = valid ? pq[i] : -INFINITY;
            mx = fmaxf(mx, sc[j]);
        }
        mx = warp_max(mx);
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            sc[j] = expf(sc[j] - mx);         // exp(-inf) = 0 for the padding slots
            sum += sc[j];
        }
        sum = warp_sum(sum);
        const float inv = 1.f / sum;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i = lane + 32 * j;
            if (i < PLD) pq[i] = sc[j] * inv;
        }
    }
    cp_async_wait_all();      // the first V chunk, requested before the softmax
    __syncthreads();

    // ---- aggregate: o[c] = sum_tap p[tap] * v[pos][c], channels on lanes, one 32-channel chunk at a time
    const int ly = warp / (TX / 3), lx0 = (warp % (TX / 3)) * 3;
#pragma unroll 1
    for (int vc = 0; vc < VC; ++vc) {
        if (vc > 0) {
            __syncthreads();                  // everybody is done with the previous chunk
            load_halo(p.v, p.ldv, (cg * VC + vc) * C);
            cp_async_wait_all();
            __syncthreads();
        }
        float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
        for (int dy = 0; dy < LW; ++dy) {
            const float* vrow = halo + ((ly + dy) * HWD + lx0) * LD + lane;   // zero outside the frame
            float vv[LW + 2];
#pragma unroll
            for (int j = 0; j < LW + 2; ++j) vv[j] = vrow[j * LD];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const float4* pp = reinterpret_cast<const float4*>(prob + (ly * TX + lx0 + i) * PLD + dy * 16);
                const float4 p0 = pp[0], p1 = pp[1], p2 = pp[2], p3 = pp[3];
                const float pa[16] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w,
                                      p2.x, p2.y, p2.z, p2.w, p3.x, p3.y, p3.z, p3.w};
#pragma unroll
                for (int dx = 0; dx < LW; ++dx) acc[i] = fmaf(pa[dx], vv[i + dx], acc[i]);
            }
        }
        const int y = ty0 + ly;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const int x = tx0 + lx0 + i;
            if (y < p.h && x < p.w) p.out[(size_t)(y * p.w + x) * p.ldo + (cg * VC + vc) * C + lane] = acc[i];
        }
    }
}

template <int TY, int TX, int KC, int VC>
__global__ void __launch_bounds__(512, 1) local_gated_tile_kernel(const LocalArgs p) {
    local_gated_tile_cta<TY, TX, KC, VC>(p);
}

// n maps of h x w pixels stacked along the rows: map b = blockIdx.z is rows [b h w, (b + 1) h w) of q, k, v and out.
template <int TY, int TX, int KC, int VC>
__global__ void __launch_bounds__(512, 1) local_gated_tile_batched_kernel(const LocalArgs p) {
    const size_t r0 = (size_t)blockIdx.z * p.h * p.w;
    LocalArgs pb = p;
    pb.q += r0 * p.ldq;
    pb.k += r0 * p.ldk;
    pb.v += r0 * p.ldv;
    pb.out += r0 * p.ldo;
    local_gated_tile_cta<TY, TX, KC, VC>(pb);
}

// the tiling of the DeAOT tile kernels: d_att = 128 in KC = 4 chunks; 1024 value channels = 4 groups of VC = 8 chunks
constexpr int LGT_TY = 8, LGT_TX = 6, LGT_KC = 4, LGT_VC = 8;
constexpr size_t LGT_SMEM = sizeof(float) * (size_t)((LGT_TY + 14) * (LGT_TX + 14) * 36 + LGT_TY * LGT_TX * LGT_KC * 32 +
                                                     LGT_TY * LGT_TX * LW * 16);

// n = 0: the one-map kernel; n >= 1: the batched kernel over n maps
static int launch_local_gated_tile(const LocalArgs& a, int n, cudaStream_t st) {
    auto k1 = local_gated_tile_kernel<LGT_TY, LGT_TX, LGT_KC, LGT_VC>;
    auto kn = local_gated_tile_batched_kernel<LGT_TY, LGT_TX, LGT_KC, LGT_VC>;
    const char* what = n ? "aotb_local_gated_tile_batched_f32" : "aotb_local_gated_tile_f32";
    static bool configured[2] = {false, false};
    if (!configured[n ? 1 : 0]) {
        cudaError_t e = cudaFuncSetAttribute(n ? kn : k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LGT_SMEM);
        if (e != cudaSuccess) {
            set_error("%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
            return AOTB_ERR_CUDA;
        }
        configured[n ? 1 : 0] = true;
    }
    dim3 grid(cdiv(a.h, LGT_TY) * cdiv(a.w, LGT_TX), 1024 / (LGT_VC * 32), n ? n : 1);
    launch(n ? kn : k1, grid, dim3(512), LGT_SMEM, st, a);
    return check_launch(what);
}

}  // namespace aotb

using namespace aotb;

extern "C" int aotb_local_attention_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                        const float* relk_w, const float* relk_b, const float* relv, float* out,
                                        int ldo, int h, int w, int H, int d_att, int d_v, void* stream) {
    AOTB_REQUIRE(q && k && v && relk_w && relk_b && out && h > 0 && w > 0 && H > 0,
                 "aotb_local_attention_f32: bad args");
    AOTB_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0, "aotb_local_attention_f32: ld %% 4");
    LocalArgs a;
    a.q = q; a.ldq = ldq; a.k = k; a.ldk = ldk; a.v = v; a.ldv = ldv;
    a.relk_w = relk_w; a.relk_b = relk_b; a.relv = relv; a.out = out; a.ldo = ldo;
    a.h = h; a.w = w; a.H = H; a.T = sqrtf((float)d_att);
    cudaStream_t st = (cudaStream_t)stream;
    if (d_att == 32 && d_v == 32 && relv) return launch_local<32, 32, true, true>(a, st);
    if (d_att == 128 && d_v == 1024 && !relv) return launch_local<128, 1024, false, false>(a, st);
    set_error("aotb_local_attention_f32: unsupported head shape d_att=%d d_v=%d relv=%d", d_att, d_v, relv != nullptr);
    return AOTB_ERR_UNSUPPORTED;
}

// Tiled kernel for the AOT head shape (d_att = d_v = 32).  relv_t = relative_emb_v transposed to [H][225][32].
extern "C" int aotb_local_attention_tile_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                             const float* relk_w, const float* relk_b, const float* relv_t, float* out,
                                             int ldo, int h, int w, int H, void* stream) {
    AOTB_REQUIRE(q && k && v && relk_w && relk_b && relv_t && out && h > 0 && w > 0 && H > 0,
                 "aotb_local_attention_tile_f32: bad args");
    AOTB_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0, "aotb_local_attention_tile_f32: ld %% 4");
    LocalArgs a;
    a.q = q; a.ldq = ldq; a.k = k; a.ldk = ldk; a.v = v; a.ldv = ldv;
    a.relk_w = relk_w; a.relk_b = relk_b; a.relv = nullptr; a.out = out; a.ldo = ldo;
    a.h = h; a.w = w; a.H = H; a.T = sqrtf(32.f);
    return launch_local_tile(a, relv_t, (cudaStream_t)stream);
}

// Tensor-core kernel for the AOT head shape: the arguments of aotb_local_attention_tile_f32.
extern "C" int aotb_local_attention_tc_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                           const float* relk_w, const float* relk_b, const float* relv_t, float* out,
                                           int ldo, int h, int w, int H, void* stream) {
    AOTB_REQUIRE(q && k && v && relk_w && relk_b && relv_t && out && h > 0 && w > 0 && H > 0,
                 "aotb_local_attention_tc_f32: bad args");
    AOTB_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0, "aotb_local_attention_tc_f32: ld %% 4");
    AOTB_REQUIRE(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)relk_w | (uintptr_t)relv_t | (uintptr_t)out) % 16 == 0,
                 "aotb_local_attention_tc_f32: q, k, v, relk_w, relv_t and out must be 16-byte aligned");
    LocalArgs a;
    a.q = q; a.ldq = ldq; a.k = k; a.ldk = ldk; a.v = v; a.ldv = ldv;
    a.relk_w = relk_w; a.relk_b = relk_b; a.relv = nullptr; a.out = out; a.ldo = ldo;
    a.h = h; a.w = w; a.H = H; a.T = sqrtf(32.f);
    return launch_local_tc(a, relv_t, (cudaStream_t)stream);
}

// Tiled kernel for the DeAOT head shape (one head, d_att = 128, d_v = 1024, no relative_emb_v): networks/layers/attention.py:789-861.
extern "C" int aotb_local_gated_tile_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                         const float* relk_w, const float* relk_b, float* out, int ldo, int h, int w,
                                         void* stream) {
    AOTB_REQUIRE(q && k && v && relk_w && relk_b && out && h > 0 && w > 0, "aotb_local_gated_tile_f32: bad args");
    AOTB_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0, "aotb_local_gated_tile_f32: ld %% 4");
    LocalArgs a;
    a.q = q; a.ldq = ldq; a.k = k; a.ldk = ldk; a.v = v; a.ldv = ldv;
    a.relk_w = relk_w; a.relk_b = relk_b; a.relv = nullptr; a.out = out; a.ldo = ldo;
    a.h = h; a.w = w; a.H = 1; a.T = sqrtf(128.f);
    return launch_local_gated_tile(a, 0, (cudaStream_t)stream);
}

// n maps of h x w pixels stacked along the rows of q, k, v and out (map b = rows [b h w, (b + 1) h w)); map b's output is bit
// for bit aotb_local_attention_tc_f32 on its rows.
extern "C" int aotb_local_attention_tc_batched_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                                   const float* relk_w, const float* relk_b, const float* relv_t, float* out,
                                                   int ldo, int h, int w, int H, int n, void* stream) {
    AOTB_REQUIRE(q && k && v && relk_w && relk_b && relv_t && out && h > 0 && w > 0 && H > 0 && n >= 1 && n <= 65535,
                 "aotb_local_attention_tc_batched_f32: bad args");
    AOTB_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0, "aotb_local_attention_tc_batched_f32: ld %% 4");
    AOTB_REQUIRE(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)relk_w | (uintptr_t)relv_t | (uintptr_t)out) % 16 == 0,
                 "aotb_local_attention_tc_batched_f32: q, k, v, relk_w, relv_t and out must be 16-byte aligned");
    LocalArgs a;
    a.q = q; a.ldq = ldq; a.k = k; a.ldk = ldk; a.v = v; a.ldv = ldv;
    a.relk_w = relk_w; a.relk_b = relk_b; a.relv = nullptr; a.out = out; a.ldo = ldo;
    a.h = h; a.w = w; a.H = H; a.T = sqrtf(32.f);
    return launch_local_tc_batched(a, relv_t, n, (cudaStream_t)stream);
}

// n maps of h x w pixels stacked along the rows of q, k, v and out (map b = rows [b h w, (b + 1) h w)); map b's output is bit
// for bit aotb_local_gated_tile_f32 on its rows.
extern "C" int aotb_local_gated_tile_batched_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                                 const float* relk_w, const float* relk_b, float* out, int ldo, int h, int w,
                                                 int n, void* stream) {
    AOTB_REQUIRE(q && k && v && relk_w && relk_b && out && h > 0 && w > 0 && n >= 1 && n <= 65535,
                 "aotb_local_gated_tile_batched_f32: bad args");
    AOTB_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0, "aotb_local_gated_tile_batched_f32: ld %% 4");
    LocalArgs a;
    a.q = q; a.ldq = ldq; a.k = k; a.ldk = ldk; a.v = v; a.ldv = ldv;
    a.relk_w = relk_w; a.relk_b = relk_b; a.relv = nullptr; a.out = out; a.ldo = ldo;
    a.h = h; a.w = w; a.H = 1; a.T = sqrtf(128.f);
    return launch_local_gated_tile(a, n, (cudaStream_t)stream);
}
