// K loop of the persistent conv chain kernel (conv_chain.cu), plus the pieces the warp-specialised per-layer kernel
// (conv_tc.cu) shares with it.  A 128-pixel x BN-channel output tile is computed by two warpgroups, 64 pixel rows each.
// Per 64-deep K chunk a warpgroup
//   - gathers the fp32 activations of ITS 64 rows straight from NHWC global memory (the caller's load_chunk: im2col is never
//     materialised), splits every value into hi = fp16(x), lo = fp16(x - hi) and stores both 64 x 64 half tiles into the
//     operand stage in the 128B-swizzled K-major layout wgmma expects,
//   - waits for the weights of the chunk (Wh, Wl as [Cout][K] fp16, K-major, loaded by TMA into the same stage),
//   - issues 4 k-steps x (Ah Wh + Al Wh + Ah Wl) as wgmma m64nBNk16 into its register accumulator,
// with three chunks of global loads in flight per thread and the MMAs of chunk c running while chunk c + 1 is converted.
// The stage ring (index g = g0 + local chunk) continues across calls; every stage use is released on s_free exactly once
// (8 warp arrivals) after both warpgroups' MMAs that read it have completed.
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace aotb {
namespace tc {

constexpr int CONV_A_BYTES = 128 * 128;        // one 128 x 64 half tile (both warpgroups' rows)

template <int BN>
__device__ __forceinline__ void wgmma_conv(float* acc, uint64_t a, uint64_t b) {
    if (BN == 256) wgmma_ss_n256(acc, a, b, 1u);
    else if (BN == 128) wgmma_ss_n128(acc, a, b, 1u);
    else wgmma_ss_n64(acc, a, b, 1u);
}

// acc: BN / 2 fp32 per thread, accumulated into (zero it before the first call of a tile).  Stage s occupies
// [Ah | Al | Bh (b_bytes) | Bl (b_bytes)] at smem + s * stage_bytes.  load_chunk(kc, float4 v[8]) loads the 16-byte segment
// q = (tid & 15) of chunk kc of rows wg * 64 + i * 8 + ((tid & 127) >> 4), i = 0..7.
template <int BN, int STAGES, class LoadChunk>
__device__ __forceinline__ void conv_kloop(float* acc, uint8_t* smem, int stage_bytes, int b_bytes, uint64_t* b_full,
                                           uint64_t* s_free, int g0, int nchunks, int kbeg, LoadChunk load_chunk, int spin,
                                           long long* prof) {
    const int t = threadIdx.x & 127, wg = threadIdx.x >> 7, q = t & 15, rsub = t >> 4;
    // byte offset of this thread's 8-byte slot inside the 128 x 64 half tile (128B swizzle; row & 7 == rsub)
    const uint32_t soff = (wg * 64 + rsub) * 128 + (((q >> 1) ^ rsub) << 4) + ((q & 1) << 3);
    const uint64_t dA0 = smem_desc_sw128(smem_u32(smem + wg * 64 * 128));
    const uint64_t dB0 = smem_desc_sw128(smem_u32(smem + 2 * CONV_A_BYTES));
    auto step = [&](int it, const float4* v) {
        const int g = g0 + it, s = g % STAGES;
        uint8_t* Ah = smem + s * stage_bytes + soff;
        uint8_t* Al = Ah + CONV_A_BYTES;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const __half2 h0 = __floats2half2_rn(v[i].x, v[i].y), h1 = __floats2half2_rn(v[i].z, v[i].w);
            const __half2 l0 = __floats2half2_rn(v[i].x - __low2float(h0), v[i].y - __high2float(h0));
            const __half2 l1 = __floats2half2_rn(v[i].z - __low2float(h1), v[i].w - __high2float(h1));
            uint2 ph, pl;
            ph.x = *reinterpret_cast<const uint32_t*>(&h0); ph.y = *reinterpret_cast<const uint32_t*>(&h1);
            pl.x = *reinterpret_cast<const uint32_t*>(&l0); pl.y = *reinterpret_cast<const uint32_t*>(&l1);
            *reinterpret_cast<uint2*>(Ah + i * 1024) = ph;      // row wg*64 + i*8 + rsub
            *reinterpret_cast<uint2*>(Al + i * 1024) = pl;
        }
        fence_proxy_async();      // generic-proxy smem writes -> visible to the tensor core (async proxy)
        asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
        if (prof && threadIdx.x == 0 && it == 0) prof[2] = clock64();
        mbar_wait_cp(&b_full[s], (g / STAGES) & 1, spin);
        if (prof && threadIdx.x == 0 && it == 0) prof[3] = clock64();
        const uint64_t so = (uint64_t)((s * stage_bytes) >> 4);
        const uint64_t ah = dA0 + so, al = ah + (CONV_A_BYTES >> 4), bh = dB0 + so, bl = bh + (uint64_t)(b_bytes >> 4);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            wgmma_conv<BN>(acc, ah + 2 * ks, bh + 2 * ks);
            wgmma_conv<BN>(acc, al + 2 * ks, bh + 2 * ks);
            wgmma_conv<BN>(acc, ah + 2 * ks, bl + 2 * ks);
        }
        wgmma_commit();
        wgmma_wait<1>();                              // the MMAs of the previous chunk have completed: release its stage
        if (it > 0) mbar_arrive_warp(&s_free[(g - 1) % STAGES]);
    };
    float4 v0[8], v1[8], v2[8];
    if (nchunks > 0) load_chunk(kbeg, v0);
    if (nchunks > 1) load_chunk(kbeg + 1, v1);
#pragma unroll 1
    for (int it = 0; it < nchunks; it += 3) {
        if (it + 2 < nchunks) load_chunk(kbeg + it + 2, v2);
        step(it, v0);
        if (it + 1 < nchunks) {
            if (it + 3 < nchunks) load_chunk(kbeg + it + 3, v0);
            step(it + 1, v1);
        }
        if (it + 2 < nchunks) {
            if (it + 4 < nchunks) load_chunk(kbeg + it + 4, v1);
            step(it + 2, v2);
        }
    }
    wgmma_wait<0>();
    reg_fence<BN / 2>(acc);
    if (prof && threadIdx.x == 0) prof[4] = clock64();
    if (nchunks > 0) mbar_arrive_warp(&s_free[(g0 + nchunks - 1) % STAGES]);
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

}  // namespace tc
}  // namespace aotb
