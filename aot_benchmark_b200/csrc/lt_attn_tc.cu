// Long-term attention (K1) on the Hopper tensor cores: fused Q K^T -> softmax -> P V, AOT head shape (H heads x d = 32),
// scores never leave the SM.
//
// Reference computation: MultiheadAttention.forward(use_linear=False), networks/layers/attention.py:82-117,
// called at networks/layers/transformer.py:346 (long-term) and :324 (self-attention, Tk = N).
//
// The kernel is attn_tc.cuh with one 32-channel chunk per query / key row and one value chunk per CTA:
// grid (query tiles, heads, KV splits), splits cut on 128-key boundaries in every layout (tile / groups / ahead / pair).
//
// Precision ("fp16x2"): every fp32 operand x is carried as hi = fp16(x), lo = fp16(x - hi); rows of the
// packed operands are [hi(32) | lo(32)] halfs = 128 bytes (the same bytes as fp32, one TMA swizzle atom).
//   exact mode  S = Qh Kh + Ql Kh + Qh Kl,  O' = (Ph + Pl) [Vh | Vl]  (fp32-faithful)
//   fast mode   S = Qh Kh,                  O' =  Ph       [Vh | Vl]
// and O = O'[:, :32] + O'[:, 32:].  Q is pre-divided by T (true division, attention.py:82) when packed.
#include "attn_tc.cuh"

namespace aotb {
namespace tc {

constexpr int LT_STAGES = 4;

PFN_encodeTiled tensor_map_encoder() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) {
            set_error("cuTensorMapEncodeTiled entry point unavailable");
            return nullptr;
        }
        fn = (PFN_encodeTiled)p;
    }
    return fn;
}

int make_tmap_rows64(CUtensorMap* out, const void* base, int rows, int heads, int box_rows) {
    PFN_encodeTiled fn = tensor_map_encoder();
    if (!fn) return AOTB_ERR_CUDA;
    cuuint64_t dims[3] = {64, (cuuint64_t)rows, (cuuint64_t)heads};
    cuuint64_t strides[2] = {128, (cuuint64_t)rows * 128};  // bytes, dims 1..2
    cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d)", (int)r);
        return AOTB_ERR_CUDA;
    }
    return AOTB_OK;
}

// ------------------------------------------------------------------ operand packing
// src fp32 [rows][ld] (head h at columns h*32) -> dst halfs [H][cap][64] at row offset: [hi(32) | lo(32)]
__global__ void pack_rows64_kernel(const float* __restrict__ src, int ld, __half* __restrict__ dst, int cap, int rows,
                                   int H, int row_off, const int* __restrict__ row_off_dev, float div) {
    pdl_sync();
    const int off = row_off_dev ? *row_off_dev : row_off;
    const size_t total = (size_t)rows * H * 8;  // 4 channels per thread
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c4 = i % 8;
        const int hh = (i / 8) % H;
        const int r = i / (8 * (size_t)H);
        float4 v = *reinterpret_cast<const float4*>(src + (size_t)r * ld + hh * 32 + c4 * 4);
        if (div != 1.f) { v.x = v.x / div; v.y = v.y / div; v.z = v.z / div; v.w = v.w / div; }
        const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
        const __half2 l0 = __floats2half2_rn(v.x - __low2float(h0), v.y - __high2float(h0));
        const __half2 l1 = __floats2half2_rn(v.z - __low2float(h1), v.w - __high2float(h1));
        __half* d = dst + ((size_t)hh * cap + off + r) * 64 + c4 * 4;
        *reinterpret_cast<__half2*>(d) = h0;
        *reinterpret_cast<__half2*>(d + 2) = h1;
        *reinterpret_cast<__half2*>(d + 32) = l0;
        *reinterpret_cast<__half2*>(d + 34) = l1;
    }
}

}  // namespace tc
}  // namespace aotb

using namespace aotb;

// Pack fp32 rows into the split-fp16 operand layout of the tensor-core attention kernel.
// src [rows][ld] fp32, dst [H][cap][64] fp16; written at rows [row_off, row_off+rows) (device counter optional);
// values are divided by `div` first (T for Q -- attention.py:82 -- 1 for K/V).
extern "C" int aotb_tc_pack_rows_f16x2(const float* src, int ld, void* dst, int cap, int rows, int H, int row_off,
                                       const int* row_off_dev, float div, void* stream) {
    AOTB_REQUIRE(src && dst && rows > 0 && H > 0 && ld % 4 == 0 && cap > 0, "aotb_tc_pack_rows_f16x2: bad args");
    AOTB_REQUIRE(row_off_dev || row_off + rows <= cap, "aotb_tc_pack_rows_f16x2: rows exceed capacity");
    const size_t total = (size_t)rows * H * 8;
    int g = (int)((total + 255) / 256);
    if (g > 132 * 8) g = 132 * 8;
    launch(tc::pack_rows64_kernel, dim3(g), dim3(256), 0, (cudaStream_t)stream, src, ld, (__half*)dst, cap, rows, H, row_off,
                                                                row_off_dev, div);
    return check_launch("aotb_tc_pack_rows_f16x2");
}

extern "C" size_t aotb_lt_attn_tc_smem_bytes(void) { return (size_t)tc::AttnSmem<1, 1, tc::LT_STAGES, 64, 2>::TOTAL; }

// The default ("tile") layout's kernel in one mode (exact bit 0), on the current device: resident CTAs per SM, registers per
// thread and local-memory bytes per thread.
extern "C" int aotb_lt_attn_tc_occupancy(int exact, int* ctas_per_sm, int* regs, int* local_bytes) {
    AOTB_REQUIRE(ctas_per_sm && regs && local_bytes, "aotb_lt_attn_tc_occupancy: bad args");
    return tc::attn_tc_occupancy<1, 1, tc::LT_STAGES, 64, 2, false>(exact & 1, ctas_per_sm, regs, local_bytes,
                                                                     "aotb_lt_attn_tc_occupancy");
}

// Qp [H][Nq_cap][64], Kp/Vp [H][kv_cap][64] packed fp16x2 operands (zero-filled beyond the live rows);
// O [N][ldo] fp32 (head h at columns h*32).  splits > 1 writes un-normalised partials
// (Opart [splits][N][H*32], Mpart/Lpart [splits][H][N]) for aotb_attn_merge_f32.
extern "C" int aotb_lt_attn_tc_f16x2(const void* Qp, int Nq_cap, const void* Kp, const void* Vp, int kv_cap, int N,
                                     int Tk, const int* Tk_dev, int H, float* O, int ldo, float* Opart, float* Mpart,
                                     float* Lpart, int splits, int exact, float* dbg, void* stream) {
    AOTB_REQUIRE(Qp && Kp && Vp && N > 0 && H > 0 && (Tk > 0 || Tk_dev) && splits >= 1,
                 "aotb_lt_attn_tc_f16x2: bad args");
    AOTB_REQUIRE(Nq_cap >= ((N + 255) / 256) * 256, "aotb_lt_attn_tc_f16x2: Q buffer must be padded to 256 rows");
    AOTB_REQUIRE(splits == 1 ? (O != nullptr && ldo % 2 == 0) : (Opart && Mpart && Lpart),
                 "aotb_lt_attn_tc_f16x2: output buffers");
    AOTB_REQUIRE(((uintptr_t)Qp | (uintptr_t)Kp | (uintptr_t)Vp) % 128 == 0, "aotb_lt_attn_tc_f16x2: alignment");
    // exact bit 1: "groups" (128-key tiles), bit 3: "ahead" (next scores under this softmax), bit 4: "pair" (64-query CTAs)
    const int groups = (exact >> 1) & 1, ahead = (exact >> 3) & 1, pair = (exact >> 4) & 1;
    AOTB_REQUIRE(groups + ahead + pair <= 1, "aotb_lt_attn_tc_f16x2: at most one layout bit");
    const int BM = pair ? 64 : 128, BK = groups ? 128 : 64;
    CUtensorMap tq, tk, tv;
    int rc;
    if ((rc = tc::make_tmap_rows64(&tq, Qp, Nq_cap, H, BM)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tk, Kp, kv_cap, H, BK)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tv, Vp, kv_cap, H, BK)) != AOTB_OK) return rc;
    tc::AttnTcArgs a;
    a.N = N; a.Tk = Tk; a.Tk_dev = Tk_dev; a.O = O; a.ldo = ldo;
    a.Opart = Opart; a.Mpart = Mpart; a.Lpart = Lpart; a.splits = splits; a.split_unit = 128;
    a.spin = (exact >> 2) & 1; a.dbg = dbg;
    const dim3 grid(cdiv(N, BM), H, splits);
    cudaStream_t st = (cudaStream_t)stream;
    const char* what = "aotb_lt_attn_tc_f16x2";
    if (groups) return tc::launch_attn_tc<1, 1, 2, 128, 2, false>(tq, tk, tv, a, grid, exact & 1, st, what);
    if (ahead) return tc::launch_attn_tc<1, 1, tc::LT_STAGES, 64, 2, true>(tq, tk, tv, a, grid, exact & 1, st, what);
    if (pair) return tc::launch_attn_tc<1, 1, tc::LT_STAGES, 64, 1, false>(tq, tk, tv, a, grid, exact & 1, st, what);
    return tc::launch_attn_tc<1, 1, tc::LT_STAGES, 64, 2, false>(tq, tk, tv, a, grid, exact & 1, st, what);
}

// The long-term attention over a bounded bank cut into its memory slots: split z = keys [z split_rows, (z + 1) split_rows)
// of the live ones, so each split's partial (m, l, O) is slot z's.  Default ("tile") layout only; the exact bits are those
// of aotb_lt_attn_tc_f16x2 (bit 0 exact, bit 2 spin) and a layout bit is refused.
extern "C" int aotb_lt_attn_tc_slots_f16x2(const void* Qp, int Nq_cap, const void* Kp, const void* Vp, int kv_cap, int N,
                                           int Tk, const int* Tk_dev, int H, float* Opart, float* Mpart, float* Lpart,
                                           int splits, int split_rows, int exact, void* stream) {
    AOTB_REQUIRE(Qp && Kp && Vp && N > 0 && H > 0 && (Tk > 0 || Tk_dev) && splits >= 2 && split_rows > 0,
                 "aotb_lt_attn_tc_slots_f16x2: bad args");
    AOTB_REQUIRE(Opart && Mpart && Lpart, "aotb_lt_attn_tc_slots_f16x2: output buffers");
    AOTB_REQUIRE(Tk_dev || Tk <= (long long)splits * split_rows, "aotb_lt_attn_tc_slots_f16x2: more keys than slots");
    AOTB_REQUIRE((exact & ~5) == 0, "aotb_lt_attn_tc_slots_f16x2: only the default layout (exact bits 0 and 2)");
    AOTB_REQUIRE(Nq_cap >= ((N + 255) / 256) * 256, "aotb_lt_attn_tc_slots_f16x2: Q buffer must be padded to 256 rows");
    AOTB_REQUIRE(((uintptr_t)Qp | (uintptr_t)Kp | (uintptr_t)Vp) % 128 == 0, "aotb_lt_attn_tc_slots_f16x2: alignment");
    CUtensorMap tq, tk, tv;
    int rc;
    if ((rc = tc::make_tmap_rows64(&tq, Qp, Nq_cap, H, 128)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tk, Kp, kv_cap, H, 64)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tv, Vp, kv_cap, H, 64)) != AOTB_OK) return rc;
    tc::AttnTcArgs a;
    a.N = N; a.Tk = Tk; a.Tk_dev = Tk_dev; a.O = nullptr; a.ldo = 0;
    a.Opart = Opart; a.Mpart = Mpart; a.Lpart = Lpart; a.splits = splits; a.split_unit = split_rows;
    a.spin = (exact >> 2) & 1; a.dbg = nullptr;
    return tc::launch_attn_tc<1, 1, tc::LT_STAGES, 64, 2, false>(tq, tk, tv, a, dim3(cdiv(N, 128), H, splits), exact & 1,
                                                                 (cudaStream_t)stream, "aotb_lt_attn_tc_slots_f16x2");
}

// n independent long-term (or self-) attentions in one launch, default ("tile") layout.  Problem b reads the query rows
// [b q_stride, b q_stride + N) of Qp [H][q_rows][64] and the key / value rows [b kv_stride, b kv_stride + Tk_b) of Kp / Vp
// [H][kv_rows][64], with Tk_b = Tk_dev[b] (int32 [n]) or Tk for every problem when Tk_dev is null; it writes rows
// [b N, (b + 1) N) of O [n N][ldo], or with splits > 1 of the partials Opart [splits][n N][H*32], Mpart / Lpart
// [splits][H][n N], which aotb_attn_merge_f32 merges over n N rows.  Row b of the result is bit for bit the
// aotb_lt_attn_tc_f16x2 launch on problem b's operands with the same split count: the CTA body is the same, a problem with
// fewer live keys gets empty splits, and keys past a problem's live count are masked whatever the rows there hold.
// exact bits: 0 exact, 2 spin.
extern "C" int aotb_lt_attn_tc_batched_f16x2(const void* Qp, int q_stride, int q_rows, const void* Kp, const void* Vp,
                                             int kv_stride, int kv_rows, int n, int N, int Tk, const int* Tk_dev, int H,
                                             float* O, int ldo, float* Opart, float* Mpart, float* Lpart, int splits,
                                             int exact, void* stream) {
    AOTB_REQUIRE(Qp && Kp && Vp && n >= 1 && N > 0 && H > 0 && (Tk > 0 || Tk_dev) && splits >= 1,
                 "aotb_lt_attn_tc_batched_f16x2: bad args");
    AOTB_REQUIRE(q_stride >= N && (long long)(n - 1) * q_stride + N <= q_rows, "aotb_lt_attn_tc_batched_f16x2: query rows");
    AOTB_REQUIRE(kv_stride > 0 && (long long)n * kv_stride <= kv_rows && (Tk_dev || Tk <= kv_stride),
                 "aotb_lt_attn_tc_batched_f16x2: key rows");
    AOTB_REQUIRE(splits == 1 ? (O != nullptr && ldo % 2 == 0) : (Opart && Mpart && Lpart),
                 "aotb_lt_attn_tc_batched_f16x2: output buffers");
    AOTB_REQUIRE((exact & ~5) == 0, "aotb_lt_attn_tc_batched_f16x2: only the default layout (exact bits 0 and 2)");
    AOTB_REQUIRE(((uintptr_t)Qp | (uintptr_t)Kp | (uintptr_t)Vp) % 128 == 0, "aotb_lt_attn_tc_batched_f16x2: alignment");
    CUtensorMap tq, tk, tv;
    int rc;
    if ((rc = tc::make_tmap_rows64(&tq, Qp, q_rows, H, 128)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tk, Kp, kv_rows, H, 64)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tv, Vp, kv_rows, H, 64)) != AOTB_OK) return rc;
    tc::AttnTcArgs a;
    a.N = N; a.Tk = Tk; a.Tk_dev = Tk_dev; a.O = O; a.ldo = ldo;
    a.Opart = Opart; a.Mpart = Mpart; a.Lpart = Lpart; a.splits = splits; a.split_unit = 128;
    a.spin = (exact >> 2) & 1; a.dbg = nullptr;
    tc::AttnTcBatch bt;
    bt.n = n; bt.qtiles = cdiv(N, 128); bt.q_stride = q_stride; bt.kv_stride = kv_stride;
    return tc::launch_attn_tc_batched<1, 1, tc::LT_STAGES, 64, 2, false>(tq, tk, tv, a, bt, dim3(n * bt.qtiles, H, splits),
                                                                         exact & 1, (cudaStream_t)stream,
                                                                         "aotb_lt_attn_tc_batched_f16x2");
}
