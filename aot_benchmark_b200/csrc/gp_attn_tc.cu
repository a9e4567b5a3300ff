// DeAOT long-term attention (GatedPropagation, K1') fused on the Hopper tensor cores: Q K^T -> softmax -> P V.
//
// Reference computation: GatedPropagation.forward, networks/layers/attention.py:672-704, as DeAOT instantiates it
// (1 head, d_qk = 128, d_v = 1024: networks/layers/transformer.py:541-548): softmax((Q / T) K^T) V over the memory bank.
//
// The kernel is attn_tc.cuh with four 32-channel chunks per query / key row (d_qk = 128) and two value chunks (64 of the
// 1024 value channels) per CTA: grid (query tiles of 128, d_v slices of 64, KV splits), splits cut on 64-key boundaries.
// O' = 128 x 1024 fp32 does not fit one CTA's registers, so every slice recomputes Q K^T; a 64-channel slice keeps the
// per-thread accumulators (2 x 32 for O', 32 for S, 32 for P) within the register file at 288 threads.
#include "attn_tc.cuh"

namespace aotb {
namespace tc {
constexpr int GP_VC = 2, GP_STAGES = 2;
}  // namespace tc
}  // namespace aotb

using namespace aotb;

// Qp [4][Nq_cap][64], Kp [4][kv_cap][64], Vp [dv/32][kv_cap][64]: split-fp16 rows packed by aotb_tc_pack_rows_f16x2 with
// one "head" per 32 channels (Q divided by T = sqrt(128) when packed).  O [N][ldo] fp32.  splits > 1 writes un-normalised
// partials (Opart [splits][N][dv], Mpart / Lpart [splits][1][N]) for aotb_attn_merge_f32 (H = 1, d_v = dv).
extern "C" int aotb_gp_attn_tc_f16x2(const void* Qp, int Nq_cap, const void* Kp, const void* Vp, int kv_cap, int N, int Tk,
                                     const int* Tk_dev, int dv, float* O, int ldo, float* Opart, float* Mpart,
                                     float* Lpart, int splits, int exact, void* stream) {
    AOTB_REQUIRE(Qp && Kp && Vp && N > 0 && (Tk > 0 || Tk_dev) && splits >= 1 && dv > 0 && dv % 128 == 0,
                 "aotb_gp_attn_tc_f16x2: bad args");
    AOTB_REQUIRE(Nq_cap >= ((N + 127) / 128) * 128, "aotb_gp_attn_tc_f16x2: Q buffer must be padded to 128 rows");
    AOTB_REQUIRE(splits == 1 ? (O != nullptr && ldo % 2 == 0) : (Opart && Mpart && Lpart),
                 "aotb_gp_attn_tc_f16x2: output buffers");
    AOTB_REQUIRE(((uintptr_t)Qp | (uintptr_t)Kp | (uintptr_t)Vp) % 128 == 0, "aotb_gp_attn_tc_f16x2: alignment");
    CUtensorMap tq, tk, tv;
    int rc;
    if ((rc = tc::make_tmap_rows64(&tq, Qp, Nq_cap, 4, 128)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tk, Kp, kv_cap, 4, 64)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tv, Vp, kv_cap, dv / 32, 64)) != AOTB_OK) return rc;
    tc::AttnTcArgs a;
    a.N = N; a.Tk = Tk; a.Tk_dev = Tk_dev; a.O = O; a.ldo = ldo;
    a.Opart = Opart; a.Mpart = Mpart; a.Lpart = Lpart; a.splits = splits; a.split_unit = 64;
    a.spin = (exact >> 2) & 1; a.dbg = nullptr;
    return tc::launch_attn_tc<4, tc::GP_VC, tc::GP_STAGES, 64, 2, false>(tq, tk, tv, a, dim3(cdiv(N, 128), dv / (32 * tc::GP_VC), splits),
                                                           exact & 1, (cudaStream_t)stream, "aotb_gp_attn_tc_f16x2");
}

// The same attention over a bounded bank cut into its memory slots: split z = keys [z split_rows, (z + 1) split_rows) of the
// live ones (see aotb_lt_attn_tc_slots_f16x2).
extern "C" int aotb_gp_attn_tc_slots_f16x2(const void* Qp, int Nq_cap, const void* Kp, const void* Vp, int kv_cap, int N,
                                           int Tk, const int* Tk_dev, int dv, float* Opart, float* Mpart, float* Lpart,
                                           int splits, int split_rows, int exact, void* stream) {
    AOTB_REQUIRE(Qp && Kp && Vp && N > 0 && (Tk > 0 || Tk_dev) && splits >= 2 && split_rows > 0 && dv > 0 && dv % 128 == 0,
                 "aotb_gp_attn_tc_slots_f16x2: bad args");
    AOTB_REQUIRE(Opart && Mpart && Lpart, "aotb_gp_attn_tc_slots_f16x2: output buffers");
    AOTB_REQUIRE(Tk_dev || Tk <= (long long)splits * split_rows, "aotb_gp_attn_tc_slots_f16x2: more keys than slots");
    AOTB_REQUIRE((exact & ~5) == 0, "aotb_gp_attn_tc_slots_f16x2: exact bits 0 and 2 only");
    AOTB_REQUIRE(Nq_cap >= ((N + 127) / 128) * 128, "aotb_gp_attn_tc_slots_f16x2: Q buffer must be padded to 128 rows");
    AOTB_REQUIRE(((uintptr_t)Qp | (uintptr_t)Kp | (uintptr_t)Vp) % 128 == 0, "aotb_gp_attn_tc_slots_f16x2: alignment");
    CUtensorMap tq, tk, tv;
    int rc;
    if ((rc = tc::make_tmap_rows64(&tq, Qp, Nq_cap, 4, 128)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tk, Kp, kv_cap, 4, 64)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tv, Vp, kv_cap, dv / 32, 64)) != AOTB_OK) return rc;
    tc::AttnTcArgs a;
    a.N = N; a.Tk = Tk; a.Tk_dev = Tk_dev; a.O = nullptr; a.ldo = 0;
    a.Opart = Opart; a.Mpart = Mpart; a.Lpart = Lpart; a.splits = splits; a.split_unit = split_rows;
    a.spin = (exact >> 2) & 1; a.dbg = nullptr;
    return tc::launch_attn_tc<4, tc::GP_VC, tc::GP_STAGES, 64, 2, false>(
        tq, tk, tv, a, dim3(cdiv(N, 128), dv / (32 * tc::GP_VC), splits), exact & 1, (cudaStream_t)stream,
        "aotb_gp_attn_tc_slots_f16x2");
}

// n independent DeAOT attentions in one launch (the batched form of aotb_gp_attn_tc_f16x2, as aotb_lt_attn_tc_batched_f16x2 is
// of the AOT kernel).  Problem b reads the query rows [b q_stride, b q_stride + N) of Qp [4][q_rows][64] and the key / value
// rows [b kv_stride, b kv_stride + Tk_b) of Kp [4][kv_rows][64] / Vp [dv/32][kv_rows][64], with Tk_b = Tk_dev[b] (int32 [n])
// or Tk for every problem when Tk_dev is null; it writes rows [b N, (b + 1) N) of O [n N][ldo], or with splits > 1 of the
// partials Opart [splits][n N][dv], Mpart / Lpart [splits][1][n N], which aotb_attn_merge_f32 (H = 1, d_v = dv) merges over
// n N rows.  Row b of the result is bit for bit the aotb_gp_attn_tc_f16x2 launch on problem b's operands with the same split
// count.  exact bits: 0 exact, 2 spin.
extern "C" int aotb_gp_attn_tc_batched_f16x2(const void* Qp, int q_stride, int q_rows, const void* Kp, const void* Vp,
                                             int kv_stride, int kv_rows, int n, int N, int Tk, const int* Tk_dev, int dv,
                                             float* O, int ldo, float* Opart, float* Mpart, float* Lpart, int splits,
                                             int exact, void* stream) {
    AOTB_REQUIRE(Qp && Kp && Vp && n >= 1 && N > 0 && (Tk > 0 || Tk_dev) && splits >= 1 && dv > 0 && dv % 128 == 0,
                 "aotb_gp_attn_tc_batched_f16x2: bad args");
    AOTB_REQUIRE(q_stride >= N && (long long)(n - 1) * q_stride + N <= q_rows, "aotb_gp_attn_tc_batched_f16x2: query rows");
    AOTB_REQUIRE(kv_stride > 0 && (long long)n * kv_stride <= kv_rows && (Tk_dev || Tk <= kv_stride),
                 "aotb_gp_attn_tc_batched_f16x2: key rows");
    AOTB_REQUIRE(splits == 1 ? (O != nullptr && ldo % 2 == 0) : (Opart && Mpart && Lpart),
                 "aotb_gp_attn_tc_batched_f16x2: output buffers");
    AOTB_REQUIRE((exact & ~5) == 0, "aotb_gp_attn_tc_batched_f16x2: exact bits 0 and 2 only");
    AOTB_REQUIRE(((uintptr_t)Qp | (uintptr_t)Kp | (uintptr_t)Vp) % 128 == 0, "aotb_gp_attn_tc_batched_f16x2: alignment");
    CUtensorMap tq, tk, tv;
    int rc;
    if ((rc = tc::make_tmap_rows64(&tq, Qp, q_rows, 4, 128)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tk, Kp, kv_rows, 4, 64)) != AOTB_OK) return rc;
    if ((rc = tc::make_tmap_rows64(&tv, Vp, kv_rows, dv / 32, 64)) != AOTB_OK) return rc;
    tc::AttnTcArgs a;
    a.N = N; a.Tk = Tk; a.Tk_dev = Tk_dev; a.O = O; a.ldo = ldo;
    a.Opart = Opart; a.Mpart = Mpart; a.Lpart = Lpart; a.splits = splits; a.split_unit = 64;
    a.spin = (exact >> 2) & 1; a.dbg = nullptr;
    tc::AttnTcBatch bt;
    bt.n = n; bt.qtiles = cdiv(N, 128); bt.q_stride = q_stride; bt.kv_stride = kv_stride;
    return tc::launch_attn_tc_batched<4, tc::GP_VC, tc::GP_STAGES, 64, 2, false>(
        tq, tk, tv, a, bt, dim3(n * bt.qtiles, dv / (32 * tc::GP_VC), splits), exact & 1, (cudaStream_t)stream,
        "aotb_gp_attn_tc_batched_f16x2");
}
