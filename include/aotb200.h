/* libaotb200.so -- C ABI of the H100-native AOT/DeAOT mask-propagation hot path.
 *
 * The reference (yoxu515/aot-benchmark @601c138) is pure Python/PyTorch and has no FFI of its
 * own (SURVEY 8b); this is the boundary the drop-in Python engines bind with ctypes, and the one
 * a reference maintainer would bind (INTEGRATION.md shows the stub).  Each entry point replaces
 * the reference code cited beside it (paths relative to the reference root).
 *
 * Conventions: every pointer is a caller-owned DEVICE pointer (fp32 unless noted) obtained from
 * torch tensors via data_ptr(); no allocation, no host sync, no exceptions; `stream` is a
 * cudaStream_t (launch is capturable in a CUDA graph); returns 0 or a negative error code,
 * message via aotb_last_error_string().  Activations are NHWC / [rows][ld] row-major; an `ld*`
 * argument is the row (pixel) stride in elements so kernels can address channel slices.
 * Activation codes: 0 none, 1 ReLU, 2 GELU(erf), 3 SiLU, 4 ReLU6.
 */
#ifndef AOTB200_H
#define AOTB200_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

int aotb_version(void);
const char* aotb_arch(void);
const char* aotb_last_error_string(void);
/* kernels launched by this library in this process so far (bench.py reports the delta). */
unsigned long long aotb_launch_count(void);
/* Launch every kernel with programmatic dependent launch (prologues overlap the previous kernel's tail). */
void aotb_set_pdl(int on);
/* Tuning / diagnostic mask of aotb_conv2d_nhwc_tc (default 0); results are identical up to fp32 summation order.
 *   bit 0: the pre-cost-model heuristic (N = 64 tiles unless a wider tile fills the GPU on its own) instead of the
 *          fitted cost model over N tile x split-K cluster size;
 *   bit 1: mbarrier waits spin without the suspend hint;
 *   bit 2: every CTA writes clock64 stamps to `workspace` as long long[ctas][12]: 0 start, 1 prologue done, 2 first A
 *          stage stored, 3 first stage consumable, 4 accumulator (of the last tile) complete, 5 producer done, 7 exit;
 *          split-K launches: 6 tile staged, 8 tile visible to the finish (cluster barrier), 9 finish stored;
 *          persistent launches: 10 accumulator of the first tile complete, 8 finish of the first tile stored (the first
 *          tile boundary on the consumer side), 9 finish of the last tile stored, 11 the CTA's tile count (not a clock);
 *   bits 4-7: force the N tile (1 = 64, 2 = 128; 0 = policy); bits 8-11: force the split-K factor
 *          (1, 2, 4, 8; 0 = policy).  Forced values that do not divide the problem are an argument error. */
int aotb_set_conv_tiling(int mode);
/* Upper bound on the CTAs of a persistent (split-K free) aotb_conv2d_nhwc_tc launch; 0 (default) = one per SM.  The tile
 * order is static, so the output does not depend on the cap. */
int aotb_set_conv_grid_cap(int ctas);
/* Stride-1 3x3 pad-1 aotb_conv2d_nhwc_tc launches without split-K whose Cin is a multiple of 64 may run on the halo
 * kernel: 8 x 16 pixel tiles whose input halo is staged once per 64-channel slice.  mode 1 (default): when the tile model
 * favours it and aotb_set_conv_tiling forces no tiling; 0: never (every launch on the chunked kernel, to compare the two); 2: every such launch. */
int aotb_set_conv_halo(int mode);

/* nn.Conv2d (+ folded FrozenBatchNorm2d, + residual, + activation) as im2col-free implicit GEMM.
 * networks/encoders/resnet.py:34-54,140-157; networks/layers/normalization.py:30-43;
 * networks/models/aot.py:19-21,83; networks/decoders/fpn.py:34-58.
 * in [B][H][W][ldin], w [KH*KW*Cin][Cout], out [B][Ho][Wo][ldout], res like out with ldres.
 * act: 0 none, 1 ReLU, 2 exact GELU, 3 SiLU, 4 ReLU6, 5 h_swish = v * relu6(v + 3) / 6 (networks/encoders/mobilenetv3.py:33-48,
 * true division by 6).  h_swish is taken by this conv, aotb_linear_f32, aotb_dwconv_nhwc_f32 and aotb_gate_scale_f32; the
 * tensor-core conv and GroupNorm accept 0-4 only. */
int aotb_conv2d_nhwc_f32(const float* in, const float* w, const float* bias, const float* res, float* out,
                         int B, int H, int W, int Cin, int ldin, int Cout, int ldout, int ldres,
                         int KH, int KW, int stride, int pad, int dil, int act, void* stream);

/* Same contract as aotb_conv2d_nhwc_f32 (dilation 1) on the Hopper tensor cores (wgmma) through split-fp16 operands:
 * wh / wl are the weights pre-split as hi = fp16(w'), lo = fp16(w' - hi), laid out [Cout][KH*KW*Cin] (K-major, K ordered
 * (ky,kx,ci), zero-padded to a multiple of 64); activations are split on the fly.  out = act(wscale * acc + bias + res):
 * wscale [Cout] (NULL = 1, 16-byte aligned like bias) undoes a per-output-channel power-of-two normalisation
 * w' = w / wscale (ops.split_fp16_scaled picks 2^13 <= max_k |w'[k][n]| < 2^14).
 * Precision: lo cannot go below the fp16 subnormal spacing 2^-24, so each split operand x carries an absolute error of up
 * to 2^-25 on top of a relative 2^-22.  The normalisation takes that floor off the weights, whose products then stay
 * within ~1e-6 of fp32 for channels of any magnitude.  Activations are split as they come: elements with |x| below about
 * 2^-3 lose relative precision, and |x| >= 65520 overflows hi (inf).
 * wl == NULL selects the single-pass kernel: activations are rounded once to hi = fp16(x), only wh is read, and each
 * k-step issues one MMA (Ah Wh) instead of three.  Every product then carries fp16 rounding of both operands (2^-11
 * relative; the weight normalisation still gives any channel scale that precision), accumulated in fp32.  The finish and
 * the range are those of the split kernel; the tile policy has its own cost-model row for it.
 * act may carry AOTB_CONV_CONST_WEIGHTS: the caller promises that no earlier kernel in the stream (or graph) writes wh / wl,
 * so the kernel requests its first weight tiles before it waits for the previous kernel (programmatic dependent launch).
 * Model weights packed once qualify; operand copies that kernels of the same frame refresh (memory-bank keys) do not.
 * Without split-K the launch is persistent: one CTA per SM walks the 128-pixel x BN output tiles in a static order and
 * gathers the next tile's operands while it finishes the current one.
 * Requires Cin % 4 == 0 and Cout % 64 == 0.  Few-tile deep-K layers run split-K: the 2 / 4 / 8 CTAs of one output
 * tile form a thread-block cluster and sum their partial tiles over distributed shared memory in rank order
 * (deterministic).  `workspace` / `workspace_bytes` are only used by the diagnostic mode of aotb_set_conv_tiling
 * (may be NULL / 0 otherwise). */
#define AOTB_CONV_CONST_WEIGHTS 256
int aotb_conv2d_nhwc_tc(const float* in, const void* wh, const void* wl, const float* bias, const float* wscale,
                        const float* res, float* out, int B, int H, int W, int Cin, int ldin, int Cout, int ldout, int ldres,
                        int KH, int KW, int stride, int pad, int act, void* workspace, size_t workspace_bytes,
                        void* stream);

/* nn.Linear on tokens: out[M][N] = act(in[M][K] @ wt[K][N] + bias + res).
 * networks/layers/transformer.py:321-367,582-665; networks/layers/attention.py:76-79,119,710,858. */
int aotb_linear_f32(const float* in, const float* wt, const float* bias, const float* res, float* out,
                    int M, int K, int ldin, int N, int ldout, int ldres, int act, void* stream);

/* Layout changes at the API edge (callers hand NCHW images, read NCHW features). */
int aotb_nchw_to_nhwc_f32(const float* in, float* out, int B, int C, int HW, void* stream);
int aotb_nhwc_to_nchw_f32(const float* in, float* out, int B, int C, int HW, void* stream);
/* [3][HW] image -> [HW][4] NHWC with a zero 4th channel (16-byte pixels for the stem convolution). */
int aotb_image_to_nhwc4_f32(const float* in, float* out, int HW, void* stream);
/* The same for B images stacked densely: [B][3][HW] -> [B][HW][4]; image b equals a one-image launch on image b. */
int aotb_image_to_nhwc4_batched_f32(const float* in, float* out, int B, int HW, void* stream);

/* nn.MaxPool2d(3, 2, 1): networks/encoders/resnet.py:79,146. */
int aotb_maxpool3x3s2_nhwc_f32(const float* in, float* out, int B, int H, int W, int C, void* stream);

/* Depthwise conv, w [KH*KW][C]: networks/layers/basic.py:15-57 (5x5 of the FFN / gated propagation),
 * networks/encoders/mobilenetv2.py:93-101 (3x3 + folded BN + ReLU6). */
int aotb_dwconv_nhwc_f32(const float* in, const float* w, const float* bias, float* out, int B, int H, int W,
                         int C, int ldin, int ldout, int KH, int KW, int stride, int pad, int dil, int act,
                         void* stream);

/* F.interpolate(mode="bilinear", align_corners=...): networks/decoders/fpn.py:45-54. */
int aotb_bilinear_nhwc_f32(const float* in, float* out, int B, int H, int W, int C, int Ho, int Wo,
                           int align_corners, void* stream);

/* Strided element-wise: op 0 copy, 1 a+b, 2 a*b, 3 silu(a), 4 silu(a)*b, 5 fill(scalar).
 * networks/layers/attention.py:585-586,707,855; networks/layers/transformer.py:602-611,625-626. */
int aotb_eltwise_f32(int op, const float* a, int lda, const float* b, int ldb, float* out, int ldo,
                     int rows, int cols, float scalar, void* stream);

/* nn.LayerNorm(C) per row; if out2 != NULL also out2 = LN(x) + add (with_pos_embed,
 * networks/layers/transformer.py:305-310,321-322). */
int aotb_layernorm_f32(const float* x, int ldx, const float* gamma, const float* beta, const float* add,
                       int ldadd, float* out, int ldo, float* out2, int ldo2, int rows, int C, void* stream);

/* Swin (shifted-)window multi-head self-attention core, batch 1 (BASELINE config 4 encoder):
 * WindowAttention.forward networks/encoders/swin/swin_transformer.py:158-196 fused with the zero padding, cyclic
 * shift, window partition / reverse and crop of SwinTransformerBlock.forward :273-316 and the shifted-window mask of
 * BasicLayer.forward :416-438.  qkv [H*W][ldqkv] = the qkv Linear applied to the UN-padded norm1 output, columns
 * [q(C) | k(C) | v(C)], head h = columns h*32..h*32+31 of each; qkv_bias [3C] stands in for padded positions (the
 * reference pads after norm1, so a padded token's q/k/v are the bias); rel_bias [heads][49][49] =
 * relative_position_bias_table[relative_position_index] permuted (:176-183); out [H*W][ldo] = softmax(q k^T / sqrt(32)
 * + rel_bias + mask) v per head, heads concatenated, before `proj`.  window must be 7, C == heads * 32. */
int aotb_window_attention_f32(const float* qkv, int ldqkv, const float* qkv_bias, const float* rel_bias, float* out,
                              int ldo, int H, int W, int C, int heads, int window, int shift, void* stream);
/* The same for B token maps stacked densely: qkv [B*H*W][ldqkv], out [B*H*W][ldo]; padding, shift, mask and crop are
 * per image, and image b equals a one-image launch on image b bit for bit. */
int aotb_window_attention_batched_f32(const float* qkv, int ldqkv, const float* qkv_bias, const float* rel_bias, float* out,
                                      int ldo, int B, int H, int W, int C, int heads, int window, int shift, void* stream);

/* PatchMerging gather (swin_transformer.py:339-360): x [H*W][ldx] (C channels) -> out [ceil(H/2)*ceil(W/2)][ldo] with
 * 4C channels ordered [(0,0) | (1,0) | (0,1) | (1,1)] of each 2x2 block, zeros outside H x W. */
int aotb_patch_merge_f32(const float* x, int ldx, float* out, int ldo, int H, int W, int C, void* stream);
/* The same for B maps stacked densely: x [B*H*W][ldx] -> out [B*ceil(H/2)*ceil(W/2)][ldo], zero padding per image. */
int aotb_patch_merge_batched_f32(const float* x, int ldx, float* out, int ldo, int B, int H, int W, int C, void* stream);

/* nn.GroupNorm(G, C) over [B][P pixels][C] + activation: networks/layers/basic.py:6-12,18,30-32,75-85.  The workspace
 * (aotb_groupnorm_workspace_bytes(B, G) bytes, reusable for any smaller G) must be zero-filled before its first use: it holds
 * the launch counter with which the last block of the statistics kernel finalises (mean, rstd) once, in a fixed order. */
size_t aotb_groupnorm_workspace_bytes(int B, int G);
int aotb_groupnorm_nhwc_f32(const float* x, int ldx, const float* gamma, const float* beta, float* out, int ldo,
                            int B, int P, int C, int G, int act, void* workspace, void* stream);

/* Split attention of ResNeSt (SplAtConv2d after its grouped conv + bn0 + ReLU, cardinality 1), one image:
 * networks/encoders/resnest/splat.py:88-105,118-132.  x [HW][ldx] holds `radix` splits of C channels (split r = channels
 * [r*C, (r+1)*C)); gap = mean over pixels of the sum of the splits, h = ReLU(gap @ w1 + b1) with w1 [C][inter] / b1 [inter] = fc1
 * with bn1 folded, logits = h @ w2 + b2 with w2 [inter][radix*C] / b2 [radix*C] = fc2, att [radix*C] = softmax over r of
 * logits[r*C + c] (radix-major, as rSoftMax writes it).  C % 4 == 0, C <= 512, inter <= 512, 2 <= radix <= 4.  The pixel sums are
 * per-CTA partials in the workspace, added in CTA order by the CTA that finishes last (deterministic).  The workspace
 * (aotb_splat_workspace_bytes(C) bytes, reusable for any smaller C) must be zero-filled before its first use: it holds the launch
 * counter, which every launch leaves at zero again (graph replays start from the same state). */
size_t aotb_splat_workspace_bytes(int C);
int aotb_splat_attention_f32(const float* x, int ldx, int HW, int C, int radix, const float* w1, const float* b1, int inter,
                             const float* w2, const float* b2, float* att, void* workspace, void* stream);
/* out [Ho][Wo][ldo] = sum_r att[r*C + c] * x[r*C + c] (splat.py:107-113), one image x [H][W][ldx].  pool_stride > 0 also applies the
 * avd pool nn.AvgPool2d(3, pool_stride, padding=1) (padding counted; networks/encoders/resnest/resnet.py:72-73,152-153), so the
 * full-resolution sum is never written; pool_stride 0: Ho = H, Wo = W. */
int aotb_splat_combine_f32(const float* x, int ldx, const float* att, float* out, int ldo, int H, int W, int C, int radix,
                           int pool_stride, void* stream);
/* Squeeze-excite gate of one image (networks/encoders/mobilenetv3.py:51-65): x [HW][ldx] (C channels), gap = mean over the
 * pixels, h = ReLU(gap @ w1 + b1) with w1 [C][inter], gate [C] = h_sigmoid(h @ w2 + b2) with w2 [inter][C].  C % 4 == 0,
 * C <= 1024, inter <= 1024.  The same deterministic multi-CTA reduction as aotb_splat_attention_f32, on a workspace of
 * aotb_splat_workspace_bytes(C) bytes, zero-filled before its first use and left with a zero counter by every launch. */
int aotb_se_gate_f32(const float* x, int ldx, int HW, int C, const float* w1, const float* b1, int inter, const float* w2,
                     const float* b2, float* gate, void* workspace, void* stream);
/* out [HW][ldo] = act(gate[c] * x[HW][ldx]) over C channels (the SE product, then the block's activation). */
int aotb_gate_scale_f32(const float* x, int ldx, const float* gate, float* out, int ldo, int HW, int C, int act, void* stream);
/* Batched forms of the four kernels above: B images stacked densely over pixels (x [B][HW][ldx], out [B][Ho*Wo][ldo]),
 * att / gate [B][radix*C].  Every image keeps its own CTA partials and launch counter (reduced in CTA order, as in the
 * one-image launch), so image b equals a one-image launch on image b bit for bit.  The workspace of the two reductions is
 * aotb_splat_workspace_batched_bytes(C, B) bytes (B = 1: aotb_splat_workspace_bytes(C)), zero-filled before its first use
 * and left with zero counters by every launch. */
size_t aotb_splat_workspace_batched_bytes(int C, int B);
int aotb_splat_attention_batched_f32(const float* x, int ldx, int B, int HW, int C, int radix, const float* w1, const float* b1,
                                     int inter, const float* w2, const float* b2, float* att, void* workspace, void* stream);
int aotb_splat_combine_batched_f32(const float* x, int ldx, const float* att, float* out, int ldo, int B, int H, int W, int C,
                                   int radix, int pool_stride, void* stream);
int aotb_se_gate_batched_f32(const float* x, int ldx, int B, int HW, int C, const float* w1, const float* b1, int inter,
                             const float* w2, const float* b2, float* gate, void* workspace, void* stream);
int aotb_gate_scale_batched_f32(const float* x, int ldx, const float* gate, float* out, int ldo, int B, int HW, int C, int act,
                                void* stream);
/* nn.AvgPool2d(k, s, pad, ceil_mode, count_include_pad) in NHWC, in [B][H][W][ldin] -> out [B][Ho][Wo][ldo] with PyTorch's
 * output extent and divisor rules: networks/encoders/resnest/resnet.py:330-342 (avg_down). */
int aotb_avgpool_nhwc_f32(const float* in, int ldin, float* out, int ldo, int B, int H, int W, int C, int k, int s, int pad,
                          int ceil_mode, int count_include_pad, void* stream);

/* softmax((Q/T) K^T) V per head, scores never materialised (fp32 reference-precision path).
 * networks/layers/attention.py:82-117 (MultiheadAttention) and :672-704 (GatedPropagation).
 * Tk_dev (optional) is a device int holding the live key count.  With Mout/Lout the kernel writes
 * the un-normalised split-KV partial (row max, row sum, O) for aotb_attn_merge_f32. */
int aotb_attention_f32(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, float* O,
                       int ldo, int N, int Tk, const int* Tk_dev, int H, int d_qk, int d_v, float* Mout,
                       float* Lout, void* stream);
int aotb_attn_merge_f32(const float* Opart, const float* Mpart, const float* Lpart, float* O, int R, int N,
                        int H, int d_v, int ldo, void* stream);
/* The same merge over the R memory slots of a bounded bank (split r = slot r, as aotb_lt_attn_tc_slots_f16x2 and
 * aotb_gp_attn_tc_slots_f16x2 write them), which also counts how much each slot was read: O is written exactly as
 * aotb_attn_merge_f32 writes it, and U[r] += sum over (query, head) of the slot's attention mass l_r exp(m_r - m) / L,
 * scaled by 1 / (layers H N) -- so the `layers` launches of one frame add that frame's mean mass per slot, which sums to 1.
 * Each CTA sums its masses per slot and the CTA that draws the last ticket adds the CTA sums in CTA order: U is bitwise
 * reproducible.  A (optional) gets the age tick: A[r] += 1 for every live slot r < *live / rows; pass it in one launch per
 * frame.  R <= 32.  `workspace` (aotb_attn_merge_usage_workspace_bytes(R) bytes, 16-byte aligned, reusable for any smaller
 * R) must be zero-filled before its first use: it holds the launch counter, which every launch leaves at zero again. */
size_t aotb_attn_merge_usage_workspace_bytes(int R);
int aotb_attn_merge_usage_f32(const float* Opart, const float* Mpart, const float* Lpart, float* O, int R, int N, int H,
                              int d_v, int ldo, float* U, int* A, const int* live, int rows, int layers, void* workspace,
                              void* stream);

/* The same merge with every rank's partials read in place over peer memory (sharded long-term bank, BASELINE configs[3]):
 * Oparts / Mparts / Lparts are HOST arrays of `ranks` (<= 8) device pointers -- the local buffer and the NVLink peer mappings
 * of a symmetric-memory allocation -- to Opart_r [splits][N][H*d_v] and Mpart_r / Lpart_r [splits][H][N]; the exchange step of
 * the split-KV attention (otherwise three NCCL all-gathers per layer) is the P2P loads of this kernel.  Partials are merged in
 * (rank, split) order on every rank: outputs are bit-identical across ranks. */
int aotb_attn_merge_peers_f32(const void* const* Oparts, const void* const* Mparts, const void* const* Lparts, int ranks,
                              int splits, float* O, int N, int H, int d_v, int ldo, void* stream);

/* 15x15 local-window attention with relative_emb_k / relative_emb_v:
 * networks/layers/attention.py:308-428 (MultiheadLocalAttentionV2) and :789-914 (LocalGatedPropagation);
 * replaces the third-party spatial_correlation_sampler call sites :341,:828. */
int aotb_local_attention_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                             const float* relk_w, const float* relk_b, const float* relv, float* out, int ldo,
                             int h, int w, int H, int d_att, int d_v, void* stream);

/* Same computation for the AOT head shape (d_att = d_v = 32) with the K / V window halos staged in shared
 * memory per 8x8 query tile; relv_t is relative_emb_v transposed to [H][225][32]. */
int aotb_local_attention_tile_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                  const float* relk_w, const float* relk_b, const float* relv_t, float* out, int ldo,
                                  int h, int w, int H, void* stream);

/* Same computation and arguments as aotb_local_attention_tile_f32 on the tensor cores (mma.sync, split fp16x2 products with
 * fp32 accumulation and an fp32 softmax), per 8x16 query tile; q, k, v, relk_w, relv_t and out 16-byte aligned, ldo % 4 == 0. */
int aotb_local_attention_tc_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                const float* relk_w, const float* relk_b, const float* relv_t, float* out, int ldo,
                                int h, int w, int H, void* stream);

/* Same computation for the DeAOT head shape (one head, d_att 128, d_v 1024, no relative_emb_v; attention.py:789-861) with the
 * window halos staged in shared memory per 8x6 query tile and the channels walked in chunks of 32. */
int aotb_local_gated_tile_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                              const float* relk_w, const float* relk_b, float* out, int ldo, int h, int w, void* stream);

/* one_hot_mask + patch_wise_id_bank conv as a gather-sum (+ LayerNorm for DeAOT):
 * utils/image.py:69-74; networks/models/aot.py:50-63,76-79; networks/models/deaot.py:51-55.
 * mask [Hm][Wm] float ids; wt [(ky*KS+kx)*nid + id][C]. */
int aotb_id_embed_f32(const float* mask, int Hm, int Wm, const float* wt, const float* bias,
                      const float* ln_gamma, const float* ln_beta, float* out, int ldo, int C, int nid,
                      int ksize, int stride, int pad, void* stream);

/* Same result through run lengths: wp = exclusive prefix sums of the table along kx, [ksize][ksize+1][nid][C=256]. */
int aotb_id_embed_runs_f32(const float* mask, int Hm, int Wm, const float* wp, const float* bias,
                           const float* ln_gamma, const float* ln_beta, float* out, int ldo, int C, int nid,
                           int ksize, int stride, int pad, void* stream);

/* networks/engines/aot_engine.py:367-378: mask ids > obj_num with -1e10, bilinear upsample to NCHW. */
int aotb_logits_postproc_f32(const float* logits_nhwc, float* lowres_nchw, float* out_nchw, int h, int w,
                             int NC, int obj_num, int Ho, int Wo, int align_corners, void* stream);
/* fused upsample + argmax (networks/managers/evaluator.py:339-361 for one engine, no TTA). */
int aotb_logits_argmax_f32(const float* lowres_nchw, float* label, int h, int w, int NC, int Ho, int Wo,
                           int align_corners, void* stream);
/* networks/engines/aot_engine.py:565-582 (AOTInferEngine.soft_logit_aggregation) for n_engines sub-engines of max_obj (= 10)
 * objects each, fused into one pass: logits[e] -> NCHW fp32 [1 + max_obj][HW] on the device (the array of pointers itself is
 * host memory); out [1 + n_engines * max_obj][HW] = logit(clamp([prod_e softmax_e[0], softmax_0[1:], softmax_1[1:], ...])). */
int aotb_soft_logit_aggregation_f32(const float* const* logits, int n_engines, int max_obj, float* out, int HW,
                                    void* stream);
/* networks/engines/aot_engine.py:515-533 (AOTInferEngine.separate_mask, label-map form): out[e][i] = mask[i] - e*max_obj if
 * e*max_obj < mask[i] <= (e+1)*max_obj else 0, for e in [0, n_engines). */
int aotb_separate_labels_f32(const float* mask, int n_engines, int max_obj, float* out, int HW, void* stream);
/* The multi-video engines' ID-bank lanes (a lane is the batched counterpart of one sub-engine; lane e of a video carries its ids
 * 10e+1 .. 10e+10).  The three arrays of pointers, the counts and the CSR tables below are host memory. */
/* aotb_soft_logit_aggregation_f32 for n_videos videos in one launch (32 per launch; more are chunked), reading a multi-video
 * decoder's output logits [lanes][h][w][NC] (NHWC, NC = 1 + max_obj = 11) directly: video b's k = lane_ptr[b+1] - lane_ptr[b]
 * (1..8) lanes are lanes[lane_ptr[b] ..] in sub-engine order, lane e masked above obj_nums[lane_ptr[b] + e] with -1e10 at
 * every bilinear tap and sampled at [Ho][Wo] (read unchanged when that is [h][w]).  out[b] [1 + k max_obj][Ho][Wo] receives the
 * merged logits and label[b] [Ho][Wo] their first argmax; either array, or any entry, may be null, not both for one video.
 * Bit for bit aotb_logits_postproc_f32 on each lane followed by aotb_soft_logit_aggregation_f32. */
int aotb_soft_logit_aggregation_batched_f32(const float* logits, int h, int w, int NC, const int* lane_ptr, const int* lanes,
                                            const int* obj_nums, int n_videos, int max_obj, int Ho, int Wo, int align_corners,
                                            float* const* out, float* const* label, void* stream);
/* aotb_separate_labels_f32 for n lanes in one launch (32 per launch; more are chunked): out[b] [HW] = labels[b] [HW] separated
 * for sub-engine parts[b], bit for bit row parts[b] of aotb_separate_labels_f32 on labels[b]. */
int aotb_separate_labels_batched_f32(const float* const* labels, const int* parts, int n, int max_obj, float* const* out,
                                     int HW, void* stream);
/* Up to 4 per-video maps gathered into lane order in one launch: for map j, lane l's n_floats[j] floats of dst[j]
 * [n_lanes][n_floats[j]] = video lane_video[l]'s of src[j] [n_videos][n_floats[j]].  lane_video is device memory (n_lanes
 * ints), so a captured launch follows a table rewritten before its replay; an entry outside [0, n_videos) copies nothing.
 * n_floats[j] must be a multiple of 4 and the maps 16-byte aligned. */
int aotb_lane_gather_f32(const float* const* src, float* const* dst, const int* n_floats, int n_maps, const int* lane_video,
                         int n_lanes, int n_videos, void* stream);
/* Frame input side (SURVEY 8 f.3): dataloaders/eval_datasets.py:60-61 + dataloaders/video_transforms.py:594-715 (MultiRestrictSize's
 * cv2.resize(INTER_CUBIC) of the float image, MultiToTensor's / 255, - mean, / std, HWC -> CHW) on the uint8 frame in one pass.
 * img uint8 [H][W][3]; ix / cx [Wo][4] and iy / cy [Ho][4] = clamped tap indices and Keys-cubic (A = -0.75) weights per output
 * column / row (all four null when Ho == H and Wo == W); flip != 0 mirrors horizontally after the resize; out fp32 [3][Ho][Wo]. */
int aotb_preprocess_bgr_u8(const void* img, int H, int W, const int* ix, const float* cx, const int* iy, const float* cy,
                           float* out, int Ho, int Wo, int flip, void* stream);
/* Mask output side: utils/image.py:103-105 (`mask_tensor.cpu().numpy().astype('uint8')`): the float label map leaves the
 * device as uint8 (1 byte per pixel over PCIe instead of 4 or 8). */
int aotb_label_to_u8(const float* label, void* out_u8, int n, void* stream);
/* F.interpolate(mode="nearest") of a label map: networks/managers/evaluator.py:418-421. */
int aotb_nearest_resize_f32(const float* in, float* out, int H, int W, int Ho, int Wo, void* stream);
/* Test-time augmentation ensemble, networks/managers/evaluator.py:332-369, in one pass: n_augs (1..8) logit maps
 * logits[e] -> [NC][h_e][w_e] fp32 on the device, with sizes[2e], sizes[2e+1] = h_e, w_e and flips[e] (the three arrays are host
 * memory); per output pixel (y, x) of [H][W]: augmentation e is upsampled bilinearly at column flips[e] ? W-1-x : x (:333-337),
 * softmaxed over NC (:339), the probabilities averaged in augmentation order (:355-358); label = first argmax (:359-361), then
 * new_label[i] where that is nonzero (:363-369; new_label may be null).  pred_prob [NC][H][W] is written when not null.
 * A map already at [H][W] (the aggregated logits of a > 10-object engine) is read unchanged. */
int aotb_tta_merge_f32(const float* const* logits, const int* sizes, const int* flips, int n_augs, int NC, int H, int W,
                       int align_corners, const float* new_label, float* label, float* pred_prob, void* stream);
/* One augmentation's memory label, networks/managers/evaluator.py:346-353 and :363-422 (:315-319 on the first frame): for
 * each pixel of out [Hi][Wi] take its nearest source (sy, sx) in [H][W] (the rule of aotb_nearest_resize_f32); base =
 * argmax softmax of the bilinear upsample of logits [NC][h][w] at (sy, sx), or 0 when logits is null; n = new_label[sy][flip ?
 * W-1-sx : sx], or 0 when new_label is null; out = n != 0 ? n : base. */
int aotb_tta_feedback_f32(const float* logits, int h, int w, int NC, int H, int W, int align_corners, int flip,
                          const float* new_label, float* out, int Hi, int Wi, void* stream);
/* aotb_tta_merge_f32 over n videos in one launch (32 per launch; more are chunked), reading each augmentation's logits straight
 * from a multi-video decoder's output instead of aotb_logits_postproc_f32's maps (networks/managers/evaluator.py:332-369 per
 * video, after networks/engines/aot_engine.py:367-378 per augmentation).  logits[e]: augmentation e's decoder output
 * [lanes][h_e][w_e][NC] (NHWC, sizes[2e], sizes[2e+1]); video b reads lane lanes[b * n_augs + e] of it, where a channel above
 * obj_nums[b] reads -1e10 at every bilinear tap, the value aotb_logits_postproc_f32 writes.  label [n][H][W]; pred_prob
 * [n][NC][H][W] when not null; new_labels: n pointers to [H][W] overlays, or null, and any entry may be null.  Video b's label
 * and prob are bit for bit aotb_logits_postproc_f32 (low-res, obj_nums[b]) on each of its lanes followed by
 * aotb_tta_merge_f32. */
int aotb_tta_merge_batched_f32(const float* const* logits, const int* sizes, const int* flips, int n_augs, const int* lanes,
                               const int* obj_nums, int n, int NC, int H, int W, int align_corners,
                               const float* const* new_labels, float* label, float* pred_prob, void* stream);
/* aotb_tta_feedback_f32 over n_lanes lanes of one multi-video decoder's output in one launch (32 per launch; more are
 * chunked).  logits: [n_lanes][h][w][NC] (NHWC), lane k masked at obj_nums[k] as aotb_logits_postproc_f32 masks it, or null
 * (base = 0 for every lane, the first-frame and teacher-forced form; obj_nums may then be null).  flips[k]; new_labels: n_lanes
 * pointers to [H][W] maps, or null, and any entry may be null.  out [n_lanes][Hi][Wi]: lane k's map is bit for bit
 * aotb_logits_postproc_f32 + aotb_tta_feedback_f32 on lane k. */
int aotb_tta_feedback_batched_f32(const float* logits, int h, int w, int NC, int n_lanes, const int* obj_nums,
                                  const int* flips, const float* const* new_labels, int H, int W, int align_corners,
                                  float* out, int Hi, int Wi, void* stream);

/* Tensor-core long-term attention (wgmma + TMA), AOT head shape H x 32, split-fp16 ("fp16x2")
 * operands: every fp32 value x is stored as hi = fp16(x), lo = fp16(x - hi) in rows [hi(32) | lo(32)].
 * The operands are not normalised: each element keeps an absolute error floor of 2^-25 (values below about 2^-3 lose
 * relative precision) and |x| >= 65520 overflows hi.  K and V rows beyond the live key count get probability 0 but still
 * enter the P V product, so they must be finite (0 * NaN is NaN); Q rows beyond N only affect rows that are not written.
 * networks/layers/attention.py:82-117 called from networks/layers/transformer.py:346 (and :324, Tk = N).
 *   aotb_tc_pack_rows_f16x2: fp32 [rows][ld] -> packed [H][cap][64] at a row offset, values / div first
 *                            (div = T for Q, attention.py:82; 1 for K and V).  Buffers must be zero-filled
 *                            beyond the live rows.
 *   aotb_lt_attn_tc_f16x2  : exact bit 0 set -> S = QhKh + QlKh + QhKl, O = (Ph + Pl)[Vh|Vl];
 *                            clear -> S = QhKh, O = Ph[Vh|Vl].  exact bit 2: the mbarrier waits poll instead of
 *                            sleeping (latency experiment; results unchanged).  splits > 1 writes split-KV partials
 *                            for aotb_attn_merge_f32 (splits cut on 128-key boundaries).  dbg (optional) receives S of
 *                            keys [0, 128) [128][128] and O' [128][64] of CTA 0. */
int aotb_tc_pack_rows_f16x2(const float* src, int ld, void* dst, int cap, int rows, int H, int row_off,
                            const int* row_off_dev, float div, void* stream);
size_t aotb_lt_attn_tc_smem_bytes(void);
/* The default layout's kernel in one mode (exact bit 0 as below) on the current device, configured as its launches are:
 * resident CTAs per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor), registers per thread and local-memory bytes per
 * thread (cudaFuncGetAttributes).  The KV-split policy assumes the first is 2 (engine.LT_TILE_CTAS_PER_SM). */
int aotb_lt_attn_tc_occupancy(int exact, int* ctas_per_sm, int* regs, int* local_bytes);
int aotb_lt_attn_tc_f16x2(const void* Qp, int Nq_cap, const void* Kp, const void* Vp, int kv_cap, int N, int Tk,
                          const int* Tk_dev, int H, float* O, int ldo, float* Opart, float* Mpart, float* Lpart,
                          int splits, int exact, float* dbg, void* stream);
/* The same attention (default layout) over a bank of memory slots of split_rows keys each: split z covers keys
 * [z split_rows, (z + 1) split_rows) of the live ones, so with splits slots and the live keys a prefix of whole slots each
 * partial (Opart [splits][N][H*32], Mpart / Lpart [splits][H][N]) is one slot's; a slot beyond the live keys gets m = -inf,
 * l = 0.  The live keys must not exceed splits * split_rows.  split_rows need not be a multiple of the 64-key tile.
 * exact: bit 0 and bit 2 as above; splits >= 2. */
int aotb_lt_attn_tc_slots_f16x2(const void* Qp, int Nq_cap, const void* Kp, const void* Vp, int kv_cap, int N, int Tk,
                                const int* Tk_dev, int H, float* Opart, float* Mpart, float* Lpart, int splits, int split_rows,
                                int exact, void* stream);

/* DeAOT long-term attention as GEMM -> row softmax -> GEMM on the tensor cores (AOTB_DEAOT_LT=gemm):
 * GatedPropagation.forward networks/layers/attention.py:672-704 with 1 head, d_qk = 128, d_v = 1024.  The two GEMMs are
 * aotb_conv2d_nhwc_tc with the bank as pre-split weights; these entry points maintain those copies and do the softmax.
 *   aotb_split_rows_f16x2: src fp32 [rows][lds] (C columns) -> hi / lo fp16 [.][ldw] rows [row_off, row_off + rows)
 *                          (hi = fp16(x), lo = fp16(x - hi)); the keys [Tk_cap][128] = weights of S = Q K^T.
 *   aotb_split_cols_f16x2: the same values written as COLUMNS [col_off, col_off + rows) of hiT / loT [C][ldt]: the
 *                          transposed value bank [1024][Tk_cap] = weights of O = P V.
 *   aotb_row_softmax_f32 : S [N][ld] in place: columns [0, live) <- softmax(scale * S[r][0:live]) (attention.py:686-693,
 *                          scale = 1 / T applied to the scores instead of to Q), columns [live, cols) <- 0; live = *Tk_dev
 *                          if given, else Tk.  Offsets / counts may be device-resident so a captured graph can be replayed. */
int aotb_split_rows_f16x2(const float* src, int lds, void* hi, void* lo, int ldw, int rows, int C, int row_off,
                          const int* row_off_dev, void* stream);
int aotb_split_cols_f16x2(const float* src, int lds, void* hiT, void* loT, int ldt, int rows, int C, int col_off,
                          const int* col_off_dev, void* stream);
int aotb_row_softmax_f32(float* S, int ld, int N, int cols, int Tk, const int* Tk_dev, float scale, void* stream);

/* DeAOT long-term attention fused on the tensor cores (AOTB_DEAOT_LT=tc, the default; gp_attn_tc.cu): GatedPropagation.forward
 * networks/layers/attention.py:672-704 with 1 head, d_qk = 128, d_v = dv (1024).  Operands in the split-fp16 row format of
 * aotb_tc_pack_rows_f16x2 with one "head" per 32 channels: Qp [4][Nq_cap][64] (Q / T, T = sqrt(128), Nq_cap a multiple of 128),
 * Kp [4][kv_cap][64], Vp [dv/32][kv_cap][64].  O [N][ldo] = softmax((Q / T) K^T) V.  exact bit 0 / bit 2 as in
 * aotb_lt_attn_tc_f16x2.  splits > 1 writes un-normalised partials Opart [splits][N][dv], Mpart / Lpart [splits][1][N] for
 * aotb_attn_merge_f32 (H = 1, d_v = dv). */
int aotb_gp_attn_tc_f16x2(const void* Qp, int Nq_cap, const void* Kp, const void* Vp, int kv_cap, int N, int Tk,
                          const int* Tk_dev, int dv, float* O, int ldo, float* Opart, float* Mpart, float* Lpart,
                          int splits, int exact, void* stream);
/* Its memory-slot form, as aotb_lt_attn_tc_slots_f16x2: Opart [splits][N][dv], Mpart / Lpart [splits][1][N]. */
int aotb_gp_attn_tc_slots_f16x2(const void* Qp, int Nq_cap, const void* Kp, const void* Vp, int kv_cap, int N, int Tk,
                                const int* Tk_dev, int dv, float* Opart, float* Mpart, float* Lpart, int splits, int split_rows,
                                int exact, void* stream);

/* Long-term memory append in place (replaces torch.cat, networks/engines/aot_engine.py:291-305). */
int aotb_bank_append_f32(const float* src, int lds, float* bank, int ldb, int rows, int cols, int offset,
                         const int* offset_dev, void* stream);
int aotb_counter_add(int* counter, int delta, void* stream);

/* Bounded long-term bank: at most cap_rows / rows memory frames, the first one pinned in rows [0, pinned_rows), the others a
 * FIFO ring over rows [pinned_rows, cap_rows).  Two device counters carry the state, so both calls can sit in a replayed graph:
 * *live = rows the attention kernels read (their Tk_dev), *write = row offset of the next store.
 *   aotb_bank_ring_store: ONE launch stores a memory frame's keys k_src [rows][ldk] (k_cols channels) and values v_src
 *                         [rows][ldv] (v_cols channels) at row *write of every copy of the bank that is given: the fp32 banks
 *                         k_bank / v_bank [cap_rows][ldkb / ldvb] (equal to the source) and the split-fp16 banks k_packed /
 *                         v_packed [cols / 32][cap_rows][64] (bit for bit the rows aotb_tc_pack_rows_f16x2 writes with
 *                         div = 1).  A null destination is skipped.  All pointers 16-byte aligned, columns and row strides
 *                         multiples of 4, packed copies need multiples of 32 channels.  A store that does not fit
 *                         (*write < 0 or *write + rows > cap_rows) writes nothing.
 *   aotb_ring_advance   : after such a store, *live = min(*live + rows, cap_rows); *write += rows, and *write = pinned_rows
 *                         if a further store of `rows` rows there would pass cap_rows.  Requires rows > 0,
 *                         pinned_rows + rows <= cap_rows and (cap_rows - pinned_rows) % rows == 0, so starting from
 *                         *write = 0 (with pinned_rows a multiple of rows) no store ever passes the end of the bank. */
int aotb_bank_ring_store(const float* k_src, int ldk, int k_cols, const float* v_src, int ldv, int v_cols, int rows,
                         float* k_bank, int ldkb, float* v_bank, int ldvb, void* k_packed, void* v_packed, int cap_rows,
                         const int* write, void* stream);
int aotb_ring_advance(int* live, int* write, int rows, int cap_rows, int pinned_rows, void* stream);
/* Usage policy of the bounded bank (instead of the FIFO order of aotb_ring_advance's write offset), run before each
 * aotb_bank_ring_store, with aotb_ring_advance after it for *live: while the bank is not full (*live / rows < cap_rows / rows)
 * *write = *live, the next free slot; once it is full, *write = s rows for the slot s in [pinned_rows / rows, cap_rows / rows)
 * with the lowest U[s] / A[s] (A[s] == 0 counts as +inf, ties go to the lowest s).  The chosen slot's U and A are reset to 0.
 * U / A [cap_rows / rows] are the counters of aotb_attn_merge_usage_f32.  pinned_rows and cap_rows are multiples of rows and
 * pinned_rows + rows <= cap_rows, so *write always addresses a whole slot of the bank. */
int aotb_ring_select_usage(const int* live, int* write, float* U, int* A, int rows, int cap_rows, int pinned_rows,
                           void* stream);

/* ---- several independent videos in one launch (MultiVideoInferEngine).  Each entry point runs n problems whose rows are
 * stacked; problem b's result is bit for bit the one-problem entry point named beside it on problem b's rows.
 *   aotb_lt_attn_tc_batched_f16x2  (aotb_lt_attn_tc_f16x2, "tile" layout): queries at rows b q_stride of Qp [H][q_rows][64],
 *       keys / values at rows b kv_stride of Kp / Vp [H][kv_rows][64], live keys Tk_dev[b] (int32 [n]; null: Tk for all);
 *       O [n N][ldo], or with splits > 1 partials Opart [splits][n N][H*32], Mpart / Lpart [splits][H][n N] for
 *       aotb_attn_merge_f32 over n N rows.  One split count for all problems; exact bits 0 (exact) and 2 (spin).
 *   aotb_local_attention_tc_batched_f32  (aotb_local_attention_tc_f32): map b = rows [b h w, (b + 1) h w) of q, k, v, out.
 *   aotb_id_embed_runs_batched_f32  (aotb_id_embed_runs_f32): label maps mask [n][Hm][Wm], output rows [b ho wo, ...).
 *   aotb_bank_ring_store_batched  (aotb_bank_ring_store): bank b = rows [b cap_rows, (b + 1) cap_rows) of every copy (the
 *       packed copies' 32-channel chunks head_rows rows apart) stores source rows [b rows, (b + 1) rows) at write[b], only
 *       when store[b] != 0.
 *   aotb_ring_advance_batched  (aotb_ring_advance): live[b] / write[b] of every bank with store[b] != 0 (n <= 1024). */
int aotb_lt_attn_tc_batched_f16x2(const void* Qp, int q_stride, int q_rows, const void* Kp, const void* Vp, int kv_stride,
                                  int kv_rows, int n, int N, int Tk, const int* Tk_dev, int H, float* O, int ldo, float* Opart,
                                  float* Mpart, float* Lpart, int splits, int exact, void* stream);
int aotb_local_attention_tc_batched_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                        const float* relk_w, const float* relk_b, const float* relv_t, float* out, int ldo,
                                        int h, int w, int H, int n, void* stream);
int aotb_id_embed_runs_batched_f32(const float* mask, int n, int Hm, int Wm, const float* wp, const float* bias,
                                   const float* ln_gamma, const float* ln_beta, float* out, int ldo, int C, int nid, int ksize,
                                   int stride, int pad, void* stream);
int aotb_bank_ring_store_batched(const float* k_src, int ldk, int k_cols, const float* v_src, int ldv, int v_cols, int rows,
                                 int n, float* k_bank, int ldkb, float* v_bank, int ldvb, void* k_packed, void* v_packed,
                                 int cap_rows, int head_rows, const int* write, const int* store, void* stream);
int aotb_ring_advance_batched(int* live, int* write, const int* store, int n, int rows, int cap_rows, int pinned_rows,
                              void* stream);

/* ---- the same for DeAOT's gated propagation (DeAOTMultiVideoInferEngine), in the form above.
 *   aotb_gp_attn_tc_batched_f16x2  (aotb_gp_attn_tc_f16x2; GatedPropagation.forward, networks/layers/attention.py:672-704, the
 *       long-term and self-attention calls of networks/layers/transformer.py:614-653): queries at rows b q_stride of
 *       Qp [4][q_rows][64], keys at rows b kv_stride of Kp [4][kv_rows][64], values of Vp [dv/32][kv_rows][64], live keys
 *       Tk_dev[b] (int32 [n]; null: Tk for all); O [n N][ldo], or with splits > 1 partials Opart [splits][n N][dv],
 *       Mpart / Lpart [splits][1][n N] for aotb_attn_merge_f32 (H = 1, d_v = dv) over n N rows.  exact bits 0 and 2.
 *   aotb_local_gated_tile_batched_f32  (aotb_local_gated_tile_f32; LocalGatedPropagation.forward, attention.py:789-861):
 *       map b = rows [b h w, (b + 1) h w) of q, k, v, out. */
int aotb_gp_attn_tc_batched_f16x2(const void* Qp, int q_stride, int q_rows, const void* Kp, const void* Vp, int kv_stride,
                                  int kv_rows, int n, int N, int Tk, const int* Tk_dev, int dv, float* O, int ldo, float* Opart,
                                  float* Mpart, float* Lpart, int splits, int exact, void* stream);
int aotb_local_gated_tile_batched_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                      const float* relk_w, const float* relk_b, float* out, int ldo, int h, int w, int n,
                                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AOTB200_H */
