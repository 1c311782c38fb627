/* mqdet_b200 — C ABI of the H100-native MQ-Det hot path.
 *
 * Every entry point takes DEVICE pointers + explicit sizes/strides + a cudaStream_t (passed as
 * void*), allocates nothing, never synchronises the device, and returns 0 on success or a
 * negative error code (the text is available from mqdet_last_error(), thread-local).
 *
 * What each group replaces in the reference (paths relative to the MQ-Det repository root):
 *   - mqdet_gemm_f16 / mqdet_layernorm / mqdet_softmax_rows: the ATen Linear/LayerNorm/softmax
 *     chains of maskrcnn_benchmark/modeling/language_backbone/modeling_bert_new.py:196-248,347-374,
 *     maskrcnn_benchmark/utils/fuse_helper.py:218-303 and
 *     maskrcnn_benchmark/modeling/rpn/modeling_bert.py:39-270.
 *   - mqdet_gcp_sparse_attn / mqdet_gcp_gate_residual_ln: MaskedCrossAttention.forward (sparse)
 *     modeling_bert_new.py:162-248 and GatedCrossAttentionBlock.forward :347-374.
 *   - mqdet_ml_nms: maskrcnn_benchmark._C.ml_nms (maskrcnn_benchmark/csrc/ml_nms.h:11-27,
 *     csrc/cuda/ml_nms.cu:79-149).
 *   - mqdet_dcnv2_im2col: maskrcnn_benchmark._C.modulated_deform_conv_forward
 *     (csrc/cuda/deform_conv_cuda.cu:496-575, deform_conv_kernel_cuda.cu:578-641).
 *   - mqdet_anchors / mqdet_atss_*: modeling/rpn/anchor_generator.py:72-137 and
 *     modeling/rpn/inference.py:620-769.
 */
#ifndef MQDET_B200_H_
#define MQDET_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MQDET_F16 0
#define MQDET_F32 1

#define MQDET_ACT_NONE 0
#define MQDET_ACT_GELU 1 /* exact erf GELU */
#define MQDET_ACT_RELU 2

#define MQDET_VEC_NONE 0
#define MQDET_VEC_SCALAR 1  /* one device float */
#define MQDET_VEC_PER_COL 2 /* length N */
#define MQDET_VEC_PER_ROW 3 /* length M */

#define MQDET_GEMM_IMPL_TC 0      /* TMA + wgmma, warp-specialised, persistent: min(tiles, SMs) CTAs (product path) */
#define MQDET_GEMM_IMPL_SIMT 1    /* plain shared-memory tiled fp32-FMA kernel (validation only) */
#define MQDET_GEMM_IMPL_TC_ONESHOT 2 /* the same tensor-core kernel launched with one CTA per tile (bit-identical results) */

const char* mqdet_last_error(void);
int mqdet_version(void);
/* Leave n SMs free of the persistent one-CTA-per-SM kernels (GEMM, dcn_conv, biattn_*): call once per process BEFORE the first launch /
 * graph capture when a collective kernel runs next to the forward (N > 1: one NCCL CTA waiting for a peer would otherwise hold the SM
 * of one persistent CTA for the whole wait).  Process-wide; 0 (default) = use every SM. */
int mqdet_reserve_sms(int n);

/* D[z] = epilogue( A[z] (M x K, fp16, K contiguous) * B[z]^T (N x K, fp16, K contiguous) ), fp32 accumulate.
 *   v = alpha*acc + bias            (scale_after_bias == 0)
 *   v = alpha*(acc + bias)          (scale_after_bias != 0)
 *   v = act(v); v = clamp(v, -clamp, +clamp) if clamp > 0
 *   v = gate * v   (gate optionally passed through tanh);  v += residual;  D = v
 * z = z1 + nb1*z2 ranges over nb1*nb2 batches; a batch stride of 0 broadcasts that operand.
 * B laid out [N, K] is exactly an nn.Linear weight, so y = x W^T needs no transposition.
 * Requirements: K % 8 == 0, lda/ldb and batch strides % 8 == 0, A/B 16-byte aligned. */
typedef struct mqdet_gemm_args {
  const void* A;
  const void* B;
  int64_t M, N, K;
  int64_t lda, ldb;
  int64_t nb1, nb2;
  int64_t a_b1, a_b2, b_b1, b_b2;
  void* C;
  int32_t c_dtype; /* MQDET_F16 / MQDET_F32 */
  int64_t ldc, c_b1, c_b2;
  float alpha;
  int32_t scale_after_bias;
  const float* bias;
  int32_t bias_mode; /* MQDET_VEC_NONE / PER_COL / PER_ROW */
  int64_t bias_b1, bias_b2;
  int32_t act;
  float clamp;
  const float* gate;
  int32_t gate_mode; /* MQDET_VEC_* */
  int32_t gate_tanh;
  const void* R; /* residual, same logical shape as D */
  int32_t r_dtype;
  int64_t ldr, r_b1, r_b2;
} mqdet_gemm_args;

int mqdet_gemm_f16(const mqdet_gemm_args* args, int impl, void* stream);

/* Dense multi-head cross-attention with head dim 32 in ONE flash-style kernel (PreSelect: MaskedCrossAttention.forward with
 * spase_forward=False, no mask, modeling_bert_new.py:186-248,398-409): out[b,t,h,:] = softmax_i(q[b,t,h,:] . k[b,i,h,:]) v[b,i,h,:].
 *   q [B][Tq][q_ld] f16 (already scaled; head h at column h*32), kv [B][I][kv_ld] f16 (K of head h at column h*32, V at
 *   v_col0 + h*32: the to_kv Linear output as is), out [B][Tq][o_ld] f16; *_b = image strides in elements.  The fp32 score
 *   tensor [B, heads, Tq, I] is never materialised (online softmax over 64-token chunks, fp32 statistics, fp16 P). */
int mqdet_dense_cross_attn(const void* q, int64_t q_ld, int64_t q_b, const void* kv, int64_t kv_ld, int64_t kv_b, int64_t v_col0,
                           void* out, int64_t o_ld, int64_t o_b, int64_t B, int64_t Tq, int64_t I, int64_t heads,
                           int64_t head_dim, void* stream);

/* Row-wise LayerNorm over the last dim D (biased variance, eps inside sqrt).
 * x: [rows, D] in_dtype with row stride ldx; out16 (fp16) and/or out32 (fp32) may be NULL.
 * If zero_row_period > 0, rows r with (r % zero_row_period) == zero_row_period-1 are treated as an
 * all-zero input row (the GCP padding vision slot, modeling_bert_new.py:176-180) and x is not read. */
int mqdet_layernorm(const void* x, int in_dtype, int64_t ldx, const float* gamma, const float* beta,
                    float eps, int64_t rows, int64_t D, void* out16, void* out32, int64_t ldo,
                    int64_t zero_row_period, void* stream);

/* The MLP half of a Swin block (swint.py:240-241) in one kernel, for C = 96 / 192:
 *   out[r] = x[r] + fc2(GELU(fc1(LN(x[r]))))
 * x, out: fp32 [rows][C] contiguous, 16-byte aligned, not overlapping; ln_w / ln_b: fp32 [C]; w1: fp16 [4C][C], b1: fp32 [4C];
 * w2: fp16 [C][4C], b2: fp32 [C] (nn.Linear layouts).  Bit-identical to mqdet_layernorm (fp16 out) -> mqdet_gemm_f16 (bias +
 * GELU, fp16 out) -> mqdet_gemm_f16 (bias + fp32 residual x, fp32 out). */
int mqdet_swin_mlp_f16(const float* x, int64_t rows, int64_t C, const float* ln_w, const float* ln_b, float eps,
                       const void* w1, const float* b1, const void* w2, const float* b2, float* out, void* stream);

/* residual add + LayerNorm:  y = LN(a + b).  a,b fp32 [rows, D]; writes fp32 and/or fp16. */
int mqdet_add_layernorm(const float* a, const float* b, const float* gamma, const float* beta, float eps,
                        int64_t rows, int64_t D, float* out32, void* out16, float clamp, void* stream);

/* Sparse GCP attention (modeling_bert_new.py:162-248 with K/V de-duplicated per unique query):
 *   q   [B*T, H*Dh] fp16 (already scaled),  kv [B, V+1, 2*H*Dh] fp16 (row V = padding slot; K | V halves)
 *   idx [B*T, S] int32 in [0, V] (V = padding);  out [B*T, H*Dh] fp16.
 * sim = q.k (+ -1e4 on padding) -> softmax over S -> zero padding probs -> sum p*v. */
int mqdet_gcp_sparse_attn(const void* q, const void* kv, const int32_t* idx, void* out, int64_t B, int64_t T,
                          int64_t V, int64_t S, int64_t H, int64_t Dh, void* stream);

/* GCP gate + residual + FFN pre-norm (modeling_bert_new.py:359-372):
 *   g = tanh(h1[r,:] . w2);  x1 = s*g + x;  writes x1 (fp32) and LN(x1; gamma,beta) (fp16).
 *   h1 [rows, Dg] fp16, w2 [Dg] fp32, s/x [rows, D] fp32.  gate_out (optional) receives g[r]. */
int mqdet_gcp_gate_residual_ln(const void* h1, const float* w2, int64_t Dg, const float* s, const float* x,
                               const float* gamma, const float* beta, float eps, int64_t rows, int64_t D,
                               float* x1_out, void* ln_out16, float* gate_out, void* stream);

/* Build the [B*T, S] index table from a 0/1 mask [B, V, T] (fp32): ascending v with mask != 0,
 * padded with V (get_index_with_padding_batch, modeling_bert_new.py:40-63). counts_out[B*T] optional. */
int mqdet_gcp_build_index(const float* mask, int64_t B, int64_t V, int64_t T, int64_t S, int32_t* idx,
                          int32_t* counts_out, void* stream);

/* Row softmax over the last dim with optional additive column mask (warp per row, fp32 math).
 *   x [rows, n] fp16/fp32 (row stride ldx) -> y fp16 [rows, n_pad] (row stride ldy); columns [n, n_pad) := 0.
 *   v = x*scale + (colmask[batch, c] == 0 ? mask_value : keep_add);  batch = row / rows_per_batch.
 *   BERT self-attention: mask_value -10000, keep_add 0.  BiAttention (fuse_helper.py:270-283): -9e15 / +1. */
int mqdet_softmax_rows(const void* x, int in_dtype, int64_t ldx, void* y, int64_t ldy, int64_t rows, int64_t n,
                       int64_t n_pad, float scale, const float* colmask, int64_t rows_per_batch, float mask_value,
                       float keep_add, void* stream);

/* Column softmax with transposed output: P[z][t][0:Np] = softmax_n(A[z][n][t]) (zero beyond N), fp16 in/out.
 * BiAttention text->image direction (fuse_helper.py:257-268) without a second QK^T product.  T <= 256, T % 8 == 0.
 * workspace: mqdet_colsoftmax_workspace_floats(Z, N, T) floats. */
int64_t mqdet_colsoftmax_workspace_floats(int64_t Z, int64_t N, int64_t T);
int mqdet_colsoftmax_transposed(const void* A, int64_t Z, int64_t N, int64_t T, void* P, int64_t Np, float* workspace,
                                void* stream);

/* Column statistics only: workspace (mqdet_colsoftmax_workspace_floats(Z, N, T) floats) receives, at float offset
 * Z * ceil(N/512) * 2 * T, stat[z][2][T] = (column max, 1 / column sum of exp) of A [Z][N][T] f16. */
int mqdet_colsoftmax_stats(const void* A, int64_t Z, int64_t N, int64_t T, float* workspace, void* stream);

/* T == 256: mqdet_colsoftmax_stats and the masked row softmax of the image -> text side in ONE pass over A, in place:
 * statistics of the unmasked scores as above; then A[z][n][:] <- softmax_t(A[z][n][t] + (colmask[z / z_per_mask][t] == 0 ?
 * mask_value : keep_add)) (fuse_helper.py:277-287).  colmask may be NULL (no mask). */
int mqdet_colstats_rowsoftmax(void* A, int64_t Z, int64_t N, int64_t T, const float* colmask, int64_t z_per_mask,
                              float mask_value, float keep_add, float* workspace, void* stream);

/* Text -> image side of BiMultiHeadAttention (maskrcnn_benchmark/utils/fuse_helper.py:257-275,289-291) fused into one
 * wgmma kernel per (image, head, 64 text tokens): out[z][t][:] = sum_n softmax_n(clamp(k_t . q_n))[n] * Vv[n][:], without
 * materialising the transposed probabilities: S^T = K Q^T (wgmma, 64 image tokens per step) -> exp(fp16-rounded score
 * - column max) -> fp16 P (register operand) -> O += P Vv (wgmma) -> O / column sum.  stat[z][2][T] as produced by
 * mqdet_colsoftmax_stats from the SAME scores (q already carries the 1/sqrt(d) scale).  z = z2 * nb1 + z1.
 *   k [z][T][d], q [z][N][d], vvT [z][d][Np] f16 (Np >= N, zero padded), out [z][T][d] f16; *_ld = row stride, *_b1 / *_b2 =
 *   batch strides in elements (multiples of 8); d == 256, T <= 256. */
int mqdet_biattn_text(const void* k, int64_t k_ld, int64_t k_b1, int64_t k_b2, const void* q, int64_t q_ld, int64_t q_b1,
                      int64_t q_b2, const void* vvT, int64_t v_ld, int64_t v_b1, int64_t v_b2, const float* stat, float clamp,
                      void* out, int64_t o_ld, int64_t o_b1, int64_t o_b2, int64_t nb1, int64_t nb2, int64_t T, int64_t N,
                      int64_t Np, int64_t d, void* stream);

/* Same kernel, VN variant: the value operand is the layer-normed image-token tensor itself, vn [z][N][256] f16 (read MN-major
 * from the same [token x channel] tile), so that out[z][t][:] = sum_n softmax_n(clamp(k_t . q_n + rowbias_t))[n] * vn[n][:] — the
 * value projection W_vv is applied AFTER the token reduction by the caller (sum_n p[n] = 1 moves the bias out as well), and the
 * [B, E, N] value tensor is never built.  colmax [z][T] f32 = column maxima of the clamped fp32 scores (mqdet_biattn_image);
 * the column sums are accumulated in-kernel from the fp32 scores (no fp16 re-quantisation).  rowbias [z][T * rb_ld] f32 or NULL:
 * an additive score term per text token.  With k := gT (the query projection folded into the keys, see mqdet_biattn_image),
 * q := vn (head stride 0) and rowbias := gbias, the kernel streams only the image tokens: q [B,N,E] is never built. */
int mqdet_biattn_text_vn(const void* k, int64_t k_ld, int64_t k_b1, int64_t k_b2, const void* q, int64_t q_ld, int64_t q_b1,
                         int64_t q_b2, const void* vn, int64_t vn_ld, int64_t vn_b1, int64_t vn_b2, const float* colmax,
                         const float* rowbias, int64_t rb_ld, float clamp, void* out, int64_t o_ld, int64_t o_b1, int64_t o_b2,
                         int64_t nb1, int64_t nb2, int64_t T, int64_t N, void* stream);

/* Image -> text side of BiMultiHeadAttention fused with the query, value and output projections, layer scale and residual
 * (maskrcnn_benchmark/utils/fuse_helper.py:240-256,277-302,420-425) in ONE wgmma kernel: per 64 image tokens and
 * head, S = vn gT_h^T + gbias_h stays in registers (fp32) -> clamp -> masked softmax over the T tokens in registers -> P (fp16,
 * registers) -> acc += P mT_h^T summed over the heads -> out = res + gamma * (acc + bias).
 * Neither q, the score matrix nor a per-head context reaches HBM.  mask [B][T] f32 (0 = padding token: probability exactly 0,
 * like the reference's -9e15; an all-masked image gets the uniform distribution the reference's fp32 sum produces) or NULL;
 * gamma / bias [256] f32 (16-byte aligned) and res may be NULL.
 *   vn [B][N][256] f16 = the layer-normed image tokens; *_ld row strides, *_b image strides, *_bh head strides (elements, x8);
 *   gT [B][H][T][256] f16 with gT[b][h][t][c] = d^-1/2 sum_dd Wq[h*256+dd][c] K[b][t][h*256+dd]: the query projection of head h
 *   folded into the key operand (S = (vn Wq_h^T + bq_h) d^-1/2 K_h^T = vn gT_h^T + gbias_h); gbias [B*H][T * gb_ld] f32 =
 *   d^-1/2 bq_h . K_h[t] (NULL: none);
 *   mT [B][H][256][T] f16 with mT[b][h][o][t] = sum_dd W_out[o][h*256+dd] V_l[b][t][h*256+dd]: the value and output projections
 *   folded ((P V_l,h) W_h^T == P (V_l,h W_h^T));  out [B][N][256] f16.  8 <= T <= 256, T % 8 == 0, head dim 256, H <= 8.
 * colmax [B*H][T] f32 receives max_n clamp(S[n][t]) — the softmax shift of the text -> image side (mqdet_biattn_text_vn).
 * workspace: mqdet_biattn_image_workspace_floats(B, H, N, T) floats. */
int64_t mqdet_biattn_image_workspace_floats(int64_t B, int64_t H, int64_t N, int64_t T);
int mqdet_biattn_image(const void* vn, int64_t vn_ld, int64_t vn_b, const void* gT, int64_t g_ld, int64_t g_bh, int64_t g_b,
                       const float* gbias, int64_t gb_ld, const void* mT, int64_t m_ld, int64_t m_bh, int64_t m_b,
                       const float* bias, const float* gamma, const void* res, int64_t res_ld, int64_t res_b, const float* mask,
                       float clamp, void* out, int64_t o_ld, int64_t o_b, float* colmax, float* workspace, int64_t B, int64_t H,
                       int64_t N, int64_t T, void* stream);

/* Text side of the dot-product token head (vldyhead.py:810,818): e = x / max(||x||, eps) written as fp16 and/or
 * fp32, dot[r] = e[r,:] . w + b0[0] (w, b0, dot optional). */
int mqdet_l2norm_rowdot(const float* x, int64_t rows, int64_t D, float eps, const float* w, const float* b0, void* e16,
                        float* e32, float* dot, void* stream);

/* fp32 -> fp16 cast (n elements), and fp16 -> fp32. */
int mqdet_cast_f32_f16(const float* x, void* y, int64_t n, void* stream);
int mqdet_cast_f16_f32(const void* x, float* y, int64_t n, void* stream);

/* GroundingDINO ContrastiveEmbed.forward tail (groundingdino_new/models/GroundingDINO/utils.py:261-266): logits [B,Q,Tmax]
 * f32 whose first T columns hold x . y^T (mqdet_gemm_f16); columns of padding tokens (text_token_mask [B,T] bytes, 0 =
 * padding) and columns T..Tmax-1 are set to -inf in place. */
int mqdet_contrastive_mask(float* logits, const uint8_t* text_token_mask, int64_t B, int64_t Q, int64_t T, int64_t Tmax,
                           void* stream);

/* Stable descending argsort of n <= 16384 fp32 scores (ties: lower index first), single CTA bitonic sort. */
int mqdet_argsort_desc(const float* scores, int64_t n, int64_t* order, void* stream);

/* Multi-label NMS, same arithmetic as maskrcnn_benchmark/csrc/cuda/ml_nms.cu (bit-identical kept set):
 *   boxes [n,4] f32 xyxy, scores [n] f32, labels [n] f32, order int64 [n] = indices by score descending.
 *   keep_out int64 [n] receives the kept ORIGINAL indices ascending, *num_keep (device int32) the count.
 *   max_det > 0 additionally applies the `score >= kth-largest kept score` cut of rpn/inference.py:757-767.
 *   workspace: mqdet_ml_nms_workspace_bytes(n) bytes.  No host sync, no D2H.  n <= 16384. */
int64_t mqdet_ml_nms_workspace_bytes(int64_t n);
int mqdet_ml_nms(const float* boxes, const float* scores, const float* labels, const int64_t* order, int64_t n,
                 float thresh, int64_t max_det, int64_t* keep_out, int32_t* num_keep, void* workspace, void* stream);

/* ---- DyHead vision path (vldyhead.py DyConv.forward :205-247) -------------------------------------------------
 * All FPN levels of an image are rows of one fp16 tensor x[B][N][C] (N = sum_l H_l*W_l, level l at row offset
 * off_l, row-major).  level_hw: HOST int32 [nlev][2] = (H_l, W_l). */
#define MQDET_MAX_LEVELS 8

/* DCNv2 sampling stage (deform_conv_kernel_cuda.cu:578-641) -> fp16 column matrix [B*rows][9*C], k = tap*C + c.
 *   branch 1: level l -> l (stride 1; rows = N)            DyConv[1]
 *   branch 2: level l-1 -> l (stride 2; rows = N - H0*W0)  DyConv[2]
 *   branch 0: level l+1 at its own size, offsets/mask of level l re-read through the OUTPUT strides (the
 *             reinterpretation quirk, deform_conv_kernel_cuda.cu:605-618; rows = N - H0*W0)   DyConv[0]
 *   om: fp32 [B][N][om_ld] pixel-major offset-conv output (18 offsets (dh,dw per tap) + 9 mask logits, sigmoid
 *       applied here); NULL -> plain 3x3 convolution sampling. */
int mqdet_dcn_cols(const void* x, const float* om, int64_t om_ld, const int32_t* level_hw, int64_t nlev, int64_t B,
                   int64_t C, int branch, void* cols, void* stream);

/* The same DCNv2 convolutions as ONE implicit GEMM on the tensor cores, without the column matrix (replaces
 * mqdet_dcn_cols + mqdet_gemm_f16 for modulated_deform_conv_cuda_forward, deform_conv_cuda.cu:493-690 inference path):
 *   y[j][B*rows_j][256] (f16) = sampled_cols_j[B*rows_j][9*256] * weight[j][256][9*256]^T + bias[j]       j < njobs <= 3
 * branch[j] selects the sampling geometry exactly as in mqdet_dcn_cols; all jobs share x / om and run in one launch.
 * branch, weight, bias, y: HOST arrays of njobs entries (device pointers inside; bias[j] may be NULL). */
#define MQDET_DCN_MAX_JOBS 3
int mqdet_dcn_conv(const void* x, const float* om, int64_t om_ld, const int32_t* level_hw, int64_t nlev, int64_t B,
                   int64_t C, int64_t njobs, const int32_t* branch, const void* const* weight, const float* const* bias,
                   void* const* y, void* stream);

/* Plain 3x3 / pad 1 / stride 1 convolution with O <= 32 output channels over all levels at once, no column matrix: the
 * offset/mask conv of DyConv (`self.offset`, vldyhead.py:150-153,207-210).  x [B,N,256] f16 (levels concatenated),
 * w [O][9*256] f16 with k = tap*256 + c (tap = ky*3 + kx), bias [O] f32 -> out [B*N, ld] f32 (columns 0..O-1 written). */
int mqdet_conv3x3_small(const void* x, const void* w, const float* bias, const int32_t* level_hw, int64_t nlev, int64_t B,
                        int64_t C, int64_t O, float* out, int64_t ld, void* stream);

/* Per-(image, segment) per-channel partial sums (sum, sum of squares, row-weighted sum) of fp16 y [B][rows][C].
 * seg_off_dev: DEVICE int32 [nseg+1] row offsets; partial: mqdet_chan_stats_floats(B, nseg, C) floats. */
int64_t mqdet_chan_stats_floats(int64_t B, int64_t nseg, int64_t C);
int mqdet_chan_stats(const void* y, const int32_t* seg_off_dev, int64_t nseg, int64_t B, int64_t rows_per_img, int64_t C,
                     const float* row_weights, float* partial, void* stream);

/* GroupNorm(groups) affine + scale-attention scalar per (image, segment) from the partial sums (vldyhead.py:226-238):
 * affine [B][nseg][2][C] (GN(y) = a*y + b), attn [B][nseg] = h_sigmoid(relu(attn_w . GAP(GN(y)) + attn_b)). */
int mqdet_gn_attn(const float* partial, const int32_t* seg_off_dev, int64_t nseg, int64_t B, int64_t C, int64_t groups,
                  int weighted, const float* gn_w, const float* gn_b, float eps, const float* attn_w, const float* attn_b,
                  float* affine, float* attn, void* stream);

/* mid = mean_k attn_k * GN_k(y_k), branch 0 bilinearly upsampled (align_corners=True) from the coarser grid.
 * mid_sums (optional): fp32 [B][nlev][mqdet_dyconv_combine_chunks()][C] per-channel sums of the stored (fp16) output over
 * the pixel ranges of each (image, level) — the global average pool DyReLU needs, so `mid` is not read again for it. */
int64_t mqdet_dyconv_combine_chunks(void);
int mqdet_dyconv_combine(const void* y1, const void* y2, const void* y0, const float* aff1, const float* aff2,
                         const float* aff0, const float* at1, const float* at2, const float* at0, const int32_t* level_hw,
                         int64_t nlev, int64_t B, int64_t C, void* mid, float* mid_sums, void* stream);

/* DyReLU (layers/dyrelu.py:80-104): coefficients per (image, level) from partial channel sums of `mid`
 * (partial [B*nseg][chunks][stats][C], statistic 0 = the plain sum: mqdet_chan_stats output has chunks = 32, stats = 3;
 * mqdet_dyconv_combine's mid_sums chunks = mqdet_dyconv_combine_chunks(), stats = 1), then out = max(mid*a1 + b1, mid*a2 + b2). */
int mqdet_dyrelu_coef(const float* partial, int64_t chunks, int64_t stats, const int32_t* seg_off_dev, int64_t nseg, int64_t B,
                      int64_t C, int64_t squeeze, const float* w1, const float* b1, const float* w2, const float* b2,
                      float* coef, void* stream);
int mqdet_dyrelu_apply(const void* mid, const float* coef, const int32_t* level_hw, int64_t nlev, int64_t B, int64_t C,
                       void* out, void* stream);

/* ---- ATSS post-processing (rpn/inference.py:620-769), device-resident, no host synchronisation ------------------
 * logits [B,N,T] (fp16/fp32), reg_ctr [B,N,5] fp32 (4 box deltas before the per-level Scale, 1 centerness logit),
 * tokmap_dev int32 [C][max_tok] token positions of score column c padded with -1 (the positive map) — one table for the
 * batch (tokmap_img_stride 0) or one per image (stride in int32 elements: prompt chunks batched as images); class_labels
 * int32 [C] (labels_img_stride 0) / per image, or NULL: the label of column c is class_labels[c], default c + 1
 * (convert_grounding_to_od_logits / _v2, rpn/inference.py:772-824); level tables on
 * the HOST (level_hw int32 [nlev][2], strides / base_anchors [nlev][4] / reg_scales [nlev] floats).
 * Per (image, level): sigmoid -> class mean -> score > pre_nms_thresh -> rank = score*sigmoid(ctr) -> exact top-k
 * (ties by ascending (location, class)) -> BoxCoder.decode against the generated anchor -> clip -> sqrt(rank).
 * Outputs (row stride out_stride >= nlev*topk per image): per-level blocks out_* at [l*topk, ...), level_counts
 * [B][nlev]; dense concatenation cat_* (level 0 first) with totals[B].  out_key (optional) = level<<40|loc<<12|cls.
 * cand_ws: mqdet_atss_workspace_bytes(...) bytes. */
int64_t mqdet_atss_workspace_bytes(const int32_t* level_hw, int64_t nlev, int64_t C, int64_t B);
int mqdet_atss_candidates(const void* logits, int logits_dtype, const float* reg_ctr, const int32_t* tokmap_dev,
                          int64_t tokmap_img_stride, const int32_t* class_labels, int64_t labels_img_stride, int64_t C,
                          int64_t max_tok, int64_t T, const int32_t* level_hw, int64_t nlev, const float* strides,
                          const float* base_anchors, const float* reg_scales, int64_t B, float pre_nms_thresh, int64_t topk,
                          int64_t out_stride, float img_w, float img_h, void* cand_ws, int32_t* level_counts,
                          float* out_boxes, float* out_scores, float* out_labels, int64_t* out_key, float* cat_boxes,
                          float* cat_scores, float* cat_labels, int32_t* totals, void* stream);

/* Batched multi-label NMS: rows of n_max (multiple of 256) candidates per image, counts on the device. */
int64_t mqdet_ml_nms_batched_workspace_bytes(int64_t B, int64_t n_max);
int mqdet_ml_nms_batched(const float* boxes, const float* scores, const float* labels, const int32_t* counts_dev, int64_t B,
                         int64_t n_max, float thresh, int64_t max_det, int64_t* keep_out, int32_t* num_keep, void* workspace,
                         void* stream);

/* det[b][i][0:6] = (x1,y1,x2,y2,score,label) of kept candidate i (< num_keep[b]), zero-padded to max_out rows:
 * the fixed-shape per-image result that is copied to the host / all-gathered over NCCL.  det holds det_rows >= max_out
 * rows per image (0 -> max_out); with det_rows > max_out, row max_out carries (float)num_keep[b] in column 0 so that the
 * detections and their count travel in ONE buffer (one D2H copy, one all-gather). */
int mqdet_gather_detections(const float* boxes, const float* scores, const float* labels, const int64_t* keep,
                            const int32_t* num_keep, int64_t B, int64_t n_max, int64_t max_out, int64_t det_rows, float* det,
                            void* stream);

/* Anchors of one FPN level (anchor_generator.py:72-109): base_anchor (HOST float[4]) shifted by (x*stride, y*stride);
 * visibility (optional uint8) = fully inside the image (STRADDLE_THRESH 0). */
int mqdet_anchors(float* out, uint8_t* visibility, int64_t grid_h, int64_t grid_w, float stride, const float* base_anchor,
                  float img_w, float img_h, void* stream);

/* ---- Swin backbone / FPN glue kernels (modeling/backbone/swint.py, fpn.py) ---------------------------------------
 * Token layout [B][H*W][C] row-major. */
/* PatchEmbed input gather (swint.py:393-431): image fp32 NCHW [B,3,H,W] -> fp16 [B*ceil(H/4)*ceil(W/4), 48]. */
int mqdet_patchify4(const float* img, int64_t B, int64_t H, int64_t W, void* out, void* stream);
/* (S)W-MSA core (swint.py:111-142,186-242): qkv fp16 [B*H*W, 3C] -> out fp16 [B*H*W, C]; pads to a multiple of the
 * window with qkv_bias rows, cyclic shift + -100 region mask by index math.  bias_pad: fp32 [heads][NP][NP] with
 * NP = window^2 rounded up to 16 (64 / 144) = log2(e) x the relative position bias inside [N][N], -inf outside (scale, bias
 * and the padding of keys / queries are then one FFMA per score; the softmax runs in the log2 domain). */
int mqdet_swin_window_attn(const void* qkv, const float* qkv_bias, const float* bias_pad, int64_t B, int64_t H, int64_t W,
                           int64_t heads, int64_t window, int64_t shift, float scale, void* out, void* stream);
/* PatchMerging gather + LayerNorm(4C) (swint.py:256-284): x fp32 [B,H*W,C] -> fp16 [B*ceil(H/2)*ceil(W/2), 4C]. */
int mqdet_patch_merge_ln(const float* x, int64_t B, int64_t H, int64_t W, int64_t C, const float* gamma, const float* beta,
                         float eps, void* out, void* stream);
/* FPN top-down merge (fpn.py:88-95): out = lateral + nearest_upsample(top); fp16 [B,H*W,C] / [B,Hs*Ws,C]. */
int mqdet_upsample_add(const void* lateral, const void* top, int64_t B, int64_t H, int64_t W, int64_t Hs, int64_t Ws,
                       int64_t C, void* out, void* stream);
/* Plain 3x3 / pad 1 / stride {1,2} im2col of fp16 NHWC [B][H*W][C] (batch stride in elements) -> [B*Ho*Wo][9C]. */
int mqdet_im2col3x3(const void* x, int64_t x_batch_stride, int64_t B, int64_t H, int64_t W, int64_t C, int64_t stride,
                    int relu_in, void* cols, void* stream);
/* AvgPool2d(2) of every pyramid level + concat (generalized_vl_rcnn_new.py:291-293): fp16 [B,N,C] -> fp32 [B,I,C]. */
int mqdet_avgpool2_levels(const void* x, const int32_t* level_hw, int64_t nlev, int64_t B, int64_t C, float* out, void* stream);

/* ---- vision-query extraction (GeneralizedVLRCNN_New.extract_query, generalized_vl_rcnn_new.py:232-288) ----------------
 * Pooler (modeling/poolers.py:46-129): FPN level of every box by LevelMapper (:11-43) + ROIAlignV2 of that level
 * (torchvision roi_align, aligned = True, sampling_ratio 0 = adaptive) over the fp16 pyramid x [B][N][C] (levels concatenated).
 * rois [R][5] = (image index, x1, y1, x2, y2) fp32 in image pixels; scales HOST float [nlev] (POOLER_SCALES).
 * mean_only != 0: out [R][C] = mean over the pooled x pooled bins (query_feats.mean(dim=[-2,-1]), :263);
 * otherwise out [R][C][pooled][pooled] fp32.  level_out int32 [R] optional. */
int mqdet_roi_align_levels(const void* x, const int32_t* level_hw, int64_t nlev, const float* scales, int64_t B, int64_t C,
                           const float* rois, int64_t R, int64_t pooled, int64_t sampling_ratio, int mean_only, float* out,
                           int32_t* level_out, void* stream);

/* ---- GroundingDINO: multi-scale deformable attention forward (groundingdino_new/models/GroundingDINO/ms_deform_attn.py:93-133,
 * 285-331; supersedes groundingdino_new._C.ms_deform_attn_forward, csrc_groundingdino/vision.cpp:53-56) ---------------------------
 * value [B][Nv][heads*32] f16 (projected, masked rows zero; levels concatenated in level_hw order); proj [B*Q][proj_ld] f32 =
 * the raw Linear outputs: sampling offsets at column ((h*L + l)*P + p)*2 + {x, y}, attention logits at aw_col0 + (h*L + l)*P + p;
 * ref [B][Q][L][ref_dim] f32 normalised reference points (ref_dim 2) or boxes (4).  Per (image, query, head): softmax over the
 * L*P logits, sampling locations, bilinear samples (zero padding, align_corners=False), weighted sum -> out [B*Q][heads*32]. */
int mqdet_ms_deform_attn(const void* value, const float* proj, int64_t proj_ld, int64_t aw_col0, const float* ref, int64_t ref_dim,
                         const int32_t* level_hw, int64_t nlev, int64_t B, int64_t Q, int64_t heads, int64_t head_dim,
                         int64_t points, void* out, int out_dtype, void* stream);

/* ---- GroundingDINO variant, small device ops (SURVEY.md §8 f1) --------------------------------------------------
 * STABLE_SOFTMAX_2D of BiMultiHeadAttention (groundingdino_new/models/GroundingDINO/fuse_modules.py:177-187): the global
 * maximum of the score tensor is subtracted before the +-5e4 clamps.
 *   mqdet_global_max_f32 : out[0] = max_i x[i] (two deterministic launches; workspace: mqdet_global_max_workspace_floats())
 *   mqdet_shift_clamp_f32: x[i] = clamp(x[i] - *shift, lo, hi) in place, shift a DEVICE scalar (no host sync) */
int64_t mqdet_global_max_workspace_floats(void);
int mqdet_global_max_f32(const float* x, int64_t n, float* out, float* workspace, void* stream);
/* the same shift + clamps fused into the row softmax (one pass less over the scores): y = softmax_j(clamp(x - *shift_dev, lo, hi) + mask),
 * fp32 rows of n == n_pad == 256 (image -> text side) or n >= 4096 (text -> image side); mask arguments as mqdet_softmax_rows */
/* reduction of a split-K product whose K slices ran as an extra batch dimension of mqdet_gemm_f16: part f32 [nb2][nb1][S][R][C] ->
 * out16[z2 * o_s2 + z1 * o_s1 + r * ldo + c] = f16(sum_s part[z2][z1][s][r][c]); C % 4 == 0 */
int mqdet_sum_splits_cast(const float* part, int64_t nb2, int64_t nb1, int64_t S, int64_t R, int64_t C, void* out16, int64_t o_s2, int64_t o_s1,
                          int64_t ldo, void* stream);
int mqdet_softmax_rows_shifted_supported(int64_t n, int64_t n_pad);
int mqdet_softmax_rows_shifted(const float* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int64_t n, int64_t n_pad,
                               const float* shift_dev, float lo, float hi, const float* colmask, int64_t rows_per_batch, float mask_value,
                               float keep_add, void* stream);
int mqdet_shift_clamp_f32(float* x, int64_t n, const float* shift, float lo, float hi, void* stream);
/* Two-stage query selection (transformer.py:288-318): topk_logits = enc_outputs_class.max(-1)[0]; torch.topk(.., 900, dim=1);
 * torch.gather of the selected rows.
 *   mqdet_row_max_f32   : out[r] = max_j x[r*ld + j], j < D
 *   mqdet_topk_desc     : idx_out[b][0..k) = indices of the k largest of keys[b][0..n), by (value descending, index ascending);
 *                         k <= min(n, 1024); one CTA per image (radix select + ordered tie fill + bitonic sort)
 *   mqdet_gather_rows_f32: dst[b][i][0..D) = act(src[b][idx[b][i]][0..D)), act = identity (sigmoid == 0) or the logistic sigmoid */
int mqdet_row_max_f32(const float* x, int64_t rows, int64_t D, int64_t ld, float* out, void* stream);
int mqdet_topk_desc(const float* keys, int64_t B, int64_t n, int64_t k, int64_t* idx_out, void* stream);
int mqdet_gather_rows_f32(const float* src, const int64_t* idx, int64_t B, int64_t rows_src, int64_t k, int64_t D, int sigmoid,
                          float* dst, void* stream);

/* ---- GroundingDINO encoder / decoder assembly (SURVEY.md §8 f1, BASELINE config 4): the device ops that are not GEMMs, LayerNorms,
 * softmaxes or ms_deform_attn -----------------------------------------------------------------------------------------------
 *   mqdet_add_cast       : out = (a + b) * rowgate[row]  (b, rowgate optional; a gated-off row is exactly 0) -> f16 and / or f32.
 *                          with_pos_embed of groundingdino_new/models/GroundingDINO/transformer.py:738,843-870 and the masked
 *                          memory of gen_encoder_output_proposals (utils.py:110-112).  D % 4 == 0, 16-byte aligned pointers.
 *   mqdet_groupnorm_rows : nn.GroupNorm(groups, C) over x [B][HW][C] (f16 | f32 rows, channel-contiguous): input_proj =
 *                          Conv2d + GroupNorm(32, 256) (groundingdino.py:214-236).  workspace: mqdet_groupnorm_rows_workspace_floats.
 *   mqdet_box_refine_sine: decoder box refinement + conditional-query embedding (transformer.py:636-650,688-700):
 *                            ref = delta ? sigmoid(delta + (ref_is_logit ? ref_in : inverse_sigmoid(ref_in)))   (util/misc.py:721-725)
 *                                        : (ref_is_logit ? sigmoid(ref_in) : ref_in)
 *                            ref_input[b][q][l] = ref * (vr[b][l].x, vr[b][l].y, vr[b][l].x, vr[b][l].y)
 *                            sine16[b][q][512]  = gen_sineembed_for_position(ref_input[:, :, 0, :])  (utils.py:203-232), optional
 *                          delta [B*nq][ldd] f32 or NULL; ref_in / ref_out [B*nq][4]; valid_ratios [B][L][2]; ref_out optional.
 *   mqdet_gdino_detections: convert_groundingdino_to_glip_output (groundingdino.py:291-335) for raw class logits [B][nq][T] f32
 *                          (-inf on padding): sigmoid, per-class mean over its tokens (tokmap int32 [C][max_tok], -1 padded),
 *                          best class (lowest index on ties), keep if score > box_threshold, boxes cxcywh (normalised) -> xyxy in
 *                          pixels of img_wh[b] = (W, H), clipped to [0, W-1] x [0, H-1], boxes with a negative side dropped; kept rows in
 *                          query order -> out [B][max_out + 1][6] = (x1, y1, x2, y2, score, label), row max_out = (count, 0, ...);
 *                          workspace: mqdet_gdino_detections_workspace_floats. */
int mqdet_add_cast(const float* a, const float* b, const float* rowgate, int64_t rows, int64_t D, void* out16, float* out32,
                   void* stream);
int64_t mqdet_groupnorm_rows_workspace_floats(int64_t B, int64_t C);
int mqdet_groupnorm_rows(const void* x, int x_dtype, int64_t B, int64_t HW, int64_t C, int64_t groups, const float* gamma,
                         const float* beta, float eps, void* out16, float* out32, float* workspace, void* stream);
int mqdet_box_refine_sine(const float* delta, int64_t ldd, const float* ref_in, int ref_is_logit, const float* valid_ratios, int64_t B,
                          int64_t nq, int64_t L, float* ref_out, float* ref_input, void* sine16, void* stream);
int64_t mqdet_gdino_detections_workspace_floats(int64_t B, int64_t nq);
int mqdet_gdino_detections(const float* logits, int64_t T, const float* boxes, const int32_t* tokmap, int64_t C, int64_t max_tok,
                           const float* img_wh, float box_threshold, int64_t B, int64_t nq, int64_t max_out, float* out,
                           float* workspace, void* stream);

/* ---- Training side of the modulated pre-training step (SURVEY.md §8 f2, BASELINE config 5): backward of the Gated Class-scalable
 * Perceiver block (modeling_bert_new.py:186-248,298-374; the block's forward is the inference path above), token focal loss,
 * global-norm clipping + AdamW.  The matrix products of the backward are mqdet_gemm_f16 launches (dX = dY W, dW = dY^T X with both
 * operands transposed to K-major by mqdet_transpose_cast); SURVEY §8(b2)'s `gcp_block_bwd` is their composition in
 * mqdet_b200/modeling/language_backbone/gcp_backward.py. --------------------------------------------------------------------
 *   mqdet_transpose_cast   : out16[c][r] = f16(scale * x[r][c]), x [R][C] (f16 | f32, row stride ld), out row stride ldo >= R; columns
 *                            R..ldo-1 are zero filled (K padding of the weight-gradient products)
 *   mqdet_layernorm_bwd    : nn.LayerNorm backward from the saved INPUT x (+ x2 when given: the two addends of a post-norm residual block)
 *                            [rows][D] f32 and dy f32: dx (= or +=), dgamma, dbeta (optional);
 *                            workspace: mqdet_layernorm_bwd_workspace_floats
 *   mqdet_gelu_bwd         : dz16 = dh * gelu'(z16) (exact erf GELU), dh f16 | f32
 *   mqdet_gcp_gate_bwd     : x1 = s * g + x with g = tanh(h1 . w2) (modeling_bert_new.py:355-361): ds = dx1 * g, dgpre = (sum_d dx1 * s)(1 - g^2),
 *                            dh1 = dgpre * w2 (f16 [rows][Dg])
 *   mqdet_colsum_weighted  : out[j] = sum_r w[r] * h16[r][j]   (d w2 of the gate projection); workspace: mqdet_colsum_weighted_workspace_floats
 *   mqdet_gcp_sparse_attn_bwd: backward of mqdet_gcp_sparse_attn: dq16 [B][T][512]; dkv f32 [B][V+1][1024] ACCUMULATED with atomics (caller
 *                            zero-initialises): K / V gradients land once per unique query row
 *   mqdet_dot_sum          : out[0] = mul * sum_i a[i] * b[i] (b == NULL: a[i]^2), times (1 - tanh(*one_minus_tanh2_of)^2) when given;
 *                            workspace: mqdet_reduce_workspace_floats
 *   mqdet_scale_cast       : out = x * alpha * (tanh?)(*scalar_dev) -> f16 and / or f32
 *   mqdet_token_focal_loss : token_sigmoid_binary_focal_loss (layers/sigmoid_focal_loss.py:127-162) over logits / targets f32 [B][N][T];
 *                            text_mask f32 [B][T] (> 0 = token in use) or NULL; loss_out[0] = sum; dlogits (optional) = grad_scale * d loss
 *   mqdet_sqnorm_partials  : partial sums of x^2 (<= 64 floats written, count returned through *partials_written, a HOST pointer)
 *   mqdet_clip_coef        : coef2[0] = min(1, max_norm / (sqrt(sum partials) + 1e-6)), coef2[1] = the norm (clip_grad_norm_)
 *   mqdet_adamw_step       : torch.optim.AdamW update of one tensor, gradient scaled by *grad_scale_dev (the clip coefficient) */
int mqdet_transpose_cast(const void* x, int x_dtype, int64_t R, int64_t C, int64_t ld, float scale, void* out16, int64_t ldo, void* stream);
int64_t mqdet_layernorm_bwd_workspace_floats(int64_t rows, int64_t D);
int mqdet_layernorm_bwd(const float* dy, const float* x, const float* x2, const float* gamma, float eps, int64_t rows, int64_t D, float* dx,
                        int accumulate, float* dgamma, float* dbeta, float* workspace, void* stream);
/* batched form: input z = z1 + nb1 * z2 at x + z1 * x_s1 + z2 * x_s2 (element strides), outputs contiguous [nb2][nb1][C][ldo] */
int mqdet_transpose_cast_batched(const void* x, int x_dtype, int64_t nb1, int64_t nb2, int64_t x_s1, int64_t x_s2, int64_t R, int64_t C,
                                 int64_t ld, float scale, void* out16, int64_t ldo, void* stream);
/* softmax backward over rows: ds16[r][j] = scale * p16[r][j] * (dp[r][j] - sum_k p16[r][k] dp[r][k]), j < n; columns n..n_pad-1 zero */
int mqdet_softmax_bwd_rows(const void* p16, int64_t ldp, const float* dp, int64_t ldd, int64_t rows, int64_t n, int64_t n_pad, float scale,
                           void* ds16, int64_t lds, void* stream);
int mqdet_gelu_bwd(const void* z16, const void* dh, int dh_dtype, int64_t n, void* dz16, void* stream);
int mqdet_gcp_gate_bwd(const float* dx1, const float* s, const float* g, const float* w2, int64_t rows, int64_t D, int64_t Dg, float* ds,
                       float* dgpre, void* dh1_16, void* stream);
int64_t mqdet_colsum_weighted_workspace_floats(int64_t C);
int mqdet_colsum_weighted(const void* h16, const float* w, int64_t rows, int64_t C, float* out, float* workspace, void* stream);
int mqdet_gcp_sparse_attn_bwd(const void* q16, const void* kv16, const int32_t* idx, const void* dout16, int64_t B, int64_t T, int64_t V,
                              int64_t S, int64_t H, int64_t Dh, void* dq16, float* dkv, void* stream);
int64_t mqdet_reduce_workspace_floats(void);
int mqdet_dot_sum(const float* a, const float* b, int64_t n, const float* one_minus_tanh2_of, float mul, float* out, float* workspace,
                  void* stream);
int mqdet_scale_cast(const float* x, const float* scalar_dev, int tanh_scalar, float alpha, int64_t n, void* out16, float* out32,
                     void* stream);
int mqdet_token_focal_loss(const float* logits, const float* targets, const float* text_mask, float alpha, float gamma, int64_t B, int64_t N,
                           int64_t T, float grad_scale, float* loss_out, float* dlogits, float* workspace, void* stream);
int mqdet_sqnorm_partials(const float* x, int64_t n, float* partial_out, int64_t max_partials, int64_t* partials_written, void* stream);
int mqdet_clip_coef(const float* partials, int64_t count, float max_norm, float* coef2, void* stream);
int mqdet_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float beta1, float beta2,
                     float eps, float weight_decay, int64_t step, const float* grad_scale_dev, void* stream);

/* ---- ATSS target assignment and the pre-training detection losses (modeling/rpn/loss.py ATSSLossComputation :519-1201) ---------
 * One anchor per location, generated from the level table (level_hw [nlev][2], strides [nlev], base_anchors [nlev][4]) exactly as
 * mqdet_atss_candidates does.  GTs come as a fixed-capacity pack: gt_boxes f32 [B][Gmax][4] (xyxy), gt_labels i32 [B][Gmax],
 * gt_count i32 [B] (device; entries >= gt_count[b] are ignored), gt_tokens f32 [B][Gmax][T] (the positive_map rows).
 *   mqdet_atss_assign : match i32 [B][N] = assigned GT or -1; img_stats f32 [B][2] (optional) = (positives, sum of centerness targets)
 *                       per image; norm f32 [4] = the batch totals twice: [0:2] is what data-parallel ranks all-reduce (sum) before
 *                       mqdet_atss_loss, [2:4] stays this rank's.  Per-level top-k ties go to the lower anchor index; an anchor claimed
 *                       by several GTs goes to the highest IoU, then the lowest GT index.  workspace: mqdet_atss_assign_workspace_bytes
 *   mqdet_atss_loss   : losses f32 [4] = (loss_reg, loss_centerness, loss_dot_product_token, loss_cls = 0); d_logits f32 [B][N][T] and
 *                       d_reg_ctr f32 [B][N][5] = their gradient w.r.t. logits [B][N][T] and the raw box / centerness output reg_ctr
 *                       [B][N][5] (channels 0-3 before the per-level Scale reg_scales [nlev]); text_mask f32 [B][T] (> 0 = in use) or
 *                       NULL; world = number of ranks that summed norm[0:2].  No host synchronisation; reductions are deterministic.
 *                       workspace: mqdet_atss_loss_workspace_floats */
int64_t mqdet_atss_assign_workspace_bytes(int64_t B, int64_t N);
int mqdet_atss_assign(const float* gt_boxes, const int32_t* gt_labels, const int32_t* gt_count, int64_t B, int64_t Gmax,
                      const int32_t* level_hw, int64_t nlev, const float* strides, const float* base_anchors, int64_t topk, void* workspace,
                      int32_t* match, float* img_stats, float* norm, void* stream);
int64_t mqdet_atss_loss_workspace_floats(int64_t B, int64_t N);
int mqdet_atss_loss(const float* logits, const float* reg_ctr, const int32_t* match, const float* gt_boxes, const int32_t* gt_labels,
                    const float* gt_tokens, int64_t B, int64_t Gmax, int64_t T, const float* text_mask, const int32_t* level_hw, int64_t nlev,
                    const float* strides, const float* base_anchors, const float* reg_scales, const float* norm, float world, float alpha,
                    float gamma, float reg_weight, float token_weight, float* workspace, float* losses, float* d_logits, float* d_reg_ctr,
                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MQDET_B200_H_ */
