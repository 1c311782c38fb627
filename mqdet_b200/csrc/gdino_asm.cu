// mqdet_b200 — device ops of the GroundingDINO encoder / decoder assembly (SURVEY.md §8 f1, BASELINE config 4) that are not
// GEMMs, LayerNorms, softmaxes or ms_deform_attn (those reuse the kernels of the GLIP path):
//   * add_cast         : (a + b) * rowgate -> fp16 / fp32       (with_pos_embed, transformer.py:738,843-870; masked memory of
//                        gen_encoder_output_proposals, utils.py:110-112)
//   * groupnorm_rows   : nn.GroupNorm over [B][HW][C] rows      (input_proj = Conv2d + GroupNorm(32, 256), groundingdino.py:214-236)
//   * box_refine_sine  : iterative box refinement + the conditional query's sine embedding of the decoder
//                        (transformer.py:636-650,688-700; utils.py:203-232; util/misc.py:721-725)
//   * gdino_detections : convert_groundingdino_to_glip_output (groundingdino.py:291-335): sigmoid, per-class token mean, best
//                        class, box threshold, cxcywh -> xyxy, clip, ordered compaction into the packed result
// All HBM / latency-bound single-pass kernels; no host synchronisation, no allocation.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) add_cast_kernel(const float4* __restrict__ a, const float4* __restrict__ b,
                                                       const float* __restrict__ rowgate, long n4, int d4,
                                                       uint2* __restrict__ o16, float4* __restrict__ o32) {
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long)gridDim.x * 256) {
    float4 v = a[i];
    if (b) {
      const float4 w = b[i];
      v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
    }
    if (rowgate) {
      const float g = __ldg(rowgate + i / d4);
      // masked_fill semantics: a gated-off row is exactly zero even if the input holds inf / nan
      if (g == 0.f) v = make_float4(0.f, 0.f, 0.f, 0.f);
      else { v.x *= g; v.y *= g; v.z *= g; v.w *= g; }
    }
    if (o32) o32[i] = v;
    if (o16) {
      const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
      uint2 u;
      u.x = *reinterpret_cast<const uint32_t*>(&h0);
      u.y = *reinterpret_cast<const uint32_t*>(&h1);
      o16[i] = u;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// GroupNorm over rows [B][HW][C]: pass 1 = per (image, row chunk, channel) sum / sum of squares (thread = channel, coalesced
// rows), pass 2 = every CTA re-derives the per-channel affine of its image from the partials (double accumulation) and applies it.
constexpr int GN_MAX_CHUNKS = 64;

template <typename T>
__device__ __forceinline__ float gn_ld(const T* p);
template <>
__device__ __forceinline__ float gn_ld<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float gn_ld<__half>(const __half* p) { return __half2float(*p); }

template <typename T>
__global__ void __launch_bounds__(256) gn_partial_kernel(const T* __restrict__ x, int HW, int C, int chunks, float* __restrict__ partial) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const int per = (HW + chunks - 1) / chunks;
  const int r0 = ch * per, r1 = min(HW, r0 + per);
  for (int c = threadIdx.x; c < C; c += 256) {
    float s = 0.f, q = 0.f;
    const T* p = x + ((long)b * HW + r0) * C + c;
    for (int r = r0; r < r1; ++r, p += C) {
      const float v = gn_ld<T>(p);
      s += v;
      q = fmaf(v, v, q);
    }
    float* o = partial + (((long)b * chunks + ch) * C + c) * 2;
    o[0] = s;
    o[1] = q;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) gn_apply_kernel(const T* __restrict__ x, int HW, int C, int groups, int chunks,
                                                       const float* __restrict__ partial, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, float eps, int rows_per_cta,
                                                       __half* __restrict__ o16, float* __restrict__ o32) {
  extern __shared__ double gn_sh[];  // [C] sums, [C] squares, then reused as float scale / shift
  double* ssum = gn_sh;
  double* ssq = gn_sh + C;
  const int b = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += 256) {
    double s = 0.0, q = 0.0;
    for (int ch = 0; ch < chunks; ++ch) {
      const float* p = partial + (((long)b * chunks + ch) * C + c) * 2;
      s += (double)p[0];
      q += (double)p[1];
    }
    ssum[c] = s;
    ssq[c] = q;
  }
  __syncthreads();
  const int cpg = C / groups;
  float sc[4], sf[4];  // C <= 1024
  int nc = 0;
  for (int c = threadIdx.x; c < C; c += 256, ++nc) {
    const int g0 = (c / cpg) * cpg;
    double s = 0.0, q = 0.0;
    for (int j = 0; j < cpg; ++j) {
      s += ssum[g0 + j];
      q += ssq[g0 + j];
    }
    const double n = (double)HW * cpg;
    const double mean = s / n;
    double var = q / n - mean * mean;
    if (var < 0.0) var = 0.0;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    sc[nc] = gamma[c] * rstd;
    sf[nc] = beta[c] - (float)mean * sc[nc];
  }
  const int r0 = blockIdx.x * rows_per_cta, r1 = min(HW, r0 + rows_per_cta);
  for (int r = r0; r < r1; ++r) {
    const long base = ((long)b * HW + r) * C;
    int k = 0;
    for (int c = threadIdx.x; c < C; c += 256, ++k) {
      const float v = fmaf(gn_ld<T>(x + base + c), sc[k], sf[k]);
      if (o32) o32[base + c] = v;
      if (o16) o16[base + c] = __float2half_rn(v);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float inv_sigmoid(float x) {
  x = fminf(fmaxf(x, 0.f), 1.f);
  return logf(fmaxf(x, 1e-3f) / fmaxf(1.f - x, 1e-3f));
}
__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

// warp per (image, query)
__global__ void __launch_bounds__(256) box_refine_sine_kernel(const float* __restrict__ delta, long ldd, const float* __restrict__ ref_in,
                                                              int ref_is_logit, const float* __restrict__ valid_ratios, int nq, int L,
                                                              long total, float* __restrict__ ref_out, float* __restrict__ ref_input,
                                                              __half* __restrict__ sine) {
  const long w = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (w >= total) return;
  const int lane = threadIdx.x & 31;
  const long b = w / nq;
  float r[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float v = __ldg(ref_in + w * 4 + c);
    if (delta) r[c] = sigmoidf_(__ldg(delta + w * ldd + c) + (ref_is_logit ? v : inv_sigmoid(v)));
    else r[c] = ref_is_logit ? sigmoidf_(v) : v;
  }
  if (lane < 4 && ref_out) ref_out[w * 4 + lane] = r[lane];
  const float* vr = valid_ratios + b * L * 2;
  for (int i = lane; i < L * 4; i += 32) {
    const int l = i >> 2, c = i & 3;
    ref_input[(w * L + l) * 4 + c] = r[c] * __ldg(vr + l * 2 + (c & 1));
  }
  if (sine) {
    // gen_sineembed_for_position on reference_points_input[:, :, 0, :]: blocks (y, x, w, h) of 128, sin on even / cos on odd k
    const float vx = __ldg(vr + 0), vy = __ldg(vr + 1);
    const float p[4] = {r[1] * vy, r[0] * vx, r[2] * vx, r[3] * vy};
    for (int j = lane; j < 512; j += 32) {
      const int blk = j >> 7, k = j & 127;
      const float dim_t = powf(10000.f, (float)(2 * (k >> 1)) / 128.f);
      const float ang = p[blk] * 6.283185307179586f / dim_t;
      sine[w * 512 + j] = __float2half_rn((k & 1) ? cosf(ang) : sinf(ang));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Pass 1: warp per (image, query), 16 queries per CTA -> scratch rows [B][nq][7] = (x1, y1, x2, y2, score, label, keep).
// Pass 2: one warp per image compacts the kept rows in query order (boolean-mask indexing) into the packed result.
constexpr int GD_WARPS = 16;
constexpr int GD_MAX_T = 256;

__global__ void __launch_bounds__(GD_WARPS * 32) gdino_score_kernel(const float* __restrict__ logits, int T, const float* __restrict__ boxes,
                                                                    const int* __restrict__ tokmap, long tokmap_img_stride,
                                                                    const int* __restrict__ class_labels, long labels_img_stride,
                                                                    int C, int max_tok, const float* __restrict__ img_wh, float thr,
                                                                    int nq, float* __restrict__ scratch) {
  __shared__ float prob[GD_WARPS][GD_MAX_T];
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * GD_WARPS + warp;
  if (q >= nq) return;
  const float W = img_wh[b * 2], H = img_wh[b * 2 + 1];
  float* pw = prob[warp];
  const float* lg = logits + ((long)b * nq + q) * T;
  for (int t = lane; t < T; t += 32) pw[t] = sigmoidf_(__ldg(lg + t));  // sigmoid(-inf) = 0
  __syncwarp();
  float best = -1.f;
  int best_c = 0x7fffffff;
  for (int c = lane; c < C; c += 32) {
    const int* tm = tokmap + b * tokmap_img_stride + (long)c * max_tok;
    float s = 0.f;
    int n = 0;
    for (int j = 0; j < max_tok; ++j) {
      const int t = tm[j];
      if (t < 0) break;
      s += pw[t];
      ++n;
    }
    const float sc = n ? s / (float)n : 0.f;
    if (sc > best) { best = sc; best_c = c; }  // ascending c within a lane: the first maximum stays
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oc = __shfl_xor_sync(0xffffffffu, best_c, o);
    if (ob > best || (ob == best && oc < best_c)) { best = ob; best_c = oc; }
  }
  if (lane == 0) {
    const float* bx = boxes + ((long)b * nq + q) * 4;
    const float cx = bx[0] * W, cy = bx[1] * H, bw = bx[2] * W, bh = bx[3] * H;
    float x1 = cx - bw / 2.f, y1 = cy - bh / 2.f;
    float x2 = bw + x1, y2 = bh + y1;
    x1 = fminf(fmaxf(x1, 0.f), W - 1.f);
    y1 = fminf(fmaxf(y1, 0.f), H - 1.f);
    x2 = fminf(fmaxf(x2, 0.f), W - 1.f);
    y2 = fminf(fmaxf(y2, 0.f), H - 1.f);
    float* r = scratch + ((long)b * nq + q) * 7;
    // columns of a per-element table are its classes in ascending label order, so the lowest column is also the lowest label
    const int label = class_labels ? class_labels[b * labels_img_stride + best_c] : best_c + 1;
    r[0] = x1; r[1] = y1; r[2] = x2; r[3] = y2; r[4] = best; r[5] = (float)label;
    // candidate_inds = max > box_threshold; remove_small_boxes(min_size=0): w = x2 - x1 + 1 >= 0 (boxlist_ops.py:78-92)
    r[6] = ((best > thr) && (x2 - x1 + 1.f >= 0.f) && (y2 - y1 + 1.f >= 0.f)) ? 1.f : 0.f;
  }
}

__global__ void __launch_bounds__(256) gdino_compact_kernel(const float* __restrict__ scratch, int nq, int max_out, float* __restrict__ out) {
  const int b = blockIdx.x, lane = threadIdx.x & 31;
  float* o = out + (long)b * (max_out + 1) * 6;
  for (int i = threadIdx.x; i < (max_out + 1) * 6; i += blockDim.x) o[i] = 0.f;
  __syncthreads();
  if (threadIdx.x >= 32) return;
  const float* sc = scratch + (long)b * nq * 7;
  int base = 0;
  for (int q0 = 0; q0 < nq; q0 += 32) {
    const int q = q0 + lane;
    const bool k = q < nq && sc[q * 7 + 6] != 0.f;
    const unsigned bal = __ballot_sync(0xffffffffu, k);
    const int pos = base + __popc(bal & ((1u << lane) - 1u));
    if (k && pos < max_out) {
#pragma unroll
      for (int c = 0; c < 6; ++c) o[pos * 6 + c] = sc[q * 7 + c];
    }
    base += __popc(bal);
  }
  if (lane == 0) o[max_out * 6] = (float)base;
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_add_cast(const float* a, const float* b, const float* rowgate, int64_t rows, int64_t D, void* out16,
                              float* out32, void* stream) {
  MQ_REQUIRE(a && (out16 || out32) && rows > 0 && D > 0 && (D % 4) == 0, "add_cast: bad arguments (D must be a multiple of 4)");
  MQ_REQUIRE(((uintptr_t)a & 15) == 0 && ((uintptr_t)b & 15) == 0 && ((uintptr_t)out32 & 15) == 0 && ((uintptr_t)out16 & 7) == 0,
             "add_cast: pointers must be 16-byte aligned");
  const long n4 = rows * D / 4;
  long blocks = (n4 + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  add_cast_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)a, (const float4*)b, rowgate, n4, (int)(D / 4),
                                                                      (uint2*)out16, (float4*)out32);
  return check_launch("add_cast_kernel");
}

extern "C" int64_t mqdet_groupnorm_rows_workspace_floats(int64_t B, int64_t C) { return B * GN_MAX_CHUNKS * C * 2; }

extern "C" int mqdet_groupnorm_rows(const void* x, int x_dtype, int64_t B, int64_t HW, int64_t C, int64_t groups, const float* gamma,
                                    const float* beta, float eps, void* out16, float* out32, float* workspace, void* stream) {
  MQ_REQUIRE(x && gamma && beta && workspace && (out16 || out32), "groupnorm_rows: null pointer");
  MQ_REQUIRE(B > 0 && HW > 0 && C > 0 && C <= 1024 && groups > 0 && (C % groups) == 0, "groupnorm_rows: bad shape (C <= 1024, C %% groups == 0)");
  int chunks = (int)((HW + 63) / 64);
  if (chunks > GN_MAX_CHUNKS) chunks = GN_MAX_CHUNKS;
  const int rows_per_cta = 32;
  const dim3 g1((unsigned)chunks, (unsigned)B), g2((unsigned)((HW + rows_per_cta - 1) / rows_per_cta), (unsigned)B);
  const size_t sh = 2 * (size_t)C * sizeof(double);
  cudaStream_t st = (cudaStream_t)stream;
  if (x_dtype == MQDET_F16) {
    gn_partial_kernel<__half><<<g1, 256, 0, st>>>((const __half*)x, (int)HW, (int)C, chunks, workspace);
    gn_apply_kernel<__half><<<g2, 256, sh, st>>>((const __half*)x, (int)HW, (int)C, (int)groups, chunks, workspace, gamma, beta, eps,
                                                 rows_per_cta, (__half*)out16, out32);
  } else {
    gn_partial_kernel<float><<<g1, 256, 0, st>>>((const float*)x, (int)HW, (int)C, chunks, workspace);
    gn_apply_kernel<float><<<g2, 256, sh, st>>>((const float*)x, (int)HW, (int)C, (int)groups, chunks, workspace, gamma, beta, eps,
                                                rows_per_cta, (__half*)out16, out32);
  }
  return check_launch("groupnorm_rows");
}

extern "C" int mqdet_box_refine_sine(const float* delta, int64_t ldd, const float* ref_in, int ref_is_logit, const float* valid_ratios,
                                     int64_t B, int64_t nq, int64_t L, float* ref_out, float* ref_input, void* sine16, void* stream) {
  MQ_REQUIRE(ref_in && valid_ratios && ref_input && B > 0 && nq > 0 && L > 0 && L <= 8, "box_refine_sine: bad arguments");
  MQ_REQUIRE(!delta || ldd >= 4, "box_refine_sine: delta row stride must be >= 4");
  const long total = B * nq;
  box_refine_sine_kernel<<<cdiv(total, 8), 256, 0, (cudaStream_t)stream>>>(delta, ldd, ref_in, ref_is_logit, valid_ratios, (int)nq, (int)L,
                                                                          total, ref_out, ref_input, (__half*)sine16);
  return check_launch("box_refine_sine_kernel");
}

extern "C" int64_t mqdet_gdino_detections_workspace_floats(int64_t B, int64_t nq) { return B * nq * 7; }

extern "C" int mqdet_gdino_detections(const float* logits, int64_t T, const float* boxes, const int32_t* tokmap,
                                      int64_t tokmap_img_stride, const int32_t* class_labels, int64_t labels_img_stride, int64_t C,
                                      int64_t max_tok, const float* img_wh, float box_threshold, int64_t B, int64_t nq,
                                      int64_t max_out, float* out, float* workspace, void* stream) {
  MQ_REQUIRE(logits && boxes && tokmap && img_wh && out && workspace, "gdino_detections: null pointer");
  MQ_REQUIRE(B > 0 && B <= 65535 && nq > 0 && T > 0 && T <= GD_MAX_T && C > 0 && max_tok > 0 && max_out > 0,
             "gdino_detections: bad shape (T <= 256)");
  MQ_REQUIRE(tokmap_img_stride >= 0 && labels_img_stride >= 0 && (tokmap_img_stride == 0 || tokmap_img_stride >= C * max_tok) &&
             (labels_img_stride == 0 || labels_img_stride >= C) && (class_labels || labels_img_stride == 0),
             "gdino_detections: bad per-element table strides");
  cudaStream_t st = (cudaStream_t)stream;
  gdino_score_kernel<<<dim3((unsigned)((nq + GD_WARPS - 1) / GD_WARPS), (unsigned)B), GD_WARPS * 32, 0, st>>>(
      logits, (int)T, boxes, tokmap, (long)tokmap_img_stride, class_labels, (long)labels_img_stride, (int)C, (int)max_tok, img_wh,
      box_threshold, (int)nq, workspace);
  gdino_compact_kernel<<<(unsigned)B, 256, 0, st>>>(workspace, (int)nq, (int)max_out, out);
  return check_launch("gdino_detections");
}
