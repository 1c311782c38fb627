// mqdet_b200 — ATSS post-processing on the device: token logits -> class scores -> candidates -> top-k -> decode.
//
// Reference: maskrcnn_benchmark/modeling/rpn/inference.py ATSSPostProcessor.forward_for_single_feature_map :620-712,
//            convert_grounding_to_od_logits :772-790, BoxCoder.decode (modeling/rpn/vldyhead.py:78-108),
//            AnchorGenerator.grid_anchors (modeling/rpn/anchor_generator.py:72-94), BoxList.clip_to_image.
//
//   1. atss_candidates_kernel: one warp per location; sigmoid of the T token logits staged in shared memory, class
//      score = mean over the class's token positions (MEAN aggregation); score > pre_nms_thresh -> candidate with
//      ranking value s = score * sigmoid(centerness); appended (64-bit key) to the (image, level) list.
//      key = orderable(s) << 32 | ~(loc*C + cls): descending key order == (s desc, loc asc, cls asc), all keys unique.
//   2. atss_select_decode_kernel: one CTA per (image, level): exact top-k by 8-pass radix select on the keys
//      (skipped when count <= k), bitonic sort, box decode against the analytically generated anchor, clip, sqrt score.
// Everything is HBM/latency bound integer + fp32 work; no host synchronisation anywhere.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int PP_MAX_T = 256;
constexpr int PP_TOPK_MAX = 1024;

struct PPLevels {
  int n;
  int H[MQDET_MAX_LEVELS], W[MQDET_MAX_LEVELS], off[MQDET_MAX_LEVELS];
  float stride[MQDET_MAX_LEVELS], base[MQDET_MAX_LEVELS][4], reg_scale[MQDET_MAX_LEVELS];
  long cand_off[MQDET_MAX_LEVELS + 1];  // offsets of each level's candidate segment inside one image's buffer
};

__device__ __forceinline__ unsigned int f2ord(float f) {
  unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned int u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

template <typename T>
__global__ void __launch_bounds__(256) atss_candidates_kernel(const T* __restrict__ logits, const float* __restrict__ reg_ctr,
                                                              const int* __restrict__ tokmap, long tokmap_img_stride, int C,
                                                              int max_tok, int Tn, PPLevels lv, int B, float thresh,
                                                              unsigned long long* __restrict__ cand, int* __restrict__ counts,
                                                              long cand_per_img) {
  __shared__ float sig[8][PP_MAX_T];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int N = lv.off[lv.n - 1] + lv.H[lv.n - 1] * lv.W[lv.n - 1];
  const long gw = (long)blockIdx.x * 8 + wib;
  if (gw >= (long)B * N) return;
  const int b = (int)(gw / N), pn = (int)(gw % N);
  int l = 0;
  while (l + 1 < lv.n && pn >= lv.off[l + 1]) ++l;
  const T* row = logits + gw * Tn;
  for (int t = lane; t < Tn; t += 32) {
    const float x = (float)row[t];
    sig[wib][t] = 1.f / (1.f + expf(-x));
  }
  __syncwarp();
  const float cs = 1.f / (1.f + expf(-reg_ctr[gw * 5 + 4]));
  const int loc = pn - lv.off[l];
  for (int c = lane; c < C; c += 32) {
    const int* tm = tokmap + (long)b * tokmap_img_stride + c * max_tok;
    float s = 0.f;
    int n = 0;
    for (int j = 0; j < max_tok; ++j) {
      const int t = tm[j];
      if (t >= 0) {
        s += sig[wib][t];
        ++n;
      }
    }
    const float score = (n > 0) ? s / (float)n : 0.f;  // label absent from the positive map: score stays 0 (:773)
    const bool hit = score > thresh;
    // warp-aggregated append: one atomic per warp and class stripe instead of one per candidate
    const unsigned ball = __ballot_sync(__activemask(), hit);
    if (ball) {
      const unsigned act = __activemask();
      const int leader = __ffs(ball) - 1;
      int base = 0;
      if (lane == leader) base = atomicAdd(&counts[b * lv.n + l], __popc(ball));
      base = __shfl_sync(act, base, leader);
      if (hit) {
        const float rank = score * cs;
        const int slot = base + __popc(ball & ((1u << lane) - 1));
        const unsigned int idx = (unsigned int)(loc * C + c);
        cand[(long)b * cand_per_img + lv.cand_off[l] + slot] = ((unsigned long long)f2ord(rank) << 32) | (unsigned int)(~idx);
      }
    }
  }
}

// One CTA (1024 threads) per (image, level).
__global__ void __launch_bounds__(1024) atss_select_decode_kernel(const unsigned long long* __restrict__ cand,
                                                                  const int* counts,
                                                                  const float* __restrict__ reg_ctr, PPLevels lv, int C,
                                                                  const int* __restrict__ class_labels, long labels_img_stride,
                                                                  int topk, float img_w, float img_h, long cand_per_img,
                                                                  int out_per_img, float* __restrict__ out_boxes,
                                                                  float* __restrict__ out_scores,
                                                                  float* __restrict__ out_labels,
                                                                  long long* __restrict__ out_key,
                                                                  int* out_counts) {
  __shared__ unsigned long long keys[PP_TOPK_MAX];
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_k, s_fill;
  const int b = blockIdx.x / lv.n, l = blockIdx.x % lv.n;
  const int N = lv.off[lv.n - 1] + lv.H[lv.n - 1] * lv.W[lv.n - 1];
  const unsigned long long* src = cand + (long)b * cand_per_img + lv.cand_off[l];
  const int n = counts[b * lv.n + l];
  const int k = min(n, topk);
  const int tid = threadIdx.x;
  unsigned long long thr = 0;  // select keys >= thr
  if (n > topk) {
    // exact k-th largest key by MSB-first 8-bit radix select (keys are unique)
    if (tid == 0) {
      s_prefix = 0;
      s_k = k;
    }
    for (int d = 7; d >= 0; --d) {
      if (tid < 256) hist[tid] = 0;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      const unsigned long long pmask = (d == 7) ? 0ull : (~0ull << ((d + 1) * 8));
      for (int i = tid; i < n; i += 1024) {
        const unsigned long long key = src[i];
        if ((key & pmask) == prefix) atomicAdd(&hist[(key >> (d * 8)) & 0xff], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        int need = s_k, bsel = 0;
        for (int v = 255; v >= 0; --v) {
          const int h = (int)hist[v];
          if (need <= h) {
            bsel = v;
            break;
          }
          need -= h;
        }
        s_k = need;
        s_prefix = prefix | ((unsigned long long)bsel << (d * 8));
      }
      __syncthreads();
    }
    thr = s_prefix;
  }
  if (tid == 0) s_fill = 0;
  for (int i = tid; i < PP_TOPK_MAX; i += 1024) keys[i] = 0ull;  // 0 sorts last (descending)
  __syncthreads();
  for (int i = tid; i < n; i += 1024) {
    const unsigned long long key = src[i];
    if (key >= thr) {
      const int slot = atomicAdd(&s_fill, 1);
      if (slot < PP_TOPK_MAX) keys[slot] = key;
    }
  }
  __syncthreads();
  // bitonic sort, descending
  for (int kk = 2; kk <= PP_TOPK_MAX; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      const int i = tid, ixj = i ^ j;
      if (ixj > i) {
        const unsigned long long a = keys[i], c = keys[ixj];
        const bool desc = ((i & kk) == 0);
        if ((a < c) == desc) {
          keys[i] = c;
          keys[ixj] = a;
        }
      }
      __syncthreads();
    }
  }
  // decode the first k entries
  const int Wl = lv.W[l];
  const long obase = (long)b * out_per_img + (long)l * topk;
  if (tid < k) {
    const unsigned long long key = keys[tid];
    const float rank = ord2f((unsigned int)(key >> 32));
    const unsigned int idx = ~(unsigned int)(key & 0xffffffffu);
    const int loc = (int)(idx / (unsigned int)C), cls = (int)(idx % (unsigned int)C);
    const float* r = reg_ctr + ((long)b * N + lv.off[l] + loc) * 5;
    const float sc = lv.reg_scale[l];
    // anchor (anchor_generator.py:111-137): base window shifted by (x*stride, y*stride)
    const float sx = (float)(loc % Wl) * lv.stride[l], sy = (float)(loc / Wl) * lv.stride[l];
    const float ax1 = sx + lv.base[l][0], ay1 = sy + lv.base[l][1], ax2 = sx + lv.base[l][2], ay2 = sy + lv.base[l][3];
    const DecodedBox d = box_decode(r[0] * sc, r[1] * sc, r[2] * sc, r[3] * sc, ax1, ay1, ax2, ay2);
    float x1 = d.x1, y1 = d.y1, x2 = d.x2, y2 = d.y2;
    // clip_to_image(remove_empty=False), TO_REMOVE = 1
    x1 = fminf(fmaxf(x1, 0.f), img_w - 1.f);
    y1 = fminf(fmaxf(y1, 0.f), img_h - 1.f);
    x2 = fminf(fmaxf(x2, 0.f), img_w - 1.f);
    y2 = fminf(fmaxf(y2, 0.f), img_h - 1.f);
    float* ob = out_boxes + (obase + tid) * 4;
    ob[0] = x1; ob[1] = y1; ob[2] = x2; ob[3] = y2;
    out_scores[obase + tid] = sqrtf(rank);
    // label of score column `cls`: cls + 1 (convert_grounding_to_od_logits :772-790) unless a label table is given (prompt
    // chunks of a many-category vocabulary: the columns of a chunk are its classes in ascending label order)
    out_labels[obase + tid] = class_labels ? (float)class_labels[(long)b * labels_img_stride + cls] : (float)(cls + 1);
    if (out_key) out_key[obase + tid] = ((long long)l << 40) | ((long long)loc << 12) | (long long)cls;
  }
  if (tid == 0) out_counts[b * lv.n + l] = k;
}

// Compacts the per-level top-k blocks of every image into one dense candidate list per image (cat_boxlist order:
// level 0 first) and records the per-image totals.
__global__ void atss_concat_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                   const float* __restrict__ labels, const int* __restrict__ lvl_counts, int nlev, int topk,
                                   int out_per_img, float* __restrict__ cboxes, float* __restrict__ cscores,
                                   float* __restrict__ clabels, int* __restrict__ totals) {
  const int b = blockIdx.x;
  int offs[MQDET_MAX_LEVELS + 1];
  offs[0] = 0;
  for (int l = 0; l < nlev; ++l) offs[l + 1] = offs[l] + lvl_counts[b * nlev + l];
  if (threadIdx.x == 0) totals[b] = offs[nlev];
  for (int l = 0; l < nlev; ++l) {
    const int cnt = offs[l + 1] - offs[l];
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      const long src = (long)b * out_per_img + (long)l * topk + i;
      const long dst = (long)b * out_per_img + offs[l] + i;
      cboxes[dst * 4 + 0] = boxes[src * 4 + 0];
      cboxes[dst * 4 + 1] = boxes[src * 4 + 1];
      cboxes[dst * 4 + 2] = boxes[src * 4 + 2];
      cboxes[dst * 4 + 3] = boxes[src * 4 + 3];
      cscores[dst] = scores[src];
      clabels[dst] = labels[src];
    }
  }
}

// anchors of one level (anchor_generator.py:72-94) + visibility flag (STRADDLE_THRESH 0, :96-109)
__global__ void anchors_kernel(float* __restrict__ out, unsigned char* __restrict__ vis, int H, int W, float stride, float b0,
                               float b1, float b2, float b3, float img_w, float img_h) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W) return;
  const float sx = (float)(i % W) * stride, sy = (float)(i / W) * stride;
  const float x1 = sx + b0, y1 = sy + b1, x2 = sx + b2, y2 = sy + b3;
  out[i * 4 + 0] = x1; out[i * 4 + 1] = y1; out[i * 4 + 2] = x2; out[i * 4 + 3] = y2;
  if (vis) vis[i] = (x1 >= 0.f) && (y1 >= 0.f) && (x2 < img_w) && (y2 < img_h);
}

// det[b][i] = (x1, y1, x2, y2, score, label) of the i-th kept candidate (ascending candidate index), i < num_keep[b]
__global__ void gather_detections_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                         const float* __restrict__ labels, const long long* __restrict__ keep,
                                         const int* __restrict__ num_keep, int n_max, int max_out, int det_rows,
                                         float* __restrict__ det) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= det_rows) return;
  float* d = det + ((long)b * det_rows + i) * 6;
  if (i == max_out) {  // packed result: the count rides in the row after the detections (one buffer -> one D2H / one all-gather)
    d[0] = (float)num_keep[b];
    d[1] = d[2] = d[3] = d[4] = d[5] = 0.f;
  } else if (i > max_out) {
    d[0] = d[1] = d[2] = d[3] = d[4] = d[5] = 0.f;
  } else if (i < num_keep[b]) {
    const long long k = keep[(long)b * n_max + i];
    const float* bx = boxes + ((long)b * n_max + k) * 4;
    d[0] = bx[0]; d[1] = bx[1]; d[2] = bx[2]; d[3] = bx[3];
    d[4] = scores[(long)b * n_max + k];
    d[5] = labels[(long)b * n_max + k];
  } else {
    d[0] = d[1] = d[2] = d[3] = d[4] = d[5] = 0.f;
  }
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_gather_detections(const float* boxes, const float* scores, const float* labels, const int64_t* keep,
                                       const int32_t* num_keep, int64_t B, int64_t n_max, int64_t max_out, int64_t det_rows,
                                       float* det, void* stream) {
  MQ_REQUIRE(boxes && scores && labels && keep && num_keep && det && B > 0 && max_out > 0, "gather_detections: bad args");
  if (det_rows <= 0) det_rows = max_out;
  MQ_REQUIRE(det_rows >= max_out, "gather_detections: det_rows %ld < max_out %ld", (long)det_rows, (long)max_out);
  gather_detections_kernel<<<dim3((unsigned)((det_rows + 127) / 128), (unsigned)B), 128, 0, (cudaStream_t)stream>>>(
      boxes, scores, labels, (const long long*)keep, num_keep, (int)n_max, (int)max_out, (int)det_rows, det);
  return check_launch("gather_detections_kernel");
}

static int fill_pp_levels(PPLevels* lv, const int32_t* level_hw, int64_t nlev, const float* strides, const float* base_anchors,
                          const float* reg_scales, int64_t C) {
  if (nlev < 1 || nlev > MQDET_MAX_LEVELS) return -1;
  lv->n = (int)nlev;
  int off = 0;
  long coff = 0;
  for (int l = 0; l < nlev; ++l) {
    lv->H[l] = level_hw[2 * l];
    lv->W[l] = level_hw[2 * l + 1];
    lv->off[l] = off;
    off += lv->H[l] * lv->W[l];
    lv->stride[l] = strides[l];
    for (int k = 0; k < 4; ++k) lv->base[l][k] = base_anchors[4 * l + k];
    lv->reg_scale[l] = reg_scales ? reg_scales[l] : 1.f;
    lv->cand_off[l] = coff;
    coff += (long)lv->H[l] * lv->W[l] * C;
  }
  lv->cand_off[nlev] = coff;
  return off;
}

extern "C" int mqdet_atss_candidates(const void* logits, int logits_dtype, const float* reg_ctr, const int32_t* tokmap_dev,
                                     int64_t tokmap_img_stride, const int32_t* class_labels, int64_t labels_img_stride,
                                     int64_t C, int64_t max_tok, int64_t T, const int32_t* level_hw, int64_t nlev,
                                     const float* strides, const float* base_anchors, const float* reg_scales, int64_t B,
                                     float pre_nms_thresh, int64_t topk, int64_t out_stride, float img_w, float img_h,
                                     void* cand_ws,
                                     int32_t* level_counts, float* out_boxes, float* out_scores, float* out_labels,
                                     int64_t* out_key, float* cat_boxes, float* cat_scores, float* cat_labels,
                                     int32_t* totals, void* stream) {
  MQ_REQUIRE(logits && reg_ctr && tokmap_dev && level_hw && strides && base_anchors && cand_ws && level_counts && out_boxes &&
                 out_scores && out_labels && cat_boxes && cat_scores && cat_labels && totals,
             "atss_candidates: null pointer");
  MQ_REQUIRE(T > 0 && T <= PP_MAX_T, "atss_candidates: T=%ld exceeds %d", (long)T, PP_MAX_T);
  MQ_REQUIRE(topk > 0 && topk <= PP_TOPK_MAX, "atss_candidates: topk=%ld exceeds %d", (long)topk, PP_TOPK_MAX);
  PPLevels lv;
  const int N = fill_pp_levels(&lv, level_hw, nlev, strides, base_anchors, reg_scales, C);
  MQ_REQUIRE(N > 0, "atss_candidates: bad level table");
  MQ_REQUIRE((long)N * C < (1l << 31), "atss_candidates: too many (location, class) pairs");
  cudaStream_t st = (cudaStream_t)stream;
  const long cand_per_img = lv.cand_off[nlev];
  MQ_REQUIRE(out_stride >= nlev * topk, "atss_candidates: out_stride %ld < nlev*topk", (long)out_stride);
  const int out_per_img = (int)out_stride;
  cudaMemsetAsync(level_counts, 0, sizeof(int32_t) * B * nlev, st);
  const long warps = B * (long)N;
  if (logits_dtype == MQDET_F32)
    atss_candidates_kernel<float><<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(
        (const float*)logits, reg_ctr, tokmap_dev, (long)tokmap_img_stride, (int)C, (int)max_tok, (int)T, lv, (int)B, pre_nms_thresh,
        (unsigned long long*)cand_ws, level_counts, cand_per_img);
  else
    atss_candidates_kernel<__half><<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(
        (const __half*)logits, reg_ctr, tokmap_dev, (long)tokmap_img_stride, (int)C, (int)max_tok, (int)T, lv, (int)B, pre_nms_thresh,
        (unsigned long long*)cand_ws, level_counts, cand_per_img);
  int rc = check_launch("atss_candidates_kernel");
  if (rc) return rc;
  // level_counts is rewritten in place with min(count, topk) by the select kernel (it reads the raw count first)
  atss_select_decode_kernel<<<(unsigned)(B * nlev), 1024, 0, st>>>((const unsigned long long*)cand_ws, level_counts, reg_ctr,
                                                                  lv, (int)C, class_labels, (long)labels_img_stride, (int)topk,
                                                                  img_w, img_h, cand_per_img,
                                                                  out_per_img, out_boxes, out_scores, out_labels,
                                                                  (long long*)out_key, level_counts);
  rc = check_launch("atss_select_decode_kernel");
  if (rc) return rc;
  atss_concat_kernel<<<(unsigned)B, 256, 0, st>>>(out_boxes, out_scores, out_labels, level_counts, (int)nlev, (int)topk,
                                                  out_per_img, cat_boxes, cat_scores, cat_labels, totals);
  return check_launch("atss_concat_kernel");
}

extern "C" int64_t mqdet_atss_workspace_bytes(const int32_t* level_hw, int64_t nlev, int64_t C, int64_t B) {
  long n = 0;
  for (int l = 0; l < nlev; ++l) n += (long)level_hw[2 * l] * level_hw[2 * l + 1];
  return n * C * B * 8;
}

extern "C" int mqdet_anchors(float* out, uint8_t* visibility, int64_t grid_h, int64_t grid_w, float stride,
                             const float* base_anchor, float img_w, float img_h, void* stream) {
  MQ_REQUIRE(out && base_anchor && grid_h > 0 && grid_w > 0, "anchors: bad args");
  const int n = (int)(grid_h * grid_w);
  anchors_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(out, visibility, (int)grid_h, (int)grid_w, stride,
                                                                    base_anchor[0], base_anchor[1], base_anchor[2],
                                                                    base_anchor[3], img_w, img_h);
  return check_launch("anchors_kernel");
}
