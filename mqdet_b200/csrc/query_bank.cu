// mqdet_b200 — the test-time vision-query update (VISION_QUERY.NUM_TURNS; maskrcnn_benchmark/engine/inference.py:383-497).
//
//   query_candidates_kernel : packed detector rows [B][M + 1][6] -> the boxes extract_query pools: score > SCORE_THRESHOLD, grown
//                             by EXPAND_RATIO about their centre (expand_bbox, generalized_vl_rcnn_new.py:32-49), clipped to the
//                             image and the empty ones removed (BoxList.clip_to_image(remove_empty=True)); image-then-row order
//   query_bank_update_kernel: one CTA per label walks the pooled features of its label in arrival order and applies the bank
//                             bookkeeping of extract_query (:268-288, exclude_similar=True): the per-label cap, the cosine test
//                             against every row already in the bank (rows appended earlier in the same call included), the append
//
// Every step reads its counts on the device, so a whole turn of the update runs without a host read.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

// One CTA; images in order, per 1024 rows a ballot scan gives every kept box its slot (row order kept).
__global__ void __launch_bounds__(1024) query_candidates_kernel(const float* __restrict__ packed, int B, int M, float score_thr,
                                                                float ratio, float hi_x, float hi_y, float* __restrict__ rois,
                                                                int* __restrict__ labels, int* __restrict__ count,
                                                                int* __restrict__ bad) {
  __shared__ int warp_tot[32];
  __shared__ int running;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int b = 0; b < B; ++b) {
    const float* rows = packed + (long)b * (M + 1) * 6;
    const float cnt = rows[(long)M * 6];
    const bool ok = cnt >= 0.f && cnt <= (float)M && cnt == floorf(cnt);
    const int n = ok ? (int)cnt : 0;
    if (!ok && threadIdx.x == 0) *bad += 1;
    for (int base = 0; base < n; base += 1024) {
      const int i = base + threadIdx.x;
      int f = 0, lab = 0;
      float x1 = 0.f, y1 = 0.f, x2 = 0.f, y2 = 0.f;
      if (i < n) {
        const float* r = rows + (long)i * 6;
        if (r[4] > score_thr) {
          // expand_bbox: w * ratio, (new - w) / 2, box + (-dw, -dh, dw, dh); one rounded fp32 operation each
          const float bw = __fsub_rn(r[2], r[0]), bh = __fsub_rn(r[3], r[1]);
          const float dw = __fdiv_rn(__fsub_rn(__fmul_rn(bw, ratio), bw), 2.f);
          const float dh = __fdiv_rn(__fsub_rn(__fmul_rn(bh, ratio), bh), 2.f);
          x1 = __fadd_rn(r[0], -dw); y1 = __fadd_rn(r[1], -dh);
          x2 = __fadd_rn(r[2], dw);  y2 = __fadd_rn(r[3], dh);
          // clip_to_image: clamp(min=0, max=size - 1) (NaN stays NaN and fails the test below, as torch.clamp's does)
          x1 = x1 < 0.f ? 0.f : (x1 > hi_x ? hi_x : x1);
          y1 = y1 < 0.f ? 0.f : (y1 > hi_y ? hi_y : y1);
          x2 = x2 < 0.f ? 0.f : (x2 > hi_x ? hi_x : x2);
          y2 = y2 < 0.f ? 0.f : (y2 > hi_y ? hi_y : y2);
          f = (y2 > y1) && (x2 > x1);
          lab = (int)r[5];
        }
      }
      const unsigned ball = __ballot_sync(0xffffffffu, f);
      if (lane == 0) warp_tot[warp] = __popc(ball);
      __syncthreads();
      int woff = 0, tot = 0;
      for (int w = 0; w < 32; ++w) {
        if (w < warp) woff += warp_tot[w];
        tot += warp_tot[w];
      }
      const int start = running;
      if (f) {
        const int pos = start + woff + __popc(ball & ((1u << lane) - 1));
        float* o = rois + (long)pos * 5;
        o[0] = (float)b; o[1] = x1; o[2] = y1; o[3] = x2; o[4] = y2;
        labels[pos] = lab;
      }
      __syncthreads();
      if (threadIdx.x == 0) running = start + tot;
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) *count = running;
}

constexpr int QB_THREADS = 256;
constexpr int QB_WARPS = QB_THREADS / 32;

// ||v||_2 of one C-vector over the CTA in a fixed order: per thread c = t, t + 256, ...; per warp the xor tree; warps 0..7 in order.
__device__ __forceinline__ float block_norm(const float* __restrict__ v, int C, float* red) {
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += QB_THREADS) s = __fadd_rn(s, __fmul_rn(v[c], v[c]));
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < QB_WARPS; ++w) t = __fadd_rn(t, red[w]);
  __syncthreads();
  return sqrtf(t);
}

// Per warp: the normalised dot product of bank row j (norm nb) with x (norm nx), lanes over c = lane, lane + 32, ...
__device__ __forceinline__ float warp_cosine(const float* __restrict__ row, float nb, const float* __restrict__ x, float nx, int C) {
  const float db = fmaxf(nb, 1e-12f), dx = fmaxf(nx, 1e-12f);   // F.normalize: v / max(||v||, eps)
  float s = 0.f;
  for (int c = threadIdx.x & 31; c < C; c += 32) s = __fadd_rn(s, __fmul_rn(__fdiv_rn(row[c], db), __fdiv_rn(x[c], dx)));
  return warp_sum(s);
}

// blockIdx.x = label.  bank [L][cap][C], bank_count [L] (rows in use), row_norm [L][cap] (||row|| of every row in use).
__global__ void __launch_bounds__(QB_THREADS) query_bank_update_kernel(const float* __restrict__ feats, const int* __restrict__ labels,
                                                                       const int* __restrict__ count, int C, int L, int cap,
                                                                       int max_query, float sim_thr, float* __restrict__ bank,
                                                                       int* __restrict__ bank_count, float* __restrict__ row_norm) {
  __shared__ float red[QB_WARPS];
  __shared__ int similar;
  const int lab = blockIdx.x;
  const int n_new = *count;
  int n = bank_count[lab];
  float* rows = bank + (long)lab * cap * C;
  float* norms = row_norm + (long)lab * cap;
  for (int i = 0; i < n_new; ++i) {
    if (labels[i] != lab) continue;
    if (n >= max_query) break;                 // the bank only grows: every later box of this label is skipped too
    const float* x = feats + (long)i * C;
    const float nx = block_norm(x, C, red);
    if (threadIdx.x == 0) similar = 0;
    __syncthreads();
    if (n > 0) {
      for (int j = threadIdx.x >> 5; j < n; j += QB_WARPS) {
        const float s = warp_cosine(rows + (long)j * C, norms[j], x, nx, C);
        if ((threadIdx.x & 31) == 0 && s > sim_thr) similar = 1;
      }
      __syncthreads();
    }
    if (!similar) {
      for (int c = threadIdx.x; c < C; c += QB_THREADS) rows[(long)n * C + c] = x[c];
      if (threadIdx.x == 0) norms[n] = nx;
      ++n;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) bank_count[lab] = n;
}

// row_norm of rows [0, bank_count[label]) of every label (a bank loaded from the host); blockIdx = (row, label).
__global__ void __launch_bounds__(QB_THREADS) query_bank_norms_kernel(const float* __restrict__ bank, const int* __restrict__ bank_count,
                                                                      int C, int cap, float* __restrict__ row_norm) {
  __shared__ float red[QB_WARPS];
  const int j = blockIdx.x, lab = blockIdx.y;
  if (j >= bank_count[lab]) return;
  const float nb = block_norm(bank + ((long)lab * cap + j) * C, C, red);
  if (threadIdx.x == 0) row_norm[(long)lab * cap + j] = nb;
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_query_candidates(const float* packed, int64_t B, int64_t M, float score_thr, float expand_ratio, int64_t img_w,
                                      int64_t img_h, float* rois, int32_t* labels, int64_t cap, int32_t* count, int32_t* bad,
                                      void* stream) {
  MQ_REQUIRE(packed && rois && labels && count && bad, "query_candidates: null pointer");
  MQ_REQUIRE(B > 0 && M > 0 && M <= (1 << 24) && img_w > 0 && img_h > 0 && img_w < (1 << 24) && img_h < (1 << 24),
             "query_candidates: bad sizes B=%ld M=%ld image %ldx%ld", (long)B, (long)M, (long)img_w, (long)img_h);
  MQ_REQUIRE(cap >= B * M && B * M < (1L << 30), "query_candidates: capacity %ld below B * M = %ld", (long)cap, (long)(B * M));
  query_candidates_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(packed, (int)B, (int)M, score_thr, expand_ratio, (float)(img_w - 1),
                                                                (float)(img_h - 1), rois, labels, count, bad);
  return check_launch("query_candidates_kernel");
}

extern "C" int mqdet_query_bank_norms(const float* bank, const int32_t* bank_count, int64_t L, int64_t cap, int64_t C, float* row_norm,
                                      void* stream) {
  MQ_REQUIRE(bank && bank_count && row_norm, "query_bank_norms: null pointer");
  MQ_REQUIRE(L > 0 && L < 65536 && cap > 0 && cap < (1 << 20) && C > 0 && L * cap * C < (1L << 40),
             "query_bank_norms: bad sizes L=%ld cap=%ld C=%ld", (long)L, (long)cap, (long)C);
  query_bank_norms_kernel<<<dim3((unsigned)cap, (unsigned)L), QB_THREADS, 0, (cudaStream_t)stream>>>(bank, bank_count, (int)C, (int)cap,
                                                                                                     row_norm);
  return check_launch("query_bank_norms_kernel");
}

extern "C" int mqdet_query_bank_update(const float* feats, const int32_t* labels, const int32_t* count, int64_t C, float* bank,
                                       int32_t* bank_count, float* row_norm, int64_t L, int64_t cap, int64_t max_query, float sim_thr,
                                       void* stream) {
  MQ_REQUIRE(feats && labels && count && bank && bank_count && row_norm, "query_bank_update: null pointer");
  MQ_REQUIRE(L > 0 && L < (1L << 31) && cap > 0 && cap < (1 << 20) && C > 0 && L * cap * C < (1L << 40) && max_query >= 0 &&
             max_query <= cap, "query_bank_update: bad sizes L=%ld cap=%ld C=%ld max_query=%ld", (long)L, (long)cap, (long)C,
             (long)max_query);
  query_bank_update_kernel<<<(unsigned)L, QB_THREADS, 0, (cudaStream_t)stream>>>(feats, labels, count, (int)C, (int)L, (int)cap,
                                                                                 (int)max_query, sim_thr, bank, bank_count, row_norm);
  return check_launch("query_bank_update_kernel");
}
