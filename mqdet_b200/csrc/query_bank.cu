// mqdet_b200 — the vision-query bank on the device: the test-time update (VISION_QUERY.NUM_TURNS; maskrcnn_benchmark/engine/
// inference.py:383-497) and the extraction over a dataset (tools/train_net.py:256-336, extract_query with exclude_similar=False).
//
//   query_candidates_kernel : packed detector rows [B][M + 1][6] -> the boxes extract_query pools: score > SCORE_THRESHOLD, grown
//                             by EXPAND_RATIO about their centre (expand_bbox, generalized_vl_rcnn_new.py:32-49), clipped to its
//                             own image's size and the empty ones removed (BoxList.clip_to_image(remove_empty=True)); image-then-row order
//   query_gt_rois_kernel    : the same boxes for ground-truth rows: each box first resized to the test size (BoxList.resize), then
//                             expanded and clipped as above; every kept row also carries its arrival number
//   query_bank_update_kernel: one CTA per label walks the pooled features of its label in arrival order and applies the bank
//                             bookkeeping of extract_query (:268-288): the per-label cap, with exclude_similar=True the cosine test
//                             against every row already in the bank (rows appended earlier in the same call included), the append
//   query_bank_merge_kernel : the banks of several ranks -> the bank one rank builds over all their rows: per label the rows in
//                             arrival order, the first max_query kept
//
// Every step reads its counts on the device, so a whole turn of the update, or a dataset walk of the extraction, runs without a
// host read.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int QC_MAX_IMAGES = 256;   // clip sizes per launch (kernel-parameter table)

// Clip bound of image b: [0, hi[n == 1 ? 0 : b][0]] x [0, hi[..][1]] = (w - 1, h - 1) of one size for all, or of each image.
struct QCSizes {
  int n;
  float hi[QC_MAX_IMAGES][2];
};

// expand_bbox then clip_to_image(remove_empty=True) of one box in place; true when it is kept.  Each step is one rounded fp32
// operation: w * ratio, (new - w) / 2, box + (-dw, -dh, dw, dh), clamp(min=0, max=size - 1) (NaN stays NaN and fails the test, as
// torch.clamp's does), x2 > x1 and y2 > y1.
__device__ __forceinline__ bool expand_clip_box(float& x1, float& y1, float& x2, float& y2, float ratio, float hi_x, float hi_y) {
  const float bw = __fsub_rn(x2, x1), bh = __fsub_rn(y2, y1);
  const float dw = __fdiv_rn(__fsub_rn(__fmul_rn(bw, ratio), bw), 2.f);
  const float dh = __fdiv_rn(__fsub_rn(__fmul_rn(bh, ratio), bh), 2.f);
  x1 = __fadd_rn(x1, -dw); y1 = __fadd_rn(y1, -dh);
  x2 = __fadd_rn(x2, dw);  y2 = __fadd_rn(y2, dh);
  x1 = x1 < 0.f ? 0.f : (x1 > hi_x ? hi_x : x1);
  y1 = y1 < 0.f ? 0.f : (y1 > hi_y ? hi_y : y1);
  x2 = x2 < 0.f ? 0.f : (x2 > hi_x ? hi_x : x2);
  y2 = y2 < 0.f ? 0.f : (y2 > hi_y ? hi_y : y2);
  return (y2 > y1) && (x2 > x1);
}

// The slot of this thread's row among the kept rows of one 1024-row step of a 1024-thread CTA (ballot scan, row order kept):
// start + the kept rows of lower threads; ``running`` advances by the step's kept rows.  Every thread of the CTA calls it.
__device__ __forceinline__ int block_compact_slot(int f, int* warp_tot, int* running) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ball = __ballot_sync(0xffffffffu, f);
  if (lane == 0) warp_tot[warp] = __popc(ball);
  __syncthreads();
  int woff = 0, tot = 0;
  for (int w = 0; w < 32; ++w) {
    if (w < warp) woff += warp_tot[w];
    tot += warp_tot[w];
  }
  const int pos = *running + woff + __popc(ball & ((1u << lane) - 1));
  __syncthreads();
  if (threadIdx.x == 0) *running += tot;
  __syncthreads();
  return pos;
}

// One CTA; images in order, per 1024 rows a ballot scan gives every kept box its slot (row order kept).
__global__ void __launch_bounds__(1024) query_candidates_kernel(const float* __restrict__ packed, int B, int M, float score_thr,
                                                                float ratio, const __grid_constant__ QCSizes sz,
                                                                float* __restrict__ rois,
                                                                int* __restrict__ labels, int* __restrict__ count,
                                                                int* __restrict__ bad) {
  __shared__ int warp_tot[32];
  __shared__ int running;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  for (int b = 0; b < B; ++b) {
    const float* rows = packed + (long)b * (M + 1) * 6;
    const float hi_x = sz.hi[sz.n == 1 ? 0 : b][0], hi_y = sz.hi[sz.n == 1 ? 0 : b][1];
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
          x1 = r[0]; y1 = r[1]; x2 = r[2]; y2 = r[3];
          f = expand_clip_box(x1, y1, x2, y2, ratio, hi_x, hi_y);
          lab = (int)r[5];
        }
      }
      const int pos = block_compact_slot(f, warp_tot, &running);
      if (f) {
        float* o = rois + (long)pos * 5;
        o[0] = (float)b; o[1] = x1; o[2] = y1; o[3] = x2; o[4] = y2;
        labels[pos] = lab;
      }
    }
  }
  if (threadIdx.x == 0) *count = running;
}

// Ground-truth table (int32 words, see mqdet_query_gt_rois): per image QG_IMG words, then the boxes f32 [nbox][4], then the labels.
constexpr int QG_IMG = 8;

// One CTA; images in order, their boxes resized (x * ratio_w, y * ratio_h), expanded and clipped, the kept ones compacted.
__global__ void __launch_bounds__(1024) query_gt_rois_kernel(const int* __restrict__ table, int B, int nbox, float ratio,
                                                             float* __restrict__ rois, int* __restrict__ labels,
                                                             int* __restrict__ arrival, int* __restrict__ count) {
  __shared__ int warp_tot[32];
  __shared__ int running;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  const float* boxes = reinterpret_cast<const float*>(table + (long)B * QG_IMG);
  const int* box_labels = table + (long)B * QG_IMG + 4L * nbox;
  for (int b = 0; b < B; ++b) {
    const int* im = table + (long)b * QG_IMG;
    const int first = im[0], n = im[1], arr0 = im[2];
    const float rw = __int_as_float(im[4]), rh = __int_as_float(im[5]), hi_x = __int_as_float(im[6]), hi_y = __int_as_float(im[7]);
    for (int base = 0; base < n; base += 1024) {
      const int i = base + threadIdx.x;
      int f = 0;
      float x1 = 0.f, y1 = 0.f, x2 = 0.f, y2 = 0.f;
      if (i < n) {
        const float* r = boxes + (long)(first + i) * 4;
        x1 = __fmul_rn(r[0], rw); y1 = __fmul_rn(r[1], rh);
        x2 = __fmul_rn(r[2], rw); y2 = __fmul_rn(r[3], rh);
        f = expand_clip_box(x1, y1, x2, y2, ratio, hi_x, hi_y);
      }
      const int pos = block_compact_slot(f, warp_tot, &running);
      if (f) {
        float* o = rois + (long)pos * 5;
        o[0] = (float)b; o[1] = x1; o[2] = y1; o[3] = x2; o[4] = y2;
        labels[pos] = box_labels[first + i];
        arrival[pos] = arr0 + i;
      }
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
// kSimilar: the cosine test of exclude_similar=True; without it a feature is appended whenever its label is below the cap.
// bank_arrival (may be null, and then arrival is not read): the arrival number of each appended feature, kept beside its row.
template <bool kSimilar>
__global__ void __launch_bounds__(QB_THREADS) query_bank_update_kernel(const float* __restrict__ feats, const int* __restrict__ labels,
                                                                       const int* __restrict__ arrival, const int* __restrict__ count,
                                                                       int C, int L, int cap, int max_query, float sim_thr,
                                                                       float* __restrict__ bank, int* __restrict__ bank_count,
                                                                       float* __restrict__ row_norm, int* __restrict__ bank_arrival) {
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
    if (kSimilar && n > 0) {
      for (int j = threadIdx.x >> 5; j < n; j += QB_WARPS) {
        const float s = warp_cosine(rows + (long)j * C, norms[j], x, nx, C);
        if ((threadIdx.x & 31) == 0 && s > sim_thr) similar = 1;
      }
      __syncthreads();
    }
    if (!similar) {
      for (int c = threadIdx.x; c < C; c += QB_THREADS) rows[(long)n * C + c] = x[c];
      if (threadIdx.x == 0) {
        norms[n] = nx;
        if (bank_arrival) bank_arrival[(long)lab * cap + n] = arrival[i];
      }
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

constexpr int QM_THREADS = 256;

// One warp per gathered row.  parts[r] = rank r's rows [n_r][2 + C] (label bits, arrival bits, the feature), sorted by label, then
// arrival; seg [G][L][2] = (first row, rows) of each label in each part.  A row's place in its label's merged order is its index
// within its own segment plus, for every other part, the rows of that label with a smaller arrival (lane r' binary-searches part
// r'; arrivals are distinct across parts).  Rows placed below max_query are written to out [L][max_query][C].
__global__ void __launch_bounds__(QM_THREADS) query_bank_merge_kernel(const float* const* __restrict__ parts, const int* __restrict__ seg,
                                                                      const int* __restrict__ part_rows, int G, int L, int C, int max_query,
                                                                      float* __restrict__ out) {
  const int r = blockIdx.y, lane = threadIdx.x & 31;
  const long i = (long)blockIdx.x * (QM_THREADS / 32) + (threadIdx.x >> 5);
  if (i >= part_rows[r]) return;
  const long W = 2L + C;
  const float* row = parts[r] + i * W;
  const int lab = __float_as_int(row[0]), arr = __float_as_int(row[1]);
  if (lab < 0 || lab >= L) return;
  int pos = 0;
  for (int q = lane; q < G; q += 32) {
    const int* s = seg + ((long)q * L + lab) * 2;
    if (q == r) {
      pos += (int)(i - s[0]);
      continue;
    }
    const float* p = parts[q] + (long)s[0] * W;
    int lo = 0, hi = s[1];                     // first row of part q's segment with arrival >= arr
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (__float_as_int(p[(long)mid * W + 1]) < arr) lo = mid + 1; else hi = mid;
    }
    pos += lo;
  }
  pos = __reduce_add_sync(0xffffffffu, pos);
  if (pos >= max_query) return;
  float* o = out + ((long)lab * max_query + pos) * C;
  for (int c = lane; c < C; c += 32) o[c] = row[2 + c];
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_query_candidates(const float* packed, int64_t B, int64_t M, float score_thr, float expand_ratio,
                                      const int64_t* img_wh, int64_t n_sizes, float* rois, int32_t* labels, int64_t cap, int32_t* count,
                                      int32_t* bad, void* stream) {
  MQ_REQUIRE(packed && img_wh && rois && labels && count && bad, "query_candidates: null pointer");
  MQ_REQUIRE(B > 0 && M > 0 && M <= (1 << 24) && (n_sizes == 1 || n_sizes == B) && n_sizes <= QC_MAX_IMAGES,
             "query_candidates: bad sizes B=%ld M=%ld with %ld image sizes (one, or one per image, at most %d)", (long)B, (long)M,
             (long)n_sizes, QC_MAX_IMAGES);
  QCSizes sz{};
  sz.n = (int)n_sizes;
  for (int64_t i = 0; i < n_sizes; ++i) {
    const int64_t w = img_wh[2 * i], h = img_wh[2 * i + 1];
    MQ_REQUIRE(w > 0 && h > 0 && w < (1 << 24) && h < (1 << 24), "query_candidates: bad sizes B=%ld M=%ld image %ld %ldx%ld", (long)B,
               (long)M, (long)i, (long)w, (long)h);
    sz.hi[i][0] = (float)(w - 1);
    sz.hi[i][1] = (float)(h - 1);
  }
  MQ_REQUIRE(cap >= B * M && B * M < (1L << 30), "query_candidates: capacity %ld below B * M = %ld", (long)cap, (long)(B * M));
  query_candidates_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(packed, (int)B, (int)M, score_thr, expand_ratio, sz, rois, labels,
                                                                count, bad);
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
  query_bank_update_kernel<true><<<(unsigned)L, QB_THREADS, 0, (cudaStream_t)stream>>>(
      feats, labels, nullptr, count, (int)C, (int)L, (int)cap, (int)max_query, sim_thr, bank, bank_count, row_norm, nullptr);
  return check_launch("query_bank_update_kernel");
}

extern "C" int mqdet_query_gt_rois(const int32_t* table, int64_t B, int64_t nbox, float expand_ratio, float* rois, int32_t* labels,
                                   int32_t* arrival, int32_t* count, void* stream) {
  MQ_REQUIRE(table && rois && labels && arrival && count, "query_gt_rois: null pointer");
  MQ_REQUIRE(B > 0 && nbox >= 0 && B * QG_IMG + 5 * nbox < (1L << 31), "query_gt_rois: bad sizes B=%ld nbox=%ld", (long)B, (long)nbox);
  query_gt_rois_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(table, (int)B, (int)nbox, expand_ratio, rois, labels, arrival, count);
  return check_launch("query_gt_rois_kernel");
}

extern "C" int mqdet_query_bank_append(const float* feats, const int32_t* labels, const int32_t* arrival, const int32_t* count,
                                       int64_t C, float* bank, int32_t* bank_count, float* row_norm, int32_t* bank_arrival, int64_t L,
                                       int64_t cap, int64_t max_query, void* stream) {
  MQ_REQUIRE(feats && labels && arrival && count && bank && bank_count && row_norm && bank_arrival, "query_bank_append: null pointer");
  MQ_REQUIRE(L > 0 && L < (1L << 31) && cap > 0 && cap < (1 << 20) && C > 0 && L * cap * C < (1L << 40) && max_query >= 0 &&
             max_query <= cap, "query_bank_append: bad sizes L=%ld cap=%ld C=%ld max_query=%ld", (long)L, (long)cap, (long)C,
             (long)max_query);
  query_bank_update_kernel<false><<<(unsigned)L, QB_THREADS, 0, (cudaStream_t)stream>>>(
      feats, labels, arrival, count, (int)C, (int)L, (int)cap, (int)max_query, 0.f, bank, bank_count, row_norm, bank_arrival);
  return check_launch("query_bank_append_kernel");
}

extern "C" int mqdet_query_bank_merge(const float* const* parts, const int32_t* seg, const int32_t* part_rows, int64_t max_rows,
                                      int64_t G, int64_t L, int64_t C, int64_t max_query, float* out, void* stream) {
  MQ_REQUIRE(parts && seg && part_rows && out, "query_bank_merge: null pointer");
  MQ_REQUIRE(G > 0 && G < 65536 && L > 0 && L < (1L << 31) && C > 0 && max_query > 0 && L * max_query * C < (1L << 40) &&
             max_rows >= 0 && max_rows < (1L << 31), "query_bank_merge: bad sizes G=%ld L=%ld C=%ld max_query=%ld max_rows=%ld",
             (long)G, (long)L, (long)C, (long)max_query, (long)max_rows);
  if (max_rows == 0) return 0;
  const long blocks = (max_rows + QM_THREADS / 32 - 1) / (QM_THREADS / 32);
  query_bank_merge_kernel<<<dim3((unsigned)blocks, (unsigned)G), QM_THREADS, 0, (cudaStream_t)stream>>>(parts, seg, part_rows, (int)G,
                                                                                                       (int)L, (int)C, (int)max_query,
                                                                                                       out);
  return check_launch("query_bank_merge_kernel");
}
