// mqdet_b200 — multi-scale / flip test-time augmentation: the cross-pass merge on the device.
//
// Reference: maskrcnn_benchmark/data/datasets/evaluation/box_aug.py (im_detect_bbox_aug :12-62, remove_boxes :150-163,
// merge_result_from_multi_scales :166-206, boxlist_nms :209-238, bbox_vote :241-287), BoxList.transpose / resize
// (structures/bounding_box.py) and csrc/cuda/nms.cu (devIoU :15-23, strict '>' :62, ascending kept indices :139-142).
//
//   hflip_pad_kernel       : normalised image -> horizontally flipped, zero-padded batch tensor
//   aug_collect_kernel     : one pass's candidates -> flip, keep range, resize -> appended behind the earlier passes
//                            (one CTA per image, ballot scan: candidate order kept; running count on the device)
//   aug_collect_packed_kernel : the same for one pass's packed detector rows (MQ-GroundingDINO), count read on the device
//   aug_tile_sort_kernel   : 64-bit keys (class rank | ~score | merged index), bitonic sort of 2048-key tiles
//   aug_merge_pass_kernel  : one doubling of the sorted run length (rank by binary search in the sibling run)
//   aug_segments_kernel    : class segment table from the sorted keys
//   aug_class_nms_kernel   : one CTA per (image, class): greedy suppression / vote clustering in score order
//   aug_emit_kernel        : per image: the PRE_NMS_TOP_N cut (radix select of the k-th largest score) and the packed result
//
// Every box arithmetic below is IEEE fp32 WITHOUT contraction (__fadd_rn / __fmul_rn): the numpy code of bbox_vote and
// tensor * python_float of BoxList.resize round every operation, and the CPU restatement compares exactly.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int AUG_MAX_CAP = 1 << 17;       // merged index field of the sort key: 17 bits
constexpr int AUG_MAX_CLASSES = 32766;     // class-rank field: 15 bits, 0x7fff = "not a listed class"
constexpr unsigned long long AUG_IDX_MASK = 0x1ffffull;
constexpr int AUG_RANK_SHIFT = 49;
constexpr unsigned AUG_NO_RANK = 0x7fffu;
constexpr int AUG_TILE = 2048;             // keys sorted in shared memory per CTA
constexpr int AUG_CH = 128;                // boxes of one class examined together
constexpr int AUG_NMS_THREADS = 512;       // AUG_CH x 4: four kept-list slices / four 32-bit mask words per box
constexpr int AUG_KCACHE = 2048;           // kept boxes held in shared memory; later ones are read from the global list
// overflow[b] holds two things: bits 0..29 count the boxes that did not fit (saturating at AUG_BAD_COUNT - 1, so the count
// never reaches bit 30), bit 30 flags a packed pass whose count row was not an integer in [0, M].  unpack reads bit 30 first.
constexpr int AUG_BAD_COUNT = 1 << 30;

__device__ __forceinline__ unsigned ordered_bits(float s) {  // ascending-sortable
  const unsigned u = __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// devIoU of nms.cu:15-23 (+1 widths), every operation rounded
__device__ __forceinline__ float aug_iou(const float4 a, const float4 b) {
  const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  const float width = fmaxf(__fadd_rn(__fsub_rn(right, left), 1.f), 0.f);
  const float height = fmaxf(__fadd_rn(__fsub_rn(bottom, top), 1.f), 0.f);
  const float inter = __fmul_rn(width, height);
  const float sa = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.f), __fadd_rn(__fsub_rn(a.w, a.y), 1.f));
  const float sb = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter));
}

__global__ void __launch_bounds__(256) hflip_pad_kernel(const float* __restrict__ in, int planes, int h, int w, int H, int W,
                                                        float* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)planes * H * W) return;
  const int x = (int)(i % W), y = (int)((i / W) % H);
  const long p = i / ((long)W * H);
  out[i] = (x < w && y < h) ? in[(p * h + y) * w + (w - 1 - x)] : 0.f;
}

// One pass's steps for one box, in the order of im_detect_bbox_aug: un-flip, keep range, resize.  -> whether the box stays.
__device__ __forceinline__ int aug_pass_box(float4& bx, int flip, float pass_w, int has_range, float lo2, float hi2, float rx,
                                            float ry) {
  if (flip) {  // BoxList.transpose(FLIP_LEFT_RIGHT), TO_REMOVE = 1
    const float x1 = __fsub_rn(__fsub_rn(pass_w, bx.z), 1.f), x2 = __fsub_rn(__fsub_rn(pass_w, bx.x), 1.f);
    bx.x = x1; bx.z = x2;
  }
  int f = 1;
  if (has_range) {  // remove_boxes: both bounds strict
    const float area = __fmul_rn(__fadd_rn(__fsub_rn(bx.z, bx.x), 1.f), __fadd_rn(__fsub_rn(bx.w, bx.y), 1.f));
    f = (area > lo2) && (area < hi2);
  }
  bx.x = __fmul_rn(bx.x, rx); bx.z = __fmul_rn(bx.z, rx);  // BoxList.resize to the original image
  bx.y = __fmul_rn(bx.y, ry); bx.w = __fmul_rn(bx.w, ry);
  return f;
}

// The two inputs of a collect, one image each: the cand_* arrays of atss_postprocess, and packed detector rows
// (x1, y1, x2, y2, score, label) as gdino_detections writes them.
struct AugCandRows {
  const float4* boxes;
  const float* scores;
  const float* labels;
  __device__ __forceinline__ void load(int i, float4& bx, float& s, int& lab) const {
    bx = boxes[i]; s = scores[i]; lab = (int)labels[i];
  }
};
struct AugPackedRows {
  const float* rows;
  __device__ __forceinline__ void load(int i, float4& bx, float& s, int& lab) const {
    const float* r = rows + (long)i * 6;
    bx = make_float4(r[0], r[1], r[2], r[3]); s = r[4]; lab = (int)r[5];
  }
};

// One CTA appends the first n rows of one image's pass behind count[0] (pointers already at the image).  Row order is kept:
// per 1024 rows a ballot scan gives every survivor its slot.
template <class Rows>
__device__ __forceinline__ void aug_collect_image(const Rows src, int n, int flip, float pass_w, int has_range, float lo2,
                                                  float hi2, float rx, float ry, float* __restrict__ boxes,
                                                  float* __restrict__ scores, int* __restrict__ labels, int cap,
                                                  int* __restrict__ count, int* __restrict__ overflow) {
  __shared__ int warp_tot[32];
  __shared__ int running;
  if (threadIdx.x == 0) running = *count;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    int f = 0, lab = 0;
    float sc = 0.f;
    float4 bx = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < n) {
      src.load(i, bx, sc, lab);
      f = aug_pass_box(bx, flip, pass_w, has_range, lo2, hi2, rx, ry);
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
    const int pos = start + woff + __popc(ball & ((1u << lane) - 1));
    if (f && pos < cap) {
      reinterpret_cast<float4*>(boxes)[pos] = bx;
      scores[pos] = sc;
      labels[pos] = lab;
    }
    __syncthreads();
    if (threadIdx.x == 0) running = start + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int r = running;
    *count = min(r, cap);
    if (r > cap) {
      const int lost = (int)min((long long)(*overflow & (AUG_BAD_COUNT - 1)) + (r - cap), (long long)AUG_BAD_COUNT - 1);
      *overflow = (*overflow & AUG_BAD_COUNT) | lost;
    }
  }
}

// One CTA per image.
__global__ void __launch_bounds__(1024) aug_collect_kernel(const float* __restrict__ cboxes, const float* __restrict__ cscores,
                                                           const float* __restrict__ clabels, const int* __restrict__ totals,
                                                           int S, int flip, float pass_w, int has_range, float lo2, float hi2,
                                                           float rx, float ry, float* __restrict__ boxes,
                                                           float* __restrict__ scores, int* __restrict__ labels, int cap,
                                                           int* __restrict__ count, int* __restrict__ overflow) {
  const int b = blockIdx.x;
  const AugCandRows src{reinterpret_cast<const float4*>(cboxes) + (long)b * S, cscores + (long)b * S, clabels + (long)b * S};
  aug_collect_image(src, min(totals[b], S), flip, pass_w, has_range, lo2, hi2, rx, ry, boxes + (long)b * cap * 4,
                    scores + (long)b * cap, labels + (long)b * cap, cap, count + b, overflow + b);
}

// One CTA per image; packed [B][M + 1][6], row M = (count, ...).  A count that is not an integer in [0, M] reads no row and
// sets AUG_BAD_COUNT in overflow[b], which unpack reports.
__global__ void __launch_bounds__(1024) aug_collect_packed_kernel(const float* __restrict__ packed, int M, int flip, float pass_w,
                                                                  int has_range, float lo2, float hi2, float rx, float ry,
                                                                  float* __restrict__ boxes, float* __restrict__ scores,
                                                                  int* __restrict__ labels, int cap, int* __restrict__ count,
                                                                  int* __restrict__ overflow) {
  const int b = blockIdx.x;
  const float* rows = packed + (long)b * (M + 1) * 6;
  const float cnt = rows[(long)M * 6];
  const bool ok = cnt >= 0.f && cnt <= (float)M && cnt == floorf(cnt);
  aug_collect_image(AugPackedRows{rows}, ok ? (int)cnt : 0, flip, pass_w, has_range, lo2, hi2, rx, ry, boxes + (long)b * cap * 4,
                    scores + (long)b * cap, labels + (long)b * cap, cap, count + b, overflow + b);
  if (!ok && threadIdx.x == 0) overflow[b] |= AUG_BAD_COUNT;
}

// ---- sort ----------------------------------------------------------------------------------------------------------
// key = class rank << 49 | ~ordered(score) << 17 | merged index: ascending keys = classes ascending, scores descending,
// equal scores by ascending merged index.  src != nullptr: sort the given keys instead of building them.
__global__ void __launch_bounds__(1024) aug_tile_sort_kernel(const float* __restrict__ scores, const int* __restrict__ labels,
                                                             const int* __restrict__ classes, int C,
                                                             const unsigned long long* __restrict__ src,
                                                             const int* __restrict__ count, int cap,
                                                             unsigned long long* __restrict__ dst) {
  __shared__ unsigned long long keys[AUG_TILE];
  const int b = blockIdx.y;
  const int n = min(count[b], cap);
  const int t0 = blockIdx.x * AUG_TILE;
  if (t0 >= n) return;
  for (int j = threadIdx.x; j < AUG_TILE; j += 1024) {
    const int i = t0 + j;
    unsigned long long k = ~0ull;
    if (i < n) {
      if (src) {
        k = src[(long)b * cap + i];
      } else {
        const int lab = labels[(long)b * cap + i];
        int lo = 0, hi = C;  // first table entry >= lab
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (classes[mid] < lab) lo = mid + 1; else hi = mid;
        }
        const unsigned rank = (lo < C && classes[lo] == lab) ? (unsigned)lo : AUG_NO_RANK;
        const unsigned u = ~ordered_bits(scores[(long)b * cap + i]);
        k = ((unsigned long long)rank << AUG_RANK_SHIFT) | ((unsigned long long)u << 17) | (unsigned long long)i;
      }
    }
    keys[j] = k;
  }
  __syncthreads();
  for (int k = 2; k <= AUG_TILE; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < AUG_TILE; i += 1024) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], c = keys[ixj];
          if ((a > c) == ((i & k) == 0)) {
            keys[i] = c;
            keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int j = threadIdx.x; j < AUG_TILE && t0 + j < n; j += 1024) dst[(long)b * cap + t0 + j] = keys[j];
}

// Runs of `run` sorted keys -> runs of 2 * run: an element of the left run goes behind the right-run keys below it, one of
// the right run behind the left-run keys not above it (equal keys keep left before right).
__global__ void __launch_bounds__(256) aug_merge_pass_kernel(const unsigned long long* __restrict__ src,
                                                             unsigned long long* __restrict__ dst,
                                                             const int* __restrict__ count, int cap, int run) {
  const int b = blockIdx.y;
  const int n = min(count[b], cap);
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  src += (long)b * cap; dst += (long)b * cap;
  const int a0 = i / (2 * run) * (2 * run);
  const int a1 = min(a0 + run, n), b1 = min(a0 + 2 * run, n);
  const unsigned long long key = src[i];
  int lo, hi, pos;
  if (i < a1) {
    lo = a1; hi = b1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (src[mid] < key) lo = mid + 1; else hi = mid;
    }
    pos = (i - a0) + (lo - a1);
  } else {
    lo = a0; hi = a1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (src[mid] <= key) lo = mid + 1; else hi = mid;
    }
    pos = (i - a1) + (lo - a0);
  }
  dst[a0 + pos] = key;
}

// seg[b][c] = first sorted position of class rank c (c = C: the boxes of no listed class), seg[b][C + 1] unused.
__global__ void __launch_bounds__(256) aug_segments_kernel(const unsigned long long* __restrict__ keys,
                                                           const int* __restrict__ count, int cap, int C,
                                                           int* __restrict__ seg) {
  const int b = blockIdx.y;
  const int n = min(count[b], cap);
  const int i = blockIdx.x * 256 + threadIdx.x;
  seg += (long)b * (C + 1);
  if (n == 0) {
    if (i == 0)
      for (int c = 0; c <= C; ++c) seg[c] = 0;
    return;
  }
  if (i >= n) return;
  keys += (long)b * cap;
  const int r = min((int)(keys[i] >> AUG_RANK_SHIFT), C);
  const int prev = i == 0 ? -1 : min((int)(keys[i - 1] >> AUG_RANK_SHIFT), C);
  for (int c = prev + 1; c <= r; ++c) seg[c] = i;
  if (i == n - 1)
    for (int c = r + 1; c <= C; ++c) seg[c] = n;
}

// ---- per-class suppression / voting --------------------------------------------------------------------------------
// One CTA per (image, class) walks the class's boxes in score order, AUG_CH at a time:
//   1. every box against the kept list so far (four threads per box, each a quarter of the list; the lowest hit wins);
//   2. the AUG_CH x AUG_CH bit matrix of the chunk;
//   3. one thread resolves the chunk serially (a box survives if no kept box and no earlier survivor of the chunk hit it);
//   4. survivors join the kept list (shared memory for the first AUG_KCACHE, always the global list);
//   5. vote: the other boxes add score * box and score to their cluster, in score order, one thread per (chunk, cluster).
// `ge` selects IoU >= th (bbox_vote) instead of IoU > th (nms.cu).  key2 of a survivor = class rank | merged index (nms) or
// class rank | cluster ordinal (vote); all other positions get ~0.
__global__ void __launch_bounds__(AUG_NMS_THREADS) aug_class_nms_kernel(
    const unsigned long long* __restrict__ keys, const float* __restrict__ boxes, const float* __restrict__ scores,
    const int* __restrict__ seg, int cap, int C, float th, int vote, unsigned long long* __restrict__ key2,
    float4* __restrict__ kbox, float4* __restrict__ kacc, float2* __restrict__ kss, int* __restrict__ kcnt) {
  const int b = blockIdx.y, c = blockIdx.x;
  const int s0 = seg[(long)b * (C + 1) + c], n = seg[(long)b * (C + 1) + c + 1] - s0;
  if (n <= 0) return;
  const long g0 = (long)b * cap + s0;  // this class's slice of the per-image arrays
  keys += g0; key2 += g0; kbox += g0;
  const float4* boxes4 = reinterpret_cast<const float4*>(boxes) + (long)b * cap;
  scores += (long)b * cap;
  const unsigned long long rankbits = (unsigned long long)c << AUG_RANK_SHIFT;
  const int tid = threadIdx.x;
  if (th <= 0.f) {  // boxlist_nms returns the class untouched
    for (int p = tid; p < n; p += AUG_NMS_THREADS) key2[p] = rankbits | (keys[p] & AUG_IDX_MASK);
    return;
  }
  __shared__ float4 kcache[AUG_KCACHE];
  __shared__ float4 cb[AUG_CH];
  __shared__ float cs[AUG_CH];
  __shared__ int cidx[AUG_CH], head[AUG_CH], kpos[AUG_CH];
  __shared__ unsigned mask[AUG_CH * 4];
  __shared__ int nk;
  if (tid == 0) nk = 0;
  const int cc = tid % AUG_CH, q = tid / AUG_CH;
  for (int base = 0; base < n; base += AUG_CH) {
    const int size = min(AUG_CH, n - base);
    __syncthreads();
    if (tid < size) {
      const int idx = (int)(keys[base + tid] & AUG_IDX_MASK);
      cidx[tid] = idx;
      cb[tid] = boxes4[idx];
      cs[tid] = scores[idx];
      head[tid] = INT_MAX;
    }
    __syncthreads();
    const int nkept = nk;
    if (cc < size) {
      const float4 me = cb[cc];
      for (int k = q; k < nkept; k += 4) {
        if (head[cc] < k) break;  // a lower kept box already hit (the list is in score order)
        const float iou = aug_iou(k < AUG_KCACHE ? kcache[k] : kbox[k], me);
        if (vote ? (iou >= th) : (iou > th)) {
          atomicMin(&head[cc], k);
          break;
        }
      }
      unsigned word = 0;
      for (int j = max(32 * q, cc + 1); j < min(32 * q + 32, size); ++j) {
        const float iou = aug_iou(me, cb[j]);
        if (vote ? (iou >= th) : (iou > th)) word |= 1u << (j & 31);
      }
      mask[cc * 4 + q] = word;
    }
    __syncthreads();
    if (tid == 0) {
      unsigned r0 = 0, r1 = 0, r2 = 0, r3 = 0;
      int k = nkept;
      for (int t = 0; t < size; ++t) {
        const unsigned r = t < 64 ? (t < 32 ? r0 : r1) : (t < 96 ? r2 : r3);
        if (head[t] == INT_MAX && !((r >> (t & 31)) & 1u)) {
          kpos[t] = k++;
          r0 |= mask[t * 4]; r1 |= mask[t * 4 + 1]; r2 |= mask[t * 4 + 2]; r3 |= mask[t * 4 + 3];
        } else {
          kpos[t] = -1;
        }
      }
      nk = k;
    }
    __syncthreads();
    if (tid < size) {
      const int k = kpos[tid];
      if (k >= 0) {
        const float4 me = cb[tid];
        const float s = cs[tid];
        if (k < AUG_KCACHE) kcache[k] = me;
        kbox[k] = me;
        if (vote) {
          kacc[g0 + k] = make_float4(__fmul_rn(me.x, s), __fmul_rn(me.y, s), __fmul_rn(me.z, s), __fmul_rn(me.w, s));
          kss[g0 + k] = make_float2(s, s);
          kcnt[g0 + k] = 1;
        }
        key2[base + tid] = rankbits | (unsigned long long)(vote ? k : cidx[tid]);
      } else {
        key2[base + tid] = ~0ull;
        if (vote && head[tid] == INT_MAX) {  // taken by a survivor of this chunk: the first one that hit it
          for (int t = 0; t < tid; ++t)
            if (kpos[t] >= 0 && ((mask[t * 4 + (tid >> 5)] >> (tid & 31)) & 1u)) {
              head[tid] = kpos[t];
              break;
            }
        }
      }
    }
    if (!vote) continue;
    __syncthreads();
    if (tid < size && kpos[tid] < 0) {
      const int h = head[tid];
      bool leader = true;
      for (int t = 0; t < tid; ++t)
        if (kpos[t] < 0 && head[t] == h) {
          leader = false;
          break;
        }
      if (leader) {  // the cluster's members of this chunk, in score order
        float4 a = kacc[g0 + h];
        float2 ss = kss[g0 + h];
        int cnt = kcnt[g0 + h];
        for (int t = tid; t < size; ++t)
          if (kpos[t] < 0 && head[t] == h) {
            const float4 m = cb[t];
            const float s = cs[t];
            a.x = __fadd_rn(a.x, __fmul_rn(m.x, s)); a.y = __fadd_rn(a.y, __fmul_rn(m.y, s));
            a.z = __fadd_rn(a.z, __fmul_rn(m.z, s)); a.w = __fadd_rn(a.w, __fmul_rn(m.w, s));
            ss.x = __fadd_rn(ss.x, s);
            ++cnt;
          }
        kacc[g0 + h] = a;
        kss[g0 + h] = ss;
        kcnt[g0 + h] = cnt;
      }
    }
  }
}

// ---- per-image cut and packed result -------------------------------------------------------------------------------
// keys = the sorted key2: the first `nres` (class rank < 0x7fff) are the results in output order.
__global__ void __launch_bounds__(1024) aug_emit_kernel(const unsigned long long* __restrict__ keys,
                                                        const float* __restrict__ boxes, const float* __restrict__ scores,
                                                        const int* __restrict__ classes, const int* __restrict__ seg,
                                                        const int* __restrict__ count, const int* __restrict__ overflow,
                                                        int cap, int C, int cluster, const float4* __restrict__ kbox,
                                                        const float4* __restrict__ kacc, const float2* __restrict__ kss,
                                                        const int* __restrict__ kcnt, int top_n, int max_out,
                                                        float* __restrict__ out) {
  const int b = blockIdx.x;
  const int n = min(count[b], cap);
  keys += (long)b * cap; scores += (long)b * cap; seg += (long)b * (C + 1);
  kbox += (long)b * cap; kacc += (long)b * cap; kss += (long)b * cap; kcnt += (long)b * cap;
  const float4* boxes4 = reinterpret_cast<const float4*>(boxes) + (long)b * cap;
  out += (long)b * (max_out + 1) * 6;
  __shared__ int nres_s, hist[256], krem_s, warp_tot[32], running;
  __shared__ unsigned prefix_s;
  const int tid = threadIdx.x;
  if (tid == 0) {
    int lo = 0, hi = n;
    const unsigned long long lim = (unsigned long long)AUG_NO_RANK << AUG_RANK_SHIFT;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (keys[mid] < lim) lo = mid + 1; else hi = mid;
    }
    nres_s = lo;
    running = 0;
  }
  __syncthreads();
  const int nres = nres_s;
  auto slot = [&](unsigned long long k) { return seg[(int)(k >> AUG_RANK_SHIFT)] + (int)(k & AUG_IDX_MASK); };
  auto score_at = [&](int p) {
    const unsigned long long k = keys[p];
    return cluster ? kss[slot(k)].y : scores[(int)(k & AUG_IDX_MASK)];
  };
  unsigned thr = 0;  // ordered bits of the lowest score that stays
  if (top_n > 0 && nres > top_n) {  // the top_n-th largest score: radix select, most significant byte first
    if (tid == 0) {
      krem_s = top_n;
      prefix_s = 0;
    }
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += 1024) hist[i] = 0;
      __syncthreads();
      const unsigned prefix = prefix_s;
      const unsigned himask = shift == 24 ? 0u : ~0u << (shift + 8);
      for (int p = tid; p < nres; p += 1024) {
        const unsigned u = ordered_bits(score_at(p));
        if ((u & himask) == prefix) atomicAdd(&hist[(u >> shift) & 255], 1);
      }
      __syncthreads();
      if (tid == 0) {
        int cum = 0, d = 255;
        for (; d > 0; --d) {
          if (cum + hist[d] >= krem_s) break;
          cum += hist[d];
        }
        krem_s -= cum;
        prefix_s = prefix | ((unsigned)d << shift);
      }
      __syncthreads();
    }
    thr = prefix_s;
  }
  const int lane = tid & 31, warp = tid >> 5;
  for (int base = 0; base < nres; base += 1024) {
    const int p = base + tid;
    int f = 0;
    float sc = 0.f;
    if (p < nres) {
      sc = score_at(p);
      f = ordered_bits(sc) >= thr;
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
    const int pos = start + woff + __popc(ball & ((1u << lane) - 1));
    if (f && pos < max_out) {
      const unsigned long long k = keys[p];
      float4 bx;
      if (cluster) {
        const int s = slot(k);
        bx = kbox[s];
        if (kcnt[s] > 1) {  // bbox_vote: sum(score * box) / sum(score)
          const float4 a = kacc[s];
          const float ss = kss[s].x;
          bx = make_float4(__fdiv_rn(a.x, ss), __fdiv_rn(a.y, ss), __fdiv_rn(a.z, ss), __fdiv_rn(a.w, ss));
        }
      } else {
        bx = boxes4[(int)(k & AUG_IDX_MASK)];
      }
      float* o = out + (long)pos * 6;
      o[0] = bx.x; o[1] = bx.y; o[2] = bx.z; o[3] = bx.w;
      o[4] = sc;
      o[5] = (float)classes[(int)(k >> AUG_RANK_SHIFT)];
    }
    __syncthreads();
    if (tid == 0) running = start + tot;
    __syncthreads();
  }
  if (tid < 6) out[(long)max_out * 6 + tid] = tid == 0 ? (float)running : (tid == 1 && overflow ? (float)overflow[b] : 0.f);
}

static inline size_t aug_align(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_hflip_pad(const float* in, int64_t planes, int64_t h, int64_t w, int64_t H, int64_t W, float* out,
                               void* stream) {
  MQ_REQUIRE(in && out, "hflip_pad: null pointer");
  MQ_REQUIRE(planes > 0 && h > 0 && w > 0 && H >= h && W >= w, "hflip_pad: bad sizes planes=%ld %ldx%ld -> %ldx%ld", (long)planes,
             (long)h, (long)w, (long)H, (long)W);
  hflip_pad_kernel<<<cdiv(planes * H * W, 256), 256, 0, (cudaStream_t)stream>>>(in, (int)planes, (int)h, (int)w, (int)H, (int)W, out);
  return check_launch("hflip_pad_kernel");
}

extern "C" int mqdet_bbox_aug_collect(const float* cand_boxes, const float* cand_scores, const float* cand_labels,
                                      const int32_t* cand_totals, int64_t B, int64_t S, int flip, float pass_w, int has_range,
                                      float lo2, float hi2, float ratio_x, float ratio_y, float* boxes, float* scores,
                                      int32_t* labels, int64_t cap, int32_t* count, int32_t* overflow, void* stream) {
  MQ_REQUIRE(cand_boxes && cand_scores && cand_labels && cand_totals && boxes && scores && labels && count && overflow,
             "bbox_aug_collect: null pointer");
  MQ_REQUIRE(B > 0 && S > 0 && cap > 0 && cap <= AUG_MAX_CAP, "bbox_aug_collect: bad sizes B=%ld S=%ld cap=%ld (cap <= %d)", (long)B,
             (long)S, (long)cap, AUG_MAX_CAP);
  aug_collect_kernel<<<(unsigned)B, 1024, 0, (cudaStream_t)stream>>>(cand_boxes, cand_scores, cand_labels, cand_totals, (int)S, flip,
                                                                     pass_w, has_range, lo2, hi2, ratio_x, ratio_y, boxes, scores,
                                                                     labels, (int)cap, count, overflow);
  return check_launch("aug_collect_kernel");
}

extern "C" int mqdet_bbox_aug_collect_packed(const float* packed, int64_t B, int64_t M, int flip, float pass_w, int has_range,
                                             float lo2, float hi2, float ratio_x, float ratio_y, float* boxes, float* scores,
                                             int32_t* labels, int64_t cap, int32_t* count, int32_t* overflow, void* stream) {
  MQ_REQUIRE(packed && boxes && scores && labels && count && overflow, "bbox_aug_collect_packed: null pointer");
  MQ_REQUIRE(B > 0 && M > 0 && M <= (1 << 24) && cap > 0 && cap <= AUG_MAX_CAP,
             "bbox_aug_collect_packed: bad sizes B=%ld M=%ld cap=%ld (M <= %d, cap <= %d)", (long)B, (long)M, (long)cap, 1 << 24,
             AUG_MAX_CAP);
  aug_collect_packed_kernel<<<(unsigned)B, 1024, 0, (cudaStream_t)stream>>>(packed, (int)M, flip, pass_w, has_range, lo2, hi2, ratio_x,
                                                                            ratio_y, boxes, scores, labels, (int)cap, count, overflow);
  return check_launch("aug_collect_packed_kernel");
}

extern "C" int64_t mqdet_nms_by_class_workspace_bytes(int64_t B, int64_t cap, int64_t C) {
  if (B <= 0 || cap <= 0 || C < 0) return 256;
  const size_t n = (size_t)B * cap;
  return (int64_t)(3 * aug_align(n * 8) + 2 * aug_align(n * 16) + aug_align(n * 8) + aug_align(n * 4) +
                   aug_align((size_t)B * (C + 2) * 4) + 256);
}

static void aug_sort(const float* scores, const int32_t* labels, const int32_t* classes, int C, const unsigned long long* src,
                     const int32_t* count, int B, int cap, unsigned long long* first, unsigned long long* other,
                     unsigned long long** result, cudaStream_t st) {
  aug_tile_sort_kernel<<<dim3(cdiv(cap, AUG_TILE), B), 1024, 0, st>>>(scores, labels, classes, C, src, count, cap, first);
  unsigned long long *a = first, *b = other;
  for (long run = AUG_TILE; run < cap; run *= 2) {
    aug_merge_pass_kernel<<<dim3(cdiv(cap, 256), B), 256, 0, st>>>(a, b, count, cap, (int)run);
    unsigned long long* t = a; a = b; b = t;
  }
  *result = a;
}

extern "C" int mqdet_nms_by_class(const float* boxes, const float* scores, const int32_t* labels, const int32_t* count,
                                  const int32_t* overflow, int64_t B, int64_t cap, const int32_t* classes, int64_t C, float thresh,
                                  int vote, int64_t top_n, int64_t max_out, float* out, void* workspace, void* stream) {
  MQ_REQUIRE(boxes && scores && labels && count && classes && out && workspace, "nms_by_class: null pointer");
  MQ_REQUIRE(B > 0 && cap > 0 && cap <= AUG_MAX_CAP && max_out > 0, "nms_by_class: bad sizes B=%ld cap=%ld max_out=%ld (cap <= %d)",
             (long)B, (long)cap, (long)max_out, AUG_MAX_CAP);
  MQ_REQUIRE(C > 0 && C <= AUG_MAX_CLASSES, "nms_by_class: 1..%d classes (got %ld)", AUG_MAX_CLASSES, (long)C);
  MQ_REQUIRE(vote == 0 || vote == 1, "nms_by_class: mode must be 0 (nms) or 1 (vote)");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = (size_t)B * cap;
  uint8_t* ws = (uint8_t*)workspace;
  unsigned long long* k0 = (unsigned long long*)ws;  ws += aug_align(n * 8);
  unsigned long long* k1 = (unsigned long long*)ws;  ws += aug_align(n * 8);
  unsigned long long* k2 = (unsigned long long*)ws;  ws += aug_align(n * 8);
  float4* kbox = (float4*)ws;                         ws += aug_align(n * 16);
  float4* kacc = (float4*)ws;                         ws += aug_align(n * 16);
  float2* kss = (float2*)ws;                          ws += aug_align(n * 8);
  int* kcnt = (int*)ws;                               ws += aug_align(n * 4);
  int* seg = (int*)ws;
  unsigned long long *sorted, *sorted2;
  aug_sort(scores, labels, classes, (int)C, nullptr, count, (int)B, (int)cap, k0, k1, &sorted, st);
  unsigned long long* spare = sorted == k0 ? k1 : k0;
  aug_segments_kernel<<<dim3(cdiv(cap, 256), (unsigned)B), 256, 0, st>>>(sorted, count, (int)cap, (int)C, seg);
  cudaMemsetAsync(k2, 0xff, n * 8, st);  // positions of no listed class stay ~0
  aug_class_nms_kernel<<<dim3((unsigned)C, (unsigned)B), AUG_NMS_THREADS, 0, st>>>(sorted, boxes, scores, seg, (int)cap, (int)C, thresh,
                                                                                   vote, k2, kbox, kacc, kss, kcnt);
  aug_sort(nullptr, nullptr, nullptr, 0, k2, count, (int)B, (int)cap, spare, k2, &sorted2, st);
  aug_emit_kernel<<<(unsigned)B, 1024, 0, st>>>(sorted2, boxes, scores, classes, seg, count, overflow, (int)cap, (int)C,
                                                vote && thresh > 0.f, kbox, kacc, kss, kcnt, (int)top_n, (int)max_out, out);
  return check_launch("nms_by_class");
}
