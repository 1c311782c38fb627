// mqdet_b200 — box AP on the device: LVIS fixed-AP (top-k per category) and standard (top 300 per image) protocols, and COCO
// (pycocotools COCOeval, bbox: top 100 per (image, category), crowd GTs, maxDets 1 / 10 / 100).  Where the two protocols differ
// the rule comes in as data (a crowd array, the federated filter on or off, the detection area filter on or off, a maxDets list),
// never as a protocol switch.
//
// Reference: maskrcnn_benchmark/data/datasets/evaluation/lvis/lvis_eval.py (LvisEvaluatorFixedAP :766-875, LVISResults :78-147,
// LVISEval._prepare :200-240, evaluate_img :318-410, accumulate :412-523), lvis.py get_ann_ids (0 < area < inf), pycocotools
// bbIou.  COCO: od_to_grounding/od_eval.py (prepare_for_coco_detection, evaluate_predictions_on_coco) and pycocotools COCOeval
// (_prepare, computeIoU, evaluateImg, accumulate).  The rules are written out in DESIGN.md section 4 ("LVIS box AP rules",
// "COCO box AP rules").
//
//   lvis_collect_kernel  : packed detector rows -> resized fp32 xywh, category / image index, arrival number; one pool slot per
//                          packed row (slot = arrival order), rows that are not detections are marked empty
//   lvis_keys_kernel     : 192-bit sort keys (three words, compared in order) for the cut, the pairing and the accumulation
//   lvis_tile_sort_kernel: bitonic sort of LV_TILE keys in shared memory
//   lvis_merge_pass_kernel: one doubling of the sorted run length (rank by binary search in the sibling run; keys are unique)
//   lvis_group_kernel    : first sorted position of every group (category or image)
//   lvis_scan_kernel     : one CTA: kept = min(k, group size), exclusive scan over the groups
//   lvis_scatter_kernel  : the cut: the first k of every group, copied to the output pool in (group, score desc, arrival) order
//   lvis_match_kernel    : one CTA per (image, category) pair: fp64 bbIou and the greedy matching of all 10 thresholds x 4 area
//                          ranges (one thread each), match / ignore bits and the rank within the pair per detection
//   lvis_accumulate_kernel: one CTA per category: TP / FP scans, precision, suffix maximum and the 101 recall samples of every
//                          (threshold, area range, maxDets entry)
//
// No float atomics; every reduction is an integer scan or a maximum, so reruns are bit-identical.  Box arithmetic is IEEE fp32
// (rule 1) and fp64 (IoU, precision, recall) without contraction (__f*_rn / __d*_rn), as the CPU restatement computes it.
#include <climits>

#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int LV_TILE = 1024;
constexpr int LV_T = 10;       // IoU thresholds
constexpr int LV_A = 4;        // area ranges
constexpr int LV_V = LV_T * LV_A;
constexpr int LV_R = 101;      // recall samples
constexpr unsigned long long LV_NONE = ~0ull;
constexpr int64_t LV_MAX_ROWS = 1 << 30;   // merge-pass run arithmetic (a0 + 2 * run) stays in int

struct Key {
  unsigned long long a, b, c;
};
__device__ __forceinline__ bool key_less(const Key& x, const Key& y) {
  return x.a != y.a ? x.a < y.a : (x.b != y.b ? x.b < y.b : x.c < y.c);
}

__device__ __forceinline__ unsigned desc_bits(float s) {  // ascending key = descending score
  const unsigned u = __float_as_uint(s);
  return ~((u & 0x80000000u) ? ~u : (u | 0x80000000u));
}

template <typename T>
__device__ __forceinline__ int lower_bound(const T* v, int n, T x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (v[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ bool contains(const unsigned long long* v, int n, unsigned long long x) {
  const int i = lower_bound(v, n, x);
  return i < n && v[i] == x;
}

// ---- collect ---------------------------------------------------------------------------------------------------------
// packed [G][B][M + 1][6]; row M of every (g, b) = (count, ...).  Slot of row (g, b, r) = base + (b * G + g) * M + r: image
// order, then chunk order, then row order, which is the order the reference's prepare() sees the concatenated BoxList rows.
__global__ void __launch_bounds__(256) lvis_collect_kernel(const float* __restrict__ packed, int G, int B, int M,
                                                           const int* __restrict__ img_idx, const float* __restrict__ ratios,
                                                           const int* __restrict__ label_map, int n_labels,
                                                           const int* __restrict__ cat_ids, int K, int drop, int wh_plus_one,
                                                           float* __restrict__ score, float4* __restrict__ box,
                                                           int* __restrict__ img, int* __restrict__ cat,
                                                           long long* __restrict__ seq, long long base, long long seq_base,
                                                           int* __restrict__ bad, int* __restrict__ bad_img) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long total = (long)G * B * M;
  if (i >= total) return;
  const int r = (int)(i % M), g = (int)((i / M) % G), b = (int)(i / ((long)M * G));
  const float* blk = packed + ((long)g * B + b) * (M + 1) * 6;
  const float cnt = blk[(long)M * 6];
  const long slot = base + i;
  seq[slot] = seq_base + i;
  int c = -1, im = img_idx[b];
  if (r == 0 && !(cnt >= 0.f && cnt <= (float)M && cnt == floorf(cnt))) atomicAdd(bad, 1);   // count row check
  if ((float)r < cnt) {
    const float* row = blk + (long)r * 6;
    int lab = (int)row[5];
    const bool mapped = !label_map || (lab >= 0 && lab < n_labels && label_map[lab] >= 0);
    if (label_map) lab = mapped ? label_map[lab] : -1;
    const int p = lower_bound(cat_ids, K, lab);
    c = (p < K && cat_ids[p] == lab) ? p : -2;   // -2: a detection of a category outside the GT file
    if (bad_img && mapped && im < 0) atomicAdd(bad_img, 1);   // a result on an image outside the GT file
    const float rx = ratios[2 * b], ry = ratios[2 * b + 1];
    const float x1 = __fmul_rn(row[0], rx), y1 = __fmul_rn(row[1], ry);
    const float x2 = __fmul_rn(row[2], rx), y2 = __fmul_rn(row[3], ry);
    float w = __fsub_rn(x2, x1), h = __fsub_rn(y2, y1);
    if (wh_plus_one) {   // BoxList.convert("xywh"): x2 - x1 + 1 in fp32
      w = __fadd_rn(w, 1.f);
      h = __fadd_rn(h, 1.f);
    }
    box[slot] = make_float4(x1, y1, w, h);
    score[slot] = row[4];
  }
  // -1 = nothing this protocol can ever count: an empty slot; drop bit 0: a category outside the GT file (fixed AP: its top-k is
  // its own; COCO: it takes no place in a pair's top 100); drop bit 1: an image outside the GT file (standard AP: its top 300 is
  // its own).  Standard AP keeps -2 rows: they take places in their image's top 300.
  if (((drop & 1) && c == -2) || ((drop & 2) && im < 0)) c = -1;
  cat[slot] = c;
  img[slot] = im;
}

// ---- keys ------------------------------------------------------------------------------------------------------------
// mode 0 (cut, fixed AP) : (category, score desc, arrival)       mode 1 (cut, standard): (image, score desc, arrival)
// mode 2 (pairing)       : (image, category, score desc, arrival) of the detections of a GT image and category; with
//                          area_filter only 0 < w * h < inf, with federated only pairs in pos_pairs or neg_pairs
// mode 4 (cut, COCO)     : (image * n_cat + category, score desc, arrival)
// mode 3 (accumulation)  : (category, score desc, image, arrival) of the paired detections; c = position in the pairing order.
//                          Equal scores of one category go by image id, then by arrival: accumulate's stable sort of the
//                          detections concatenated in image order, each image's already in (score desc, arrival) order.
__global__ void __launch_bounds__(256) lvis_keys_kernel(int mode, int n, const float* __restrict__ score,
                                                        const float4* __restrict__ box, const int* __restrict__ img,
                                                        const int* __restrict__ cat, const long long* __restrict__ seq,
                                                        const unsigned long long* __restrict__ pos_pairs, int n_pos,
                                                        const unsigned long long* __restrict__ neg_pairs, int n_neg,
                                                        const Key* __restrict__ paired, int n_cat, int federated, int area_filter,
                                                        Key* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Key k{LV_NONE, LV_NONE, (unsigned long long)i};
  if (mode <= 1 || mode == 4) {
    const int grp = mode == 0 ? cat[i] : mode == 1 ? img[i] : (img[i] < 0 || cat[i] < 0 ? -1 : img[i] * n_cat + cat[i]);
    if (cat[i] != -1 && grp >= 0) {
      k.a = ((unsigned long long)grp << 32) | desc_bits(score[i]);
      k.b = (unsigned long long)seq[i];
    }
  } else if (mode == 2) {
    const int im = img[i], c = cat[i];
    if (im >= 0 && c >= 0) {
      const float4 bx = box[i];
      const double area = __dmul_rn((double)bx.z, (double)bx.w);
      const unsigned long long pc = ((unsigned long long)im << 32) | (unsigned)c;
      if ((!area_filter || (area > 0.0 && area < __longlong_as_double(0x7ff0000000000000ll))) &&
          (!federated || contains(pos_pairs, n_pos, pc) || contains(neg_pairs, n_neg, pc))) {
        k.a = pc;
        k.b = ((unsigned long long)desc_bits(score[i]) << 32) | (unsigned long long)(unsigned)seq[i];
      }
    }
  } else if (paired[i].a != LV_NONE) {
    const int p = (int)paired[i].c;
    k.a = ((unsigned long long)cat[p] << 32) | desc_bits(score[p]);
    k.b = ((unsigned long long)img[p] << 32) | (unsigned long long)(unsigned)seq[p];
  }
  keys[i] = k;
}

// ---- sort ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) lvis_tile_sort_kernel(Key* __restrict__ keys, int n) {
  __shared__ Key s[LV_TILE];
  const int t0 = blockIdx.x * LV_TILE;
  for (int j = threadIdx.x; j < LV_TILE; j += 512) s[j] = t0 + j < n ? keys[t0 + j] : Key{LV_NONE, LV_NONE, LV_NONE};
  __syncthreads();
  for (int k = 2; k <= LV_TILE; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < LV_TILE; i += 512) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const Key x = s[i], y = s[ixj];
          if (key_less(y, x) == ((i & k) == 0)) {
            s[i] = y;
            s[ixj] = x;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int j = threadIdx.x; j < LV_TILE && t0 + j < n; j += 512) keys[t0 + j] = s[j];
}

__global__ void __launch_bounds__(256) lvis_merge_pass_kernel(const Key* __restrict__ src, Key* __restrict__ dst, int n,
                                                              int run) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const int a0 = i / (2 * run) * (2 * run);
  const int a1 = min(a0 + run, n), b1 = min(a0 + 2 * run, n);
  const Key key = src[i];
  int lo, hi;
  if (i < a1) { lo = a1; hi = b1; } else { lo = a0; hi = a1; }
  const int base = lo;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (key_less(src[mid], key)) lo = mid + 1; else hi = mid;
  }
  dst[a0 + (i < a1 ? i - a0 : i - a1) + (lo - base)] = key;
}

// ---- the cut ---------------------------------------------------------------------------------------------------------
// start[g] = first sorted position of group g (g = n_groups: the end of the valid keys)
__global__ void __launch_bounds__(256) lvis_group_kernel(const Key* __restrict__ keys, int n, int n_groups,
                                                         int* __restrict__ start) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g > n_groups) return;
  const unsigned long long x = g == n_groups ? LV_NONE : (unsigned long long)g << 32;
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid].a < x) lo = mid + 1; else hi = mid;
  }
  start[g] = lo;
}

// One CTA: off[g] = sum over groups before g of min(k, size); off[n_groups] = total kept (also written to *count).
__global__ void __launch_bounds__(1024) lvis_scan_kernel(const int* __restrict__ start, int n_groups, int k, int* __restrict__ off,
                                                         int* __restrict__ count) {
  __shared__ int warp_sum[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n_groups; base += 1024) {
    const int g = base + threadIdx.x;
    const int v = g < n_groups ? min(k, start[g + 1] - start[g]) : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    int wo = 0, tot = 0;
    for (int w = 0; w < 32; ++w) {
      if (w < warp) wo += warp_sum[w];
      tot += warp_sum[w];
    }
    const int c0 = carry;
    if (g < n_groups) off[g] = c0 + wo + x - v;
    __syncthreads();
    if (threadIdx.x == 0) carry = c0 + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    off[n_groups] = carry;
    *count = carry;
  }
}

__global__ void __launch_bounds__(256) lvis_scatter_kernel(const Key* __restrict__ keys, int n, const int* __restrict__ start,
                                                           const int* __restrict__ off, int k, const float* __restrict__ score,
                                                           const float4* __restrict__ box, const int* __restrict__ img,
                                                           const int* __restrict__ cat, const long long* __restrict__ seq,
                                                           float* __restrict__ o_score, float4* __restrict__ o_box,
                                                           int* __restrict__ o_img, int* __restrict__ o_cat,
                                                           long long* __restrict__ o_seq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Key key = keys[i];
  if (key.a == LV_NONE) return;
  const int g = (int)(key.a >> 32);
  const int r = i - start[g];
  if (r >= k) return;
  const int p = (int)key.c, o = off[g] + r;
  o_score[o] = score[p]; o_box[o] = box[p]; o_img[o] = img[p]; o_cat[o] = cat[p]; o_seq[o] = seq[p];
}

// ---- matching --------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double bb_iou(const float4 d, const double4 g, bool crowd) {   // pycocotools bbIou
  const double dx = d.x, dy = d.y, dw = d.z, dh = d.w;
  const double w = __dsub_rn(fmin(__dadd_rn(dw, dx), __dadd_rn(g.z, g.x)), fmax(dx, g.x));
  if (w <= 0.0) return 0.0;
  const double h = __dsub_rn(fmin(__dadd_rn(dh, dy), __dadd_rn(g.w, g.y)), fmax(dy, g.y));
  if (h <= 0.0) return 0.0;
  const double in = __dmul_rn(w, h);
  if (crowd) return __ddiv_rn(in, __dmul_rn(dw, dh));   // a crowd GT: the union is the detection
  return __ddiv_rn(in, __dsub_rn(__dadd_rn(__dmul_rn(dw, dh), __dmul_rn(g.z, g.w)), in));
}

// Block = one position of the pairing order; only the first detection of each (image, category) pair does work.  Thread v < 40
// runs threshold v % 10 in area range v / 10 over the pair's detections in order.  used = per-(variant, GT) matched flags; a
// crowd GT (gt_crowd non-null) is never used up.  A match to the GT with id 0 uses it up but counts as no match (pycocotools'
// dtm holds the GT id and tests it for != 0): not a TP, ignored only for its GT or for its own area.
__global__ void __launch_bounds__(64) lvis_match_kernel(const Key* __restrict__ keys, int n_valid, const float4* __restrict__ box,
                                                        const unsigned long long* __restrict__ gt_pair, int n_gt,
                                                        const double4* __restrict__ gt_box, const double* __restrict__ gt_area,
                                                        const int* __restrict__ gt_ign, const long long* __restrict__ gt_id,
                                                        const int* __restrict__ gt_crowd,
                                                        const unsigned long long* __restrict__ nel_pairs, int n_nel,
                                                        const double* __restrict__ iou_thrs, const double* __restrict__ area_rng,
                                                        unsigned char* __restrict__ used, unsigned long long* __restrict__ tp_bits,
                                                        unsigned long long* __restrict__ ig_bits, int* __restrict__ match_gt,
                                                        int* __restrict__ rank) {
  const int s = blockIdx.x;
  const unsigned long long pc = keys[s].a;
  if (pc == LV_NONE || (s > 0 && keys[s - 1].a == pc)) return;
  __shared__ int e_s;
  if (threadIdx.x == 0) {
    int lo = s, hi = n_valid;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (keys[mid].a <= pc) lo = mid + 1; else hi = mid;
    }
    e_s = lo;
  }
  __syncthreads();
  const int e = e_s;
  const int v = threadIdx.x;
  if (v == LV_V)
    for (int i = s; i < e; ++i) rank[i] = i - s;
  if (v >= LV_V) return;
  const int t = v % LV_T, ar = v / LV_T;
  const double lo_a = area_rng[2 * ar], hi_a = area_rng[2 * ar + 1];
  const double thr = fmin(iou_thrs[t], 1.0 - 1e-10);
  const int g0 = lower_bound(gt_pair, n_gt, pc);
  int g1 = g0;
  while (g1 < n_gt && gt_pair[g1] == pc) ++g1;
  const bool nel = contains(nel_pairs, n_nel, pc);
  unsigned char* u = used + (long)v * n_gt;
  for (int j = g0; j < g1; ++j) u[j] = 0;
  const unsigned long long bit = 1ull << v;
  for (int i = s; i < e; ++i) {
    const float4 d = box[(int)keys[i].c];
    double best = thr;
    int m = -1, m_ig = 0;
    if (g1 > g0) {
      for (int pass = 0; pass < 2; ++pass) {   // GTs of the range first, then the ignored ones, each in annotation order
        if (pass == 1 && m > -1 && m_ig == 0) break;
        for (int j = g0; j < g1; ++j) {
          const int ig = gt_ign[j] || gt_area[j] < lo_a || gt_area[j] > hi_a;
          const bool crowd = gt_crowd && gt_crowd[j];
          if (ig != pass || (u[j] && !crowd)) continue;
          const double iou = bb_iou(d, gt_box[j], crowd);
          if (iou < best) continue;
          best = iou;
          m = j;
          m_ig = ig;
        }
      }
    }
    const double da = __dmul_rn((double)d.z, (double)d.w);
    const bool matched = m >= 0 && gt_id[m] != 0;
    bool ignored = false;
    if (m >= 0) {
      u[m] = 1;
      ignored = m_ig;
    }
    if (!matched) ignored = ignored || da < lo_a || da > hi_a || nel;
    if (match_gt) match_gt[(long)i * LV_V + v] = matched ? (int)gt_id[m] : 0;
    if (matched) atomicOr(tp_bits + i, bit);
    if (ignored) atomicOr(ig_bits + i, bit);
  }
}

// ---- accumulation ----------------------------------------------------------------------------------------------------
constexpr int LV_ACC = 256;

__device__ __forceinline__ int block_incl_scan(int x, int* ws) {   // inclusive sum over the block, LV_ACC threads
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) ws[warp] = x;
  __syncthreads();
  int wo = 0;
  for (int w = 0; w < warp; ++w) wo += ws[w];
  __syncthreads();
  return x + wo;
}

// Block = one category.  keys = accumulation order (mode 3, sorted); c of a key = position in the pairing order.  maxDets entry m
// (max_dets null: one entry, no bound) counts a detection only when its rank within its pair is below max_dets[m]; the others
// add neither TP nor FP, which leaves the samples of the shorter list unchanged (a left search never lands on them first except
// at recall 0, where the suffix maximum is the same).
__global__ void __launch_bounds__(LV_ACC) lvis_accumulate_kernel(const Key* __restrict__ keys, int n_valid, int K,
                                                                  const unsigned long long* __restrict__ tp_bits,
                                                                  const unsigned long long* __restrict__ ig_bits,
                                                                  const int* __restrict__ rank, const int* __restrict__ max_dets,
                                                                  int M,
                                                                  const int* __restrict__ num_gt, const double* __restrict__ rec_thrs,
                                                                  int* __restrict__ tp_ws, int* __restrict__ fp_ws,
                                                                  double* __restrict__ q_ws, double* __restrict__ precision,
                                                                  double* __restrict__ recall) {
  const int k = blockIdx.x;
  __shared__ int s_se[2];
  __shared__ int ws[32];
  __shared__ int carry[2];
  __shared__ double dws[32];
  __shared__ double dcarry;
  if (threadIdx.x < 2) {
    const unsigned long long x = (unsigned long long)(k + threadIdx.x) << 32;
    int lo = 0, hi = n_valid;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (keys[mid].a < x) lo = mid + 1; else hi = mid;
    }
    s_se[threadIdx.x] = lo;
  }
  __syncthreads();
  const int s = s_se[0], n = s_se[1] - s_se[0];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double eps = 2.220446049250313e-16;   // np.spacing(1)
  for (int vm = 0; vm < LV_V * M; ++vm) {
    const int v = vm / M, mi = vm % M;
    const int t = v % LV_T, ar = v / LV_T;
    const int ng = num_gt[k * LV_A + ar];
    if (ng == 0) continue;   // stays -1
    const int md = max_dets ? max_dets[mi] : INT_MAX;
    const unsigned long long bit = 1ull << v;
    if (threadIdx.x < 2) carry[threadIdx.x] = 0;
    __syncthreads();
    for (int base = 0; base < n; base += LV_ACC) {
      const int i = base + threadIdx.x;
      int tp = 0, fp = 0;
      if (i < n) {
        const int p = (int)keys[s + i].c;
        const bool m = tp_bits[p] & bit, ig = ig_bits[p] & bit;
        const bool in = !max_dets || rank[p] < md;
        tp = in && m && !ig;
        fp = in && !m && !ig;
      }
      const int c0 = carry[0], c1 = carry[1];
      const int tps = block_incl_scan(tp, ws) + c0;
      const int fps = block_incl_scan(fp, ws) + c1;
      if (i < n) { tp_ws[s + i] = tps; fp_ws[s + i] = fps; }
      __syncthreads();
      if (threadIdx.x == LV_ACC - 1) { carry[0] = tps; carry[1] = fps; }
      __syncthreads();
    }
    // suffix maximum of pr = tp / (fp + tp + eps), from the right
    if (threadIdx.x == 0) dcarry = 0.0;
    __syncthreads();
    for (int base = ((n - 1) / LV_ACC) * LV_ACC; n > 0 && base >= 0; base -= LV_ACC) {
      const int i = base + (LV_ACC - 1 - threadIdx.x);   // thread 0 holds the rightmost element of the chunk
      double x = 0.0;
      if (i < n) {
        const double tp = (double)tp_ws[s + i], fp = (double)fp_ws[s + i];
        x = __ddiv_rn(tp, __dadd_rn(__dadd_rn(fp, tp), eps));
      }
      for (int o = 1; o < 32; o <<= 1) {
        const double y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x = fmax(x, y);
      }
      if (lane == 31) dws[warp] = x;
      __syncthreads();
      double wo = dcarry;
      for (int w = 0; w < warp; ++w) wo = fmax(wo, dws[w]);
      x = fmax(x, wo);
      if (i < n) q_ws[s + i] = x;
      __syncthreads();
      if (threadIdx.x == LV_ACC - 1) dcarry = x;
      __syncthreads();
    }
    const double ngd = (double)ng;
    for (int r = threadIdx.x; r < LV_R; r += LV_ACC) {   // searchsorted(rc, rec_thrs, "left"); past the end stays 0
      const double thr_r = rec_thrs[r];
      int lo = 0, hi = n;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ddiv_rn((double)tp_ws[s + mid], ngd) < thr_r) lo = mid + 1; else hi = mid;
      }
      precision[((((long)t * LV_R + r) * K + k) * LV_A + ar) * M + mi] = lo < n ? q_ws[s + lo] : 0.0;
    }
    if (threadIdx.x == 0) recall[(((long)t * K + k) * LV_A + ar) * M + mi] = n ? __ddiv_rn((double)tp_ws[s + n - 1], ngd) : 0.0;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) lvis_order_kernel(const Key* __restrict__ paired, int n, int* __restrict__ order) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) order[i] = paired[i].a == LV_NONE ? -1 : (int)paired[i].c;
}

static inline size_t lv_align(size_t x) { return (x + 255) & ~(size_t)255; }

static Key* lv_sort(Key* a, Key* b, int n, cudaStream_t st) {
  if (n <= 0) return a;
  lvis_tile_sort_kernel<<<cdiv(n, LV_TILE), 512, 0, st>>>(a, n);
  for (long run = LV_TILE; run < n; run *= 2) {
    lvis_merge_pass_kernel<<<cdiv(n, 256), 256, 0, st>>>(a, b, n, (int)run);
    Key* t = a; a = b; b = t;
  }
  return a;
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_lvis_collect(const float* packed, int64_t G, int64_t B, int64_t M, const int32_t* img_idx, const float* ratios,
                                  const int32_t* label_map, int64_t n_labels, const int32_t* cat_ids, int64_t K, int drop,
                                  int wh_plus_one, float* score, float* box, int32_t* img, int32_t* cat, int64_t* seq, int64_t base,
                                  int64_t seq_base, int32_t* bad, int32_t* bad_img, void* stream) {
  MQ_REQUIRE(packed && img_idx && ratios && cat_ids && score && box && img && cat && seq && bad, "lvis_collect: null pointer");
  MQ_REQUIRE(G > 0 && B > 0 && M > 0 && K > 0 && base >= 0 && seq_base >= 0, "lvis_collect: bad sizes G=%ld B=%ld M=%ld K=%ld",
             (long)G, (long)B, (long)M, (long)K);
  MQ_REQUIRE(drop >= 0 && drop <= 3, "lvis_collect: drop flags %d outside 0..3", drop);
  MQ_REQUIRE(base + G * B * M <= LV_MAX_ROWS && seq_base + G * B * M <= (int64_t)UINT32_MAX, "lvis_collect: pool or arrival count overflow");
  lvis_collect_kernel<<<cdiv(G * B * M, 256), 256, 0, (cudaStream_t)stream>>>(
      packed, (int)G, (int)B, (int)M, img_idx, ratios, label_map, (int)n_labels, cat_ids, (int)K, drop, wh_plus_one, score,
      (float4*)box, img, cat, (long long*)seq, base, seq_base, bad, bad_img);
  return check_launch("lvis_collect_kernel");
}

extern "C" int64_t mqdet_lvis_cut_workspace_bytes(int64_t n, int64_t n_groups) {
  if (n < 0 || n_groups < 0) return 256;
  return (int64_t)(2 * lv_align((size_t)n * sizeof(Key)) + 2 * lv_align((size_t)(n_groups + 1) * 4) + 256);
}

extern "C" int mqdet_lvis_cut(const float* score, const float* box, const int32_t* img, const int32_t* cat, const int64_t* seq,
                              int64_t n, int group, int64_t n_groups, int64_t n_cat, int64_t k, float* o_score, float* o_box,
                              int32_t* o_img, int32_t* o_cat, int64_t* o_seq, int32_t* count, void* workspace, void* stream) {
  MQ_REQUIRE(score && box && img && cat && seq && o_score && o_box && o_img && o_cat && o_seq && count && workspace,
             "lvis_cut: null pointer");
  MQ_REQUIRE(n >= 0 && n <= LV_MAX_ROWS && n_groups > 0 && n_groups < INT32_MAX && k > 0, "lvis_cut: bad sizes n=%ld groups=%ld k=%ld",
             (long)n, (long)n_groups, (long)k);
  MQ_REQUIRE(group >= 0 && group <= 2 && (group != 2 || (n_cat > 0 && n_groups % n_cat == 0)),
             "lvis_cut: grouping %d with %ld groups of %ld categories", group, (long)n_groups, (long)n_cat);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* ws = (uint8_t*)workspace;
  Key* k0 = (Key*)ws;  ws += lv_align((size_t)n * sizeof(Key));
  Key* k1 = (Key*)ws;  ws += lv_align((size_t)n * sizeof(Key));
  int* start = (int*)ws;  ws += lv_align((size_t)(n_groups + 1) * 4);
  int* off = (int*)ws;
  if (n > 0)
    lvis_keys_kernel<<<cdiv(n, 256), 256, 0, st>>>(group == 2 ? 4 : group, (int)n, score, (const float4*)box, img, cat,
                                                   (const long long*)seq, nullptr, 0, nullptr, 0, nullptr, (int)n_cat, 0, 0, k0);
  Key* sorted = lv_sort(k0, k1, (int)n, st);
  lvis_group_kernel<<<cdiv(n_groups + 1, 256), 256, 0, st>>>(sorted, (int)n, (int)n_groups, start);
  lvis_scan_kernel<<<1, 1024, 0, st>>>(start, (int)n_groups, (int)k, off, count);
  if (n > 0)
    lvis_scatter_kernel<<<cdiv(n, 256), 256, 0, st>>>(sorted, (int)n, start, off, (int)k, score, (const float4*)box, img, cat,
                                                      (const long long*)seq, o_score, (float4*)o_box, o_img, o_cat, (long long*)o_seq);
  return check_launch("lvis_cut");
}

extern "C" int64_t mqdet_lvis_evaluate_workspace_bytes(int64_t n, int64_t n_gt) {
  if (n < 0 || n_gt < 0) return 256;
  const size_t m = (size_t)n;
  return (int64_t)(3 * lv_align(m * sizeof(Key)) + 3 * lv_align(m * 4) + lv_align(m * 8) + lv_align((size_t)LV_V * n_gt) + 256);
}

extern "C" int mqdet_lvis_evaluate(const float* score, const float* box, const int32_t* img, const int32_t* cat, const int64_t* seq,
                                   int64_t n, int64_t K, int federated, const int64_t* pos_pairs, int64_t n_pos, const int64_t* neg_pairs,
                                   int64_t n_neg, const int64_t* nel_pairs, int64_t n_nel, int area_filter, const int64_t* gt_pair,
                                   const double* gt_box, const double* gt_area, const int32_t* gt_ignore, const int32_t* gt_crowd,
                                   const int64_t* gt_id, int64_t n_gt, const int32_t* num_gt, const double* iou_thrs,
                                   const double* rec_thrs, const double* area_rng, const int32_t* max_dets, int64_t n_max_dets,
                                   double* precision, double* recall, int32_t* n_paired, int32_t* order, int64_t* tp_bits,
                                   int64_t* ig_bits, int32_t* match_gt, void* workspace, void* stream) {
  MQ_REQUIRE(score && box && img && cat && seq && num_gt && iou_thrs && rec_thrs && area_rng && precision && recall && n_paired &&
             order && tp_bits && ig_bits && workspace, "lvis_evaluate: null pointer");
  MQ_REQUIRE(n >= 0 && n <= LV_MAX_ROWS && K > 0 && n_gt >= 0 && n_gt <= INT32_MAX, "lvis_evaluate: bad sizes n=%ld K=%ld n_gt=%ld",
             (long)n, (long)K, (long)n_gt);
  MQ_REQUIRE(n_max_dets >= 1 && n_max_dets <= 16 && (max_dets || n_max_dets == 1), "lvis_evaluate: %ld maxDets entries",
             (long)n_max_dets);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t m = (size_t)n;
  const int M = (int)n_max_dets;
  uint8_t* ws = (uint8_t*)workspace;
  Key* k0 = (Key*)ws;                          ws += lv_align(m * sizeof(Key));
  Key* k1 = (Key*)ws;                          ws += lv_align(m * sizeof(Key));
  Key* k2 = (Key*)ws;                          ws += lv_align(m * sizeof(Key));
  int* tp_ws = (int*)ws;                       ws += lv_align(m * 4);
  int* fp_ws = (int*)ws;                       ws += lv_align(m * 4);
  int* rank = (int*)ws;                        ws += lv_align(m * 4);
  double* q_ws = (double*)ws;                  ws += lv_align(m * 8);
  unsigned char* used = (unsigned char*)ws;
  MQ_REQUIRE(cudaMemsetAsync(n_paired, 0, 4, st) == cudaSuccess, "lvis_evaluate: memset failed");
  if (n == 0) {
    lvis_accumulate_kernel<<<(unsigned)K, LV_ACC, 0, st>>>(k0, 0, (int)K, nullptr, nullptr, rank, max_dets, M, num_gt, rec_thrs, tp_ws,
                                                           fp_ws, q_ws, precision, recall);
    return check_launch("lvis_evaluate");
  }
  lvis_keys_kernel<<<cdiv(n, 256), 256, 0, st>>>(2, (int)n, score, (const float4*)box, img, cat, (const long long*)seq,
                                                 (const unsigned long long*)pos_pairs, (int)n_pos, (const unsigned long long*)neg_pairs,
                                                 (int)n_neg, nullptr, 0, federated, area_filter, k0);
  Key* paired = lv_sort(k0, k1, (int)n, st);
  lvis_group_kernel<<<1, 256, 0, st>>>(paired, (int)n, 0, n_paired);   // first position of the unpaired (NONE) keys
  lvis_order_kernel<<<cdiv(n, 256), 256, 0, st>>>(paired, (int)n, order);
  MQ_REQUIRE(cudaMemsetAsync(tp_bits, 0, m * 8, st) == cudaSuccess && cudaMemsetAsync(ig_bits, 0, m * 8, st) == cudaSuccess,
             "lvis_evaluate: memset failed");
  lvis_match_kernel<<<(unsigned)n, 64, 0, st>>>(paired, (int)n, (const float4*)box, (const unsigned long long*)gt_pair, (int)n_gt,
                                                (const double4*)gt_box, gt_area, gt_ignore, (const long long*)gt_id, gt_crowd,
                                                (const unsigned long long*)nel_pairs, (int)n_nel, iou_thrs, area_rng, used,
                                                (unsigned long long*)tp_bits, (unsigned long long*)ig_bits, match_gt, rank);
  Key* other = paired == k0 ? k1 : k0;
  lvis_keys_kernel<<<cdiv(n, 256), 256, 0, st>>>(3, (int)n, score, (const float4*)box, img, cat, (const long long*)seq, nullptr, 0,
                                                 nullptr, 0, paired, 0, 0, 0, k2);
  Key* acc = lv_sort(k2, other, (int)n, st);
  lvis_accumulate_kernel<<<(unsigned)K, LV_ACC, 0, st>>>(acc, (int)n, (int)K, (const unsigned long long*)tp_bits,
                                                         (const unsigned long long*)ig_bits, rank, max_dets, M, num_gt, rec_thrs, tp_ws,
                                                         fp_ws, q_ws, precision, recall);
  return check_launch("lvis_evaluate");
}
