// mqdet_b200 — ATSS target assignment and the pre-training detection losses on the device, with their gradients at the
// head outputs (dot-product token logits [B][N][T], raw box / centerness GEMM output reg_ctr [B][N][5]).
//
// Reference: maskrcnn_benchmark/modeling/rpn/loss.py ATSSLossComputation.prepare_targets :655-832, GIoULoss :612-653,
//            compute_centerness_targets :834-847, __call__ :850-1201; structures/boxlist_ops.py boxlist_iou :97-132;
//            layers/sigmoid_focal_loss.py token_sigmoid_binary_focal_loss :130-171.
//
// Assignment (one anchor per location; anchors generated analytically as in the post-processing):
//   1. atss_assign_kernel: one CTA per (image, GT).  Per level, the k = min(topk, level size) anchors with the smallest
//      centre distance (ties -> lower anchor index: the 64-bit key is distance bits << 32 | index), IoU of those candidates,
//      threshold = mean + unbiased std, positives = IoU >= threshold with the anchor centre inside the GT by > 0.01.
//      Conflicts: per-anchor atomicMax of (IoU bits << 32 | ~gt) -> highest IoU, then lowest GT index.  No [N x G] matrix.
//   2. atss_match_kernel: key -> match[b][n] (-1 = unmatched), per-block (num positives, sum centerness targets).
//   3. atss_norm_kernel: per-image sums and the normaliser buffer norm[4] = (num_pos, sum ctr) twice: [0:2] is what the
//      ranks all-reduce, [2:4] stays local (the reference's zero-positive / zero-weight branches are per rank).
// Losses (read the normalisers from device memory: no host synchronisation, capturable at a fixed GT capacity):
//   4. atss_token_loss_kernel: focal loss over all B*N*T elements under the text mask, targets built on the fly from match
//      and the GT token rows (one-hot at T-1 for unmatched anchors); writes d_logits.
//   5. atss_box_loss_kernel: GIoU (centerness-weighted) and centerness BCE over the positives; writes d_reg_ctr.
//   6. atss_loss_finalize_kernel: the partial sums in a fixed order -> losses (reg, centerness, token, cls = 0).
// Every reduction is two-stage with a fixed grid: no float atomics, the same bits on every run.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int AL_THREADS = 256;
constexpr int AL_TOPK_MAX = 16;
constexpr int AL_TOKEN_BLOCKS = 1024;

struct ALLevels {
  int n;
  int H[MQDET_MAX_LEVELS], W[MQDET_MAX_LEVELS], off[MQDET_MAX_LEVELS + 1];
  float stride[MQDET_MAX_LEVELS], base[MQDET_MAX_LEVELS][4], reg_scale[MQDET_MAX_LEVELS];
};

__device__ __forceinline__ int level_of(const ALLevels& lv, int n) {
  int l = 0;
  while (l + 1 < lv.n && n >= lv.off[l + 1]) ++l;
  return l;
}

// anchor_generator.py:72-94: base window of the level shifted by (x * stride, y * stride)
__device__ __forceinline__ void anchor_box(const ALLevels& lv, int l, int loc, float& x1, float& y1, float& x2, float& y2) {
  const float sx = (float)(loc % lv.W[l]) * lv.stride[l], sy = (float)(loc / lv.W[l]) * lv.stride[l];
  x1 = sx + lv.base[l][0];
  y1 = sy + lv.base[l][1];
  x2 = sx + lv.base[l][2];
  y2 = sy + lv.base[l][3];
}

__device__ __forceinline__ unsigned long long block_min_u64(unsigned long long v, unsigned long long* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long u = __shfl_xor_sync(0xffffffffu, v, o);
    v = u < v ? u : v;
  }
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  v = sh[0];
#pragma unroll
  for (int w = 1; w < AL_THREADS / 32; ++w) v = sh[w] < v ? sh[w] : v;
  __syncthreads();
  return v;  // valid in every thread
}

__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = threadIdx.x < AL_THREADS / 32 ? sh[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) r = warp_sum(r);
  __syncthreads();
  return r;  // valid in thread 0
}

template <int KMAX>
__global__ void __launch_bounds__(AL_THREADS) atss_assign_kernel(const float* __restrict__ gt_boxes, const int* __restrict__ gt_count,
                                                                 int Gmax, ALLevels lv, int topk,
                                                                 unsigned long long* __restrict__ keys) {
  __shared__ int s_cand[MQDET_MAX_LEVELS * AL_TOPK_MAX];
  __shared__ float s_iou[MQDET_MAX_LEVELS * AL_TOPK_MAX];
  __shared__ unsigned long long s_red[AL_THREADS / 32];
  __shared__ float s_thr;
  const int g = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  if (g >= min(gt_count[b], Gmax)) return;
  const int N = lv.off[lv.n];
  const float* gb = gt_boxes + ((long)b * Gmax + g) * 4;
  const float gx1 = gb[0], gy1 = gb[1], gx2 = gb[2], gy2 = gb[3];
  const float gcx = (gx2 + gx1) / 2.f, gcy = (gy2 + gy1) / 2.f;
  int nc = 0;
  for (int l = 0; l < lv.n; ++l) {
    const int hw = lv.H[l] * lv.W[l];
    const int k = min(topk, hw);
    unsigned long long best[KMAX];  // this thread's smallest keys, ascending
#pragma unroll
    for (int j = 0; j < KMAX; ++j) best[j] = ~0ull;
    for (int i = tid; i < hw; i += AL_THREADS) {
      float ax1, ay1, ax2, ay2;
      anchor_box(lv, l, i, ax1, ay1, ax2, ay2);
      const float dx = (ax2 + ax1) / 2.f - gcx, dy = (ay2 + ay1) / 2.f - gcy;
      // (a - g).pow(2).sum(-1).sqrt() rounded like the reference: no contraction into FMAs
      const float d = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
      unsigned long long key = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)i;
      if (key < best[KMAX - 1]) {
#pragma unroll
        for (int j = 0; j < KMAX; ++j) {
          if (key < best[j]) {
            const unsigned long long t = best[j];
            best[j] = key;
            key = t;
          }
        }
      }
    }
    for (int r = 0; r < k; ++r) {  // k rounds of a block-wide minimum over the list heads
      const unsigned long long m = block_min_u64(best[0], s_red);
      if (best[0] == m) {  // keys are unique: exactly one thread pops
#pragma unroll
        for (int j = 0; j < KMAX - 1; ++j) best[j] = best[j + 1];
        best[KMAX - 1] = ~0ull;
      }
      if (tid == 0) s_cand[nc + r] = lv.off[l] + (int)(m & 0xffffffffu);
    }
    nc += k;
  }
  __syncthreads();
  float acx = 0.f, acy = 0.f;
  if (tid < nc) {
    const int n = s_cand[tid];
    const int l = level_of(lv, n);
    float ax1, ay1, ax2, ay2;
    anchor_box(lv, l, n - lv.off[l], ax1, ay1, ax2, ay2);
    acx = (ax2 + ax1) / 2.f;
    acy = (ay2 + ay1) / 2.f;
    // boxlist_iou, TO_REMOVE = 1, rounded like the reference (no FMA contraction)
    const float a1 = __fmul_rn(ax2 - ax1 + 1.f, ay2 - ay1 + 1.f), a2 = __fmul_rn(gx2 - gx1 + 1.f, gy2 - gy1 + 1.f);
    const float w = fmaxf(fminf(ax2, gx2) - fmaxf(ax1, gx1) + 1.f, 0.f);
    const float h = fmaxf(fminf(ay2, gy2) - fmaxf(ay1, gy1) + 1.f, 0.f);
    const float inter = __fmul_rn(w, h);
    s_iou[tid] = __fdiv_rn(inter, __fsub_rn(__fadd_rn(a1, a2), inter));
  }
  __syncthreads();
  if (tid == 0) {
    // mean + unbiased std of the candidate IoUs (one candidate: std is NaN as in torch, so nothing is positive)
    double s = 0.0, ss = 0.0;
    for (int i = 0; i < nc; ++i) s += s_iou[i];
    const double mean = s / nc;
    for (int i = 0; i < nc; ++i) ss += (s_iou[i] - mean) * (s_iou[i] - mean);
    s_thr = nc > 1 ? (float)(mean + sqrt(ss / (nc - 1))) : __int_as_float(0x7fc00000);
  }
  __syncthreads();
  if (tid < nc) {
    const float iou = s_iou[tid];
    const float inside = fminf(fminf(acx - gx1, acy - gy1), fminf(gx2 - acx, gy2 - acy));
    if (iou >= s_thr && inside > 0.01f)
      atomicMax(&keys[(long)b * N + s_cand[tid]],
                ((unsigned long long)(__float_as_uint(iou) | 0x80000000u) << 32) | (unsigned)(~g));
  }
}

// Regression target of an anchor matched to GT box g (BoxCoder.encode, vldyhead.py:57-76) decoded back into a box
// (the reference decodes the encoded target for both the GIoU target box and the centerness target), and its centerness.
__device__ __forceinline__ DecodedBox gt_target(float ax1, float ay1, float ax2, float ay2, const float* g, float& ctr) {
  const float ew = ax2 - ax1 + 1.f, eh = ay2 - ay1 + 1.f;
  const float ecx = (ax2 + ax1) / 2.f, ecy = (ay2 + ay1) / 2.f;
  const float gw = g[2] - g[0] + 1.f, gh = g[3] - g[1] + 1.f;
  const float gcx = (g[2] + g[0]) / 2.f, gcy = (g[3] + g[1]) / 2.f;
  const float t0 = 10.f * (gcx - ecx) / ew, t1 = 10.f * (gcy - ecy) / eh;
  const float t2 = 5.f * logf(gw / ew), t3 = 5.f * logf(gh / eh);
  const DecodedBox d = box_decode(t0, t1, t2, t3, ax1, ay1, ax2, ay2);
  const float l = ecx - d.x1, t = ecy - d.y1, r = d.x2 - ecx, bb = d.y2 - ecy;
  ctr = sqrtf((fminf(l, r) / fmaxf(l, r)) * (fminf(t, bb) / fmaxf(t, bb)));
  return d;
}

__global__ void __launch_bounds__(AL_THREADS) atss_match_kernel(const unsigned long long* __restrict__ keys,
                                                                const float* __restrict__ gt_boxes,
                                                                const int* __restrict__ gt_labels, int Gmax, ALLevels lv,
                                                                int* __restrict__ match, float* __restrict__ partial) {
  __shared__ float sh[AL_THREADS / 32];
  const int b = blockIdx.y, n = blockIdx.x * AL_THREADS + threadIdx.x;
  const int N = lv.off[lv.n];
  float pos = 0.f, ctr = 0.f;
  if (n < N) {
    const unsigned long long key = keys[(long)b * N + n];
    const int m = key ? (int)~(unsigned)(key & 0xffffffffu) : -1;
    match[(long)b * N + n] = m;
    if (m >= 0 && gt_labels[(long)b * Gmax + m] > 0) {
      const int l = level_of(lv, n);
      float ax1, ay1, ax2, ay2;
      anchor_box(lv, l, n - lv.off[l], ax1, ay1, ax2, ay2);
      gt_target(ax1, ay1, ax2, ay2, gt_boxes + ((long)b * Gmax + m) * 4, ctr);
      pos = 1.f;
    }
  }
  pos = block_sum(pos, sh);
  ctr = block_sum(ctr, sh);
  if (threadIdx.x == 0) {
    float* p = partial + ((long)b * gridDim.x + blockIdx.x) * 2;
    p[0] = pos;
    p[1] = ctr;
  }
}

// img_stats[b] = (num_pos, sum ctr) of image b; norm = (sum num_pos, sum ctr, the same two again)
__global__ void __launch_bounds__(AL_THREADS) atss_norm_kernel(const float* __restrict__ partial, int nblk, int B,
                                                               float* __restrict__ img_stats, float* __restrict__ norm) {
  __shared__ float sh[AL_THREADS / 32];
  float tp = 0.f, tc = 0.f;
  for (int b = 0; b < B; ++b) {
    float p = 0.f, c = 0.f;
    for (int i = threadIdx.x; i < nblk; i += AL_THREADS) {
      p += partial[((long)b * nblk + i) * 2];
      c += partial[((long)b * nblk + i) * 2 + 1];
    }
    p = block_sum(p, sh);
    c = block_sum(c, sh);
    if (threadIdx.x == 0) {
      if (img_stats) {
        img_stats[2 * b] = p;
        img_stats[2 * b + 1] = c;
      }
      tp += p;
      tc += c;
    }
  }
  if (threadIdx.x == 0) {
    norm[0] = norm[2] = tp;
    norm[1] = norm[3] = tc;
  }
}

__device__ __forceinline__ float num_pos_avg(const float* norm, float world) { return fmaxf(norm[0] / world, 1.f); }

// One warp per anchor row; the token target of element t is gt_tokens[b][match][t] for a matched anchor, else (t == T-1).
__global__ void __launch_bounds__(AL_THREADS) atss_token_loss_kernel(const float* __restrict__ logits, const int* __restrict__ match,
                                                                     const float* __restrict__ gt_tokens, int Gmax,
                                                                     const float* __restrict__ text_mask, int T, int N, long rows,
                                                                     float alpha, float gamma, const float* __restrict__ norm,
                                                                     float world, float weight, float* __restrict__ partial,
                                                                     float* __restrict__ dlogits) {
  __shared__ float sh[AL_THREADS / 32];
  const int lane = threadIdx.x & 31;
  const float gs = weight / num_pos_avg(norm, world);
  float acc = 0.f;
  for (long row = (long)blockIdx.x * (AL_THREADS / 32) + (threadIdx.x >> 5); row < rows;
       row += (long)gridDim.x * (AL_THREADS / 32)) {
    const long b = row / N;
    const int m = match[row];
    const float* tok = m >= 0 ? gt_tokens + ((long)b * Gmax + m) * T : nullptr;
    const float* tm = text_mask ? text_mask + b * T : nullptr;
    const float* x = logits + row * T;
    float* dx = dlogits + row * T;
    for (int t = lane; t < T; t += 32) {
      float l = 0.f, d = 0.f;
      if (!tm || tm[t] > 0.f) token_focal_elem(x[t], tok ? tok[t] : (t == T - 1 ? 1.f : 0.f), alpha, gamma, l, d);
      acc += l;
      dx[t] = d * gs;
    }
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}

// gradient of torch.max(a, b) / torch.min(a, b): to the selected input, split in halves on a tie
__device__ __forceinline__ void dmax(float a, float b, float g, float& ga, float& gb) {
  if (a > b) ga += g;
  else if (a < b) gb += g;
  else { ga += 0.5f * g; gb += 0.5f * g; }
}
__device__ __forceinline__ void dmin(float a, float b, float g, float& ga, float& gb) {
  if (a < b) ga += g;
  else if (a > b) gb += g;
  else { ga += 0.5f * g; gb += 0.5f * g; }
}

// One thread per anchor: GIoU + centerness BCE of the positives (label > 0), d_reg_ctr of every anchor.
__global__ void __launch_bounds__(AL_THREADS) atss_box_loss_kernel(const float* __restrict__ reg_ctr, const int* __restrict__ match,
                                                                   const float* __restrict__ gt_boxes, const int* __restrict__ gt_labels,
                                                                   int Gmax, ALLevels lv, const float* __restrict__ norm, float world,
                                                                   float reg_weight, float* __restrict__ partial,
                                                                   float* __restrict__ d_reg_ctr) {
  __shared__ float sh[AL_THREADS / 32];
  const int b = blockIdx.y, n = blockIdx.x * AL_THREADS + threadIdx.x;
  const int N = lv.off[lv.n];
  float lw = 0.f, lsum = 0.f, bce = 0.f;
  if (n < N) {
    const long row = (long)b * N + n;
    const int m = match[row];
    float g5[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (m >= 0 && gt_labels[(long)b * Gmax + m] > 0) {
      const int l = level_of(lv, n);
      float ax1, ay1, ax2, ay2;
      anchor_box(lv, l, n - lv.off[l], ax1, ay1, ax2, ay2);
      float w;
      const DecodedBox tb = gt_target(ax1, ay1, ax2, ay2, gt_boxes + ((long)b * Gmax + m) * 4, w);
      const float* r = reg_ctr + row * 5;
      const float sc = lv.reg_scale[l];
      const float p0 = r[0] * sc, p1 = r[1] * sc, p2 = r[2] * sc, p3 = r[3] * sc;
      const DecodedBox pb = box_decode(p0, p1, p2, p3, ax1, ay1, ax2, ay2);
      // GIoULoss (loss.py:612-653)
      const float px1 = pb.x1, py1 = pb.y1, px2 = fmaxf(pb.x1, pb.x2), py2 = fmaxf(pb.y1, pb.y2);
      const float pa = (px2 - px1) * (py2 - py1);
      const float ta = (tb.x2 - tb.x1) * (tb.y2 - tb.y1);
      const float ix1 = fmaxf(px1, tb.x1), iy1 = fmaxf(py1, tb.y1), ix2 = fminf(px2, tb.x2), iy2 = fminf(py2, tb.y2);
      const bool overlap = (iy2 > iy1) && (ix2 > ix1);
      const float ai = overlap ? (ix2 - ix1) * (iy2 - iy1) : 0.f;
      const float ex1 = fminf(px1, tb.x1), ey1 = fminf(py1, tb.y1), ex2 = fmaxf(px2, tb.x2), ey2 = fmaxf(py2, tb.y2);
      const float ae = (ex2 - ex1) * (ey2 - ey1) + 1e-7f;
      const float au = pa + ta - ai + 1e-7f;
      const float iou = ai / au;
      const float loss = 1.f - (iou - (ae - au) / ae);
      lw = loss * w;
      lsum = loss;
      // d loss_reg / d loss_i: centerness-weighted when the local weights sum to > 0 (norm[3]), / the all-rank normaliser
      const float coef = reg_weight / (norm[1] / world);
      const float g = norm[3] > 0.f ? w * coef : coef;
      float g_ai = -g / au;
      const float g_au = g * ai / (au * au) - g / ae;
      const float g_ae = g * au / (ae * ae);
      const float g_pa = g_au;
      g_ai -= g_au;
      float gpx1 = 0.f, gpy1 = 0.f, gpx2 = 0.f, gpy2 = 0.f, gt_ = 0.f;  // gt_: sink for the target's (unused) share
      if (overlap) {
        const float gx2i = g_ai * (iy2 - iy1), gy2i = g_ai * (ix2 - ix1);
        dmax(px1, tb.x1, -gx2i, gpx1, gt_);
        dmax(py1, tb.y1, -gy2i, gpy1, gt_);
        dmin(px2, tb.x2, gx2i, gpx2, gt_);
        dmin(py2, tb.y2, gy2i, gpy2, gt_);
      }
      const float gx2e = g_ae * (ey2 - ey1), gy2e = g_ae * (ex2 - ex1);
      dmin(px1, tb.x1, -gx2e, gpx1, gt_);
      dmin(py1, tb.y1, -gy2e, gpy1, gt_);
      dmax(px2, tb.x2, gx2e, gpx2, gt_);
      dmax(py2, tb.y2, gy2e, gpy2, gt_);
      gpx2 += g_pa * (py2 - py1);
      gpx1 -= g_pa * (py2 - py1);
      gpy2 += g_pa * (px2 - px1);
      gpy1 -= g_pa * (px2 - px1);
      // px2 = max(x1, x2), py2 = max(y1, y2)
      float gx1 = gpx1, gy1 = gpy1, gx2 = 0.f, gy2 = 0.f;
      dmax(pb.x1, pb.x2, gpx2, gx1, gx2);
      dmax(pb.y1, pb.y2, gpy2, gy1, gy2);
      // decode: x1/x2 = pcx -+ 0.5 (pw - 1), pcx = dx w + cx, pw = exp(dw) w; dw clamped from above (zero gradient there)
      const float aw = ax2 - ax1 + 1.f, ah = ay2 - ay1 + 1.f;
      const float g_pcx = gx1 + gx2, g_pcy = gy1 + gy2;
      const float g_pw = 0.5f * (gx2 - gx1), g_ph = 0.5f * (gy2 - gy1);
      g5[0] = g_pcx * aw / 10.f * sc;
      g5[1] = g_pcy * ah / 10.f * sc;
      g5[2] = p2 / 5.f <= BOX_DECODE_CLAMP ? g_pw * pb.pw / 5.f * sc : 0.f;
      g5[3] = p3 / 5.f <= BOX_DECODE_CLAMP ? g_ph * pb.ph / 5.f * sc : 0.f;
      // centerness: BCE with logits against the centerness target, / num_pos_avg
      const float x = r[4];
      bce = fmaxf(x, 0.f) - x * w + log1pf(expf(-fabsf(x)));
      g5[4] = (1.f / (1.f + expf(-x)) - w) / num_pos_avg(norm, world);
    }
    float* o = d_reg_ctr + row * 5;
#pragma unroll
    for (int j = 0; j < 5; ++j) o[j] = g5[j];
  }
  lw = block_sum(lw, sh);
  lsum = block_sum(lsum, sh);
  bce = block_sum(bce, sh);
  if (threadIdx.x == 0) {
    float* p = partial + ((long)b * gridDim.x + blockIdx.x) * 3;
    p[0] = lw;
    p[1] = lsum;
    p[2] = bce;
  }
}

// losses = (loss_reg, loss_centerness, loss_dot_product_token, loss_cls = 0)
__global__ void __launch_bounds__(AL_THREADS) atss_loss_finalize_kernel(const float* __restrict__ tok_partial, int ntok,
                                                                        const float* __restrict__ box_partial, int nbox,
                                                                        const float* __restrict__ norm, float world,
                                                                        float reg_weight, float* __restrict__ losses) {
  __shared__ float sh[AL_THREADS / 32];
  float t = 0.f, lw = 0.f, ls = 0.f, bc = 0.f;
  for (int i = threadIdx.x; i < ntok; i += AL_THREADS) t += tok_partial[i];
  for (int i = threadIdx.x; i < nbox; i += AL_THREADS) {
    lw += box_partial[3 * i];
    ls += box_partial[3 * i + 1];
    bc += box_partial[3 * i + 2];
  }
  t = block_sum(t, sh);
  lw = block_sum(lw, sh);
  ls = block_sum(ls, sh);
  bc = block_sum(bc, sh);
  if (threadIdx.x == 0) {
    const float npa = num_pos_avg(norm, world);
    const bool any_pos = norm[2] > 0.f;  // this rank's positives (loss.py:1185-1195)
    losses[0] = any_pos ? (norm[3] > 0.f ? lw : ls) / (norm[1] / world) * reg_weight : 0.f;
    losses[1] = any_pos ? bc / npa : 0.f;
    losses[2] = t / npa;
    losses[3] = 0.f;
  }
}

static int fill_al_levels(ALLevels* lv, const int32_t* level_hw, int64_t nlev, const float* strides, const float* base_anchors,
                          const float* reg_scales) {
  if (nlev < 1 || nlev > MQDET_MAX_LEVELS) return -1;
  lv->n = (int)nlev;
  long off = 0;
  for (int l = 0; l < nlev; ++l) {
    if (level_hw[2 * l] < 1 || level_hw[2 * l + 1] < 1) return -1;
    lv->H[l] = level_hw[2 * l];
    lv->W[l] = level_hw[2 * l + 1];
    lv->off[l] = (int)off;
    off += (long)lv->H[l] * lv->W[l];
    if (off >= (1l << 31)) return -1;
    lv->stride[l] = strides[l];
    for (int k = 0; k < 4; ++k) lv->base[l][k] = base_anchors[4 * l + k];
    lv->reg_scale[l] = reg_scales ? reg_scales[l] : 1.f;
  }
  lv->off[nlev] = (int)off;
  return (int)off;
}

static inline long al_blocks(long N) { return (N + AL_THREADS - 1) / AL_THREADS; }

}  // namespace mqdet

using namespace mqdet;

extern "C" int64_t mqdet_atss_assign_workspace_bytes(int64_t B, int64_t N) {
  if (B < 1 || N < 1) return 0;
  return B * N * 8 + B * al_blocks(N) * 2 * 4;
}

extern "C" int mqdet_atss_assign(const float* gt_boxes, const int32_t* gt_labels, const int32_t* gt_count, int64_t B, int64_t Gmax,
                                 const int32_t* level_hw, int64_t nlev, const float* strides, const float* base_anchors, int64_t topk,
                                 void* workspace, int32_t* match, float* img_stats, float* norm, void* stream) {
  MQ_REQUIRE(gt_boxes && gt_labels && gt_count && level_hw && strides && base_anchors && workspace && match && norm,
             "atss_assign: null pointer");
  MQ_REQUIRE(B >= 1 && B <= 65535, "atss_assign: B=%ld out of range 1..65535", (long)B);
  MQ_REQUIRE(Gmax >= 1 && Gmax <= (1l << 31) - 1, "atss_assign: GT capacity Gmax=%ld must be >= 1", (long)Gmax);
  MQ_REQUIRE(topk >= 1 && topk <= AL_TOPK_MAX, "atss_assign: topk=%ld out of range 1..%d", (long)topk, AL_TOPK_MAX);
  ALLevels lv;
  const int N = fill_al_levels(&lv, level_hw, nlev, strides, base_anchors, nullptr);
  MQ_REQUIRE(N > 0, "atss_assign: bad level table");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* keys = (unsigned long long*)workspace;
  float* partial = (float*)(keys + B * (long)N);
  if (cudaMemsetAsync(keys, 0, sizeof(unsigned long long) * B * (long)N, st) != cudaSuccess) return check_launch("atss_assign memset");
  const dim3 grid_g((unsigned)Gmax, (unsigned)B);
  if (topk <= 9)
    atss_assign_kernel<9><<<grid_g, AL_THREADS, 0, st>>>(gt_boxes, gt_count, (int)Gmax, lv, (int)topk, keys);
  else
    atss_assign_kernel<AL_TOPK_MAX><<<grid_g, AL_THREADS, 0, st>>>(gt_boxes, gt_count, (int)Gmax, lv, (int)topk, keys);
  int rc = check_launch("atss_assign_kernel");
  if (rc) return rc;
  const int nblk = (int)al_blocks(N);
  atss_match_kernel<<<dim3((unsigned)nblk, (unsigned)B), AL_THREADS, 0, st>>>(keys, gt_boxes, gt_labels, (int)Gmax, lv, match, partial);
  rc = check_launch("atss_match_kernel");
  if (rc) return rc;
  atss_norm_kernel<<<1, AL_THREADS, 0, st>>>(partial, nblk, (int)B, img_stats, norm);
  return check_launch("atss_norm_kernel");
}

extern "C" int64_t mqdet_atss_loss_workspace_floats(int64_t B, int64_t N) {
  if (B < 1 || N < 1) return 0;
  return AL_TOKEN_BLOCKS + B * al_blocks(N) * 3;
}

extern "C" int mqdet_atss_loss(const float* logits, const float* reg_ctr, const int32_t* match, const float* gt_boxes,
                               const int32_t* gt_labels, const float* gt_tokens, int64_t B, int64_t Gmax, int64_t T,
                               const float* text_mask, const int32_t* level_hw, int64_t nlev, const float* strides,
                               const float* base_anchors, const float* reg_scales, const float* norm, float world, float alpha,
                               float gamma, float reg_weight, float token_weight, float* workspace, float* losses,
                               float* d_logits, float* d_reg_ctr, void* stream) {
  MQ_REQUIRE(logits && reg_ctr && match && gt_boxes && gt_labels && gt_tokens && level_hw && strides && base_anchors && reg_scales &&
                 norm && workspace && losses && d_logits && d_reg_ctr,
             "atss_loss: null pointer");
  MQ_REQUIRE(B >= 1 && B <= 65535, "atss_loss: B=%ld out of range 1..65535", (long)B);
  MQ_REQUIRE(Gmax >= 1, "atss_loss: GT capacity Gmax=%ld must be >= 1", (long)Gmax);
  MQ_REQUIRE(T >= 1 && T <= (1l << 30), "atss_loss: bad token count T=%ld", (long)T);
  MQ_REQUIRE(world >= 1.f, "atss_loss: world size %g < 1", (double)world);
  ALLevels lv;
  const int N = fill_al_levels(&lv, level_hw, nlev, strides, base_anchors, reg_scales);
  MQ_REQUIRE(N > 0, "atss_loss: bad level table");
  cudaStream_t st = (cudaStream_t)stream;
  const long rows = B * (long)N;
  const long warps_needed = (rows + AL_THREADS / 32 - 1) / (AL_THREADS / 32);
  const int ntok = (int)(warps_needed < AL_TOKEN_BLOCKS ? warps_needed : AL_TOKEN_BLOCKS);
  float* tok_partial = workspace;
  float* box_partial = workspace + AL_TOKEN_BLOCKS;
  atss_token_loss_kernel<<<ntok, AL_THREADS, 0, st>>>(logits, match, gt_tokens, (int)Gmax, text_mask, (int)T, N, rows, alpha, gamma,
                                                      norm, world, token_weight, tok_partial, d_logits);
  int rc = check_launch("atss_token_loss_kernel");
  if (rc) return rc;
  const int nblk = (int)al_blocks(N);
  atss_box_loss_kernel<<<dim3((unsigned)nblk, (unsigned)B), AL_THREADS, 0, st>>>(reg_ctr, match, gt_boxes, gt_labels, (int)Gmax, lv,
                                                                                 norm, world, reg_weight, box_partial, d_reg_ctr);
  rc = check_launch("atss_box_loss_kernel");
  if (rc) return rc;
  atss_loss_finalize_kernel<<<1, AL_THREADS, 0, st>>>(tok_partial, ntok, box_partial, (int)(B * nblk), norm, world, reg_weight, losses);
  return check_launch("atss_loss_finalize_kernel");
}
