// mqdet_b200 — GroundingDINO set-prediction training losses on the device: the Hungarian matching cost, the linear sum
// assignment, and the token focal / L1 / GIoU losses with their gradients at the decoder outputs of every layer
// (pred_logits [L][B][Q][T] raw, pred_boxes [L][B][Q][4] sigmoid cxcywh).
//
// Reference: groundingdino_new/models/GroundingDINO/matcher.py HungarianMatcher.forward :49-86, loss.py SetCriterion :42-178,
//            util/box_ops.py :9-62, maskrcnn_benchmark/layers/sigmoid_focal_loss.py token_sigmoid_binary_focal_loss :130-171,
//            scipy.optimize.linear_sum_assignment (the shortest augmenting path method of D. F. Crouse, "On implementing 2D
//            rectangular assignment algorithms", IEEE TAES 52(4), 2016).
//
//   1. gdino_cost_kernel: C[l][b][q][g] = w_bbox * L1 + w_class * class - w_giou * GIoU for g < gt_count[b] (0 beyond), one
//      64-query x 32-GT tile per CTA.  class = mean over g's positive tokens of pos - neg (the focal costs of p = sigmoid(x));
//      it is the product [Q x T] . [T x G] of those differences with the 0/1 token indicators, staged through shared memory
//      in 32-token slices.  -inf logits give p = 0 and finite costs.  A GT with no positive token gets class cost 0.
//      norm[0] = sum_b gt_count[b] (the set-loss normaliser before the all-rank sum).
//   2. lsa_kernel: one warp per (layer, image) problem, see the comment above it.
//   3. gdino_token_loss_kernel / gdino_box_loss_kernel / gdino_loss_finalize_kernel: the losses of every layer, with d_logits
//      and d_boxes = the gradient of sum_l (w_ce loss_ce + w_bbox loss_bbox + w_giou loss_giou) (the reference's returned
//      dict, summed).  Every reduction is two-stage with a fixed grid: no float atomics, the same bits on every run.
// No host synchronisation anywhere: the normaliser stays on the device, so the whole chain is capturable at a fixed Gmax.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

#include <climits>

namespace mqdet {
namespace {

constexpr int GC_TQ = 64, GC_TG = 32, GC_TT = 32;  // cost tile: queries x GTs x tokens per slice
constexpr int GC_THREADS = 256;
constexpr int GL_THREADS = 256;
constexpr int GL_TOKEN_BLOCKS = 128;  // token-loss CTAs per layer (fixed: the partial sums are reduced in a fixed order)
constexpr int LSA_MAX_Q = 4096;

struct XYXY {
  float x0, y0, x1, y1;
};

// box_cxcywh_to_xyxy (box_ops.py:9-12)
__device__ __forceinline__ XYXY to_xyxy(const float* b) {
  const float hw = __fmul_rn(0.5f, b[2]), hh = __fmul_rn(0.5f, b[3]);
  return {__fsub_rn(b[0], hw), __fsub_rn(b[1], hh), __fadd_rn(b[0], hw), __fadd_rn(b[1], hh)};
}

struct GiouParts {
  float iw, ih, inter, a1, uni, ew, eh, area;
};

// generalized_box_iou (box_ops.py:22-62) of one pair, keeping what the gradient needs
__device__ __forceinline__ float giou_fwd(const XYXY& p, const XYXY& t, GiouParts& s) {
  s.a1 = __fmul_rn(p.x1 - p.x0, p.y1 - p.y0);
  const float a2 = __fmul_rn(t.x1 - t.x0, t.y1 - t.y0);
  s.iw = fmaxf(fminf(p.x1, t.x1) - fmaxf(p.x0, t.x0), 0.f);
  s.ih = fmaxf(fminf(p.y1, t.y1) - fmaxf(p.y0, t.y0), 0.f);
  s.inter = __fmul_rn(s.iw, s.ih);
  s.uni = __fsub_rn(__fadd_rn(s.a1, a2), s.inter);
  const float iou = __fdiv_rn(s.inter, __fadd_rn(s.uni, 1e-6f));
  s.ew = fmaxf(fmaxf(p.x1, t.x1) - fminf(p.x0, t.x0), 0.f);
  s.eh = fmaxf(fmaxf(p.y1, t.y1) - fminf(p.y0, t.y0), 0.f);
  s.area = __fmul_rn(s.ew, s.eh);
  return __fsub_rn(iou, __fdiv_rn(__fsub_rn(s.area, s.uni), __fadd_rn(s.area, 1e-6f)));
}

// gradient of torch.maximum(a, b) / torch.minimum(a, b): to the selected input, in halves on a tie
__device__ __forceinline__ float gmax_a(float a, float b, float g) { return a > b ? g : (a < b ? 0.f : 0.5f * g); }
__device__ __forceinline__ float gmin_a(float a, float b, float g) { return a < b ? g : (a > b ? 0.f : 0.5f * g); }

// s * (1 - GIoU(pred, target)) and its gradient w.r.t. the predicted cxcywh (torch conventions: clamp(min=0) passes the
// gradient at 0, min / max split it on a tie; the target side receives nothing)
__device__ __forceinline__ float giou_loss_grad(const float* pb, const float* gb, float s, float g[4]) {
  const XYXY p = to_xyxy(pb), t = to_xyxy(gb);
  GiouParts q;
  const float giou = giou_fwd(p, t, q);
  const float G = -s;  // d loss / d giou
  const float U = q.uni + 1e-6f, A = q.area + 1e-6f;
  const float g_uni = G * (-q.inter / (U * U) + 1.f / A);
  const float g_inter = G / U - g_uni;
  const float g_area = G * (-U / (A * A));
  const float g_a1 = g_uni;
  float gx0 = 0.f, gy0 = 0.f, gx1 = 0.f, gy1 = 0.f;
  // inter = clamp(min(x1) - max(x0), 0) * clamp(min(y1) - max(y0), 0)
  if (fminf(p.x1, t.x1) - fmaxf(p.x0, t.x0) >= 0.f) {
    const float gw = g_inter * q.ih;
    gx1 += gmin_a(p.x1, t.x1, gw);
    gx0 -= gmax_a(p.x0, t.x0, gw);
  }
  if (fminf(p.y1, t.y1) - fmaxf(p.y0, t.y0) >= 0.f) {
    const float gh = g_inter * q.iw;
    gy1 += gmin_a(p.y1, t.y1, gh);
    gy0 -= gmax_a(p.y0, t.y0, gh);
  }
  // enclosing area = clamp(max(x1) - min(x0), 0) * clamp(max(y1) - min(y0), 0)
  if (fmaxf(p.x1, t.x1) - fminf(p.x0, t.x0) >= 0.f) {
    const float gw = g_area * q.eh;
    gx1 += gmax_a(p.x1, t.x1, gw);
    gx0 -= gmin_a(p.x0, t.x0, gw);
  }
  if (fmaxf(p.y1, t.y1) - fminf(p.y0, t.y0) >= 0.f) {
    const float gh = g_area * q.ew;
    gy1 += gmax_a(p.y1, t.y1, gh);
    gy0 -= gmin_a(p.y0, t.y0, gh);
  }
  // a1 = (x1 - x0) * (y1 - y0)
  gx1 += g_a1 * (p.y1 - p.y0);
  gx0 -= g_a1 * (p.y1 - p.y0);
  gy1 += g_a1 * (p.x1 - p.x0);
  gy0 -= g_a1 * (p.x1 - p.x0);
  // x0 / x1 = cx -+ 0.5 w
  g[0] = gx0 + gx1;
  g[1] = gy0 + gy1;
  g[2] = 0.5f * (gx1 - gx0);
  g[3] = 0.5f * (gy1 - gy0);
  return s * (1.f - giou);
}

__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = threadIdx.x < GL_THREADS / 32 ? sh[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) r = warp_sum(r);
  __syncthreads();
  return r;  // valid in thread 0
}

__device__ __forceinline__ float num_boxes(const float* norm, float world) { return fmaxf(norm[0] / world, 1.f); }

__device__ __forceinline__ int gt_n(const int* gt_count, int b, int Gmax) { return min(max(gt_count[b], 0), Gmax); }

// ---- 1. matching cost -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(GC_THREADS) gdino_cost_kernel(const float* __restrict__ logits, const float* __restrict__ boxes,
                                                                const float* __restrict__ gt_boxes, const int* __restrict__ gt_count,
                                                                const float* __restrict__ gt_tokens, int B, int Q, int T, int Gmax,
                                                                float alpha, float w_class, float w_bbox, float w_giou,
                                                                float* __restrict__ cost, float* __restrict__ norm) {
  __shared__ float s_d[GC_TQ][GC_TT + 1];
  __shared__ float s_w[GC_TG][GC_TT + 1];
  const int lb = blockIdx.z, b = lb % B, tid = threadIdx.x;
  const int q0 = blockIdx.x * GC_TQ, g0 = blockIdx.y * GC_TG;
  const int G = gt_n(gt_count, b, Gmax);
  if (norm && (blockIdx.x | blockIdx.y | blockIdx.z) == 0 && tid == 0) {
    int s = 0;
    for (int i = 0; i < B; ++i) s += gt_n(gt_count, i, Gmax);
    norm[0] = (float)s;
  }
  const int tx = tid & 15, ty = tid >> 4;  // GTs g0 + tx + 16 j, queries q0 + ty + 16 k
  float acc[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}}, cnt[2] = {0.f, 0.f};
  if (g0 < G) {  // uniform over the CTA
    for (int t0 = 0; t0 < T; t0 += GC_TT) {
      for (int e = tid; e < GC_TQ * GC_TT; e += GC_THREADS) {
        const int qi = e / GC_TT, ti = e % GC_TT, q = q0 + qi, t = t0 + ti;
        float d = 0.f;
        if (q < Q && t < T) {
          // matcher.py:61-64 (gamma = 2)
          const float x = logits[((long)lb * Q + q) * T + t];
          const float p = 1.f / (1.f + expf(-x));
          const float pos = alpha * ((1.f - p) * (1.f - p)) * (-logf(p + 1e-8f));
          const float neg = (1.f - alpha) * (p * p) * (-logf(1.f - p + 1e-8f));
          d = pos - neg;
        }
        s_d[qi][ti] = d;
      }
      for (int e = tid; e < GC_TG * GC_TT; e += GC_THREADS) {
        const int gi = e / GC_TT, ti = e % GC_TT, g = g0 + gi, t = t0 + ti;
        s_w[gi][ti] = (g < G && t < T && gt_tokens[((long)b * Gmax + g) * T + t] > 0.f) ? 1.f : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int ti = 0; ti < GC_TT; ++ti) {
        const float w0 = s_w[tx][ti], w1 = s_w[tx + 16][ti];
        cnt[0] += w0;
        cnt[1] += w1;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float d = s_d[ty + 16 * k][ti];
          acc[k][0] = fmaf(d, w0, acc[k][0]);
          acc[k][1] = fmaf(d, w1, acc[k][1]);
        }
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int q = q0 + ty + 16 * k;
    if (q >= Q) continue;
    const float* pb = boxes + ((long)lb * Q + q) * 4;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int g = g0 + tx + 16 * j;
      if (g >= Gmax) continue;
      float c = 0.f;
      if (g < G) {
        const float* gb = gt_boxes + ((long)b * Gmax + g) * 4;
        const float cls = cnt[j] > 0.f ? acc[k][j] / cnt[j] : 0.f;
        const float l1 = fabsf(pb[0] - gb[0]) + fabsf(pb[1] - gb[1]) + fabsf(pb[2] - gb[2]) + fabsf(pb[3] - gb[3]);
        GiouParts s;
        const float giou = giou_fwd(to_xyxy(pb), to_xyxy(gb), s);
        c = (w_bbox * l1 + w_class * cls) + w_giou * (-giou);
      }
      cost[((long)lb * Q + q) * Gmax + g] = c;
    }
  }
}

// ---- 2. linear sum assignment ---------------------------------------------------------------------------------------
// cost [P][Q][Gmax] -> cost_t [P][Gmax][Q], so that a GT's row of the transposed problem is contiguous
__global__ void lsa_transpose_kernel(const float* __restrict__ cost, int Q, int Gmax, float* __restrict__ cost_t) {
  __shared__ float tile[32][33];
  const long p = blockIdx.z;
  const int q0 = blockIdx.x * 32, g0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int q = q0 + r, g = g0 + threadIdx.x;
    if (q < Q && g < Gmax) tile[r][threadIdx.x] = cost[(p * Q + q) * Gmax + g];
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int g = g0 + r, q = q0 + threadIdx.x;
    if (q < Q && g < Gmax) cost_t[(p * Gmax + g) * Q + q] = tile[threadIdx.x][r];
  }
}

// One warp per problem: the shortest augmenting path method that scipy.optimize.linear_sum_assignment implements, with the
// same operations in the same order, so that the result is index for index scipy's on the same fp32 matrix, ties included.
//
// The problem of p is the [Q x G] block cost[p][:, :G], G = counts[p % ncounts].  As in scipy, a tall matrix (G < Q) is
// solved transposed: nr = G rows (GTs) and nc = Q columns (queries); a square one (G = Q) as it is.  The cost is widened to
// double, and so are the dual potentials u (rows), v (columns) and the shortest path costs; rows are added one at a time:
//   * Dijkstra from the new row i over the columns still in the "remaining" list: reduced cost
//     r = ((minVal + c[i][j]) - u[i]) - v[j] (that evaluation order), relaxing spc[j] / path[j] when r < spc[j];
//   * the next column is the minimum of spc over the list, where a tie is resolved the way scipy's sequential scan resolves
//     it: it replaces its running best when spc[j] < best, or when spc[j] == best and column j is unassigned.  So among the
//     columns at the minimum, the LAST unassigned one in list order wins; if none is unassigned, the FIRST one.  The warp
//     computes the same winner with a min-reduction over the key (spc, -1 - position if unassigned else position);
//   * the list starts reversed (position k holds column nc - 1 - k) and loses the chosen entry by swap-removal with its
//     last entry, exactly as scipy's list does, so positions (and with them the tie winners) agree;
//   * the path ends at an unassigned column (the sink); then u[i] += minVal, u[r] += minVal - spc[col4row[r]] for the other
//     rows visited, v[j] -= minVal - spc[j] for the columns visited, and the path is flipped.
// Each list position is owned by one lane; relaxations touch distinct columns, so no two lanes write the same word.
// Output: match[p][q] = the GT matched to query q, or -1.  Costs must be finite (scipy raises on NaN / -inf).
__global__ void __launch_bounds__(32) lsa_kernel(const float* __restrict__ cost, const float* __restrict__ cost_t,
                                                 const int* __restrict__ counts, int ncounts, int Q, int Gmax,
                                                 int* __restrict__ match) {
  extern __shared__ double lsa_smem[];
  const int p = blockIdx.x, lane = threadIdx.x;
  const int G = min(max(counts[p % ncounts], 0), Gmax);
  int* out = match + (long)p * Q;
  for (int q = lane; q < Q; q += 32) out[q] = -1;
  if (G == 0) return;
  __syncwarp();
  const bool tr = G < Q;
  const int nr = tr ? G : Q, nc = tr ? Q : G;
  const float* base = tr ? cost_t + (long)p * Gmax * Q : cost + (long)p * Q * Gmax;
  const long ld = tr ? Q : Gmax;
  double* u = lsa_smem;
  double* v = u + Q;
  double* spc = v + Q;
  int* path = (int*)(spc + Q);
  int* col4row = path + Q;
  int* row4col = col4row + Q;
  int* rem = row4col + Q;
  unsigned char* SR = (unsigned char*)(rem + Q);
  unsigned char* SC = SR + Q;
  for (int k = lane; k < nr; k += 32) {
    u[k] = 0.0;
    col4row[k] = -1;
  }
  for (int k = lane; k < nc; k += 32) {
    v[k] = 0.0;
    row4col[k] = -1;
    path[k] = -1;
  }
  for (int cur = 0; cur < nr; ++cur) {
    for (int k = lane; k < nc; k += 32) {
      rem[k] = nc - k - 1;
      SC[k] = 0;
      spc[k] = INFINITY;
    }
    for (int k = lane; k < nr; k += 32) SR[k] = 0;
    __syncwarp();
    double minVal = 0.0;
    int numRem = nc, i = cur, sink = -1;
    while (sink == -1) {
      if (lane == 0) SR[i] = 1;
      const float* row = base + (long)i * ld;
      const double ui = u[i];
      double best = INFINITY;
      int bkey = INT_MAX, bpos = -1;
      for (int it = lane; it < numRem; it += 32) {
        const int j = rem[it];
        const double r = minVal + (double)row[j] - ui - v[j];
        double s = spc[j];
        if (r < s) {
          path[j] = i;
          spc[j] = r;
          s = r;
        }
        const int key = row4col[j] == -1 ? -1 - it : it;
        if (s < best || (s == best && key < bkey)) {
          best = s;
          bkey = key;
          bpos = it;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int ok = __shfl_xor_sync(0xffffffffu, bkey, o);
        const int op = __shfl_xor_sync(0xffffffffu, bpos, o);
        if (ob < best || (ob == best && ok < bkey)) {
          best = ob;
          bkey = ok;
          bpos = op;
        }
      }
      __syncwarp();
      minVal = best;
      if (bpos < 0 || minVal == INFINITY) return;  // infeasible (non-finite costs): the problem keeps match = -1
      const int j = rem[bpos];
      if (row4col[j] == -1) sink = j;
      else i = row4col[j];
      __syncwarp();
      if (lane == 0) {
        SC[j] = 1;
        rem[bpos] = rem[numRem - 1];
      }
      --numRem;
      __syncwarp();
    }
    if (lane == 0) u[cur] += minVal;
    for (int k = lane; k < nr; k += 32)
      if (SR[k] && k != cur) u[k] += minVal - spc[col4row[k]];
    for (int k = lane; k < nc; k += 32)
      if (SC[k]) v[k] -= minVal - spc[k];
    __syncwarp();
    if (lane == 0) {
      int j = sink;
      while (true) {
        const int r = path[j];
        row4col[j] = r;
        const int t = col4row[r];
        col4row[r] = j;
        j = t;
        if (r == cur) break;
      }
    }
    __syncwarp();
  }
  for (int k = lane; k < nr; k += 32) {
    if (tr) out[col4row[k]] = k;
    else out[k] = col4row[k];
  }
}

// ---- 3. losses and gradients ----------------------------------------------------------------------------------------
// One warp per query row: token focal loss under the text mask (loss.py:42-67); the target row is the matched GT's token row,
// or one-hot at T-1 for an unmatched query and for a GT whose row sums to 0 (loss.py:58-60).  Writes d_logits.
__global__ void __launch_bounds__(GL_THREADS) gdino_token_loss_kernel(const float* __restrict__ logits, const int* __restrict__ match,
                                                                      const float* __restrict__ gt_tokens, int Gmax,
                                                                      const float* __restrict__ text_mask, int T, int B, int Q,
                                                                      float alpha, float gamma, const float* __restrict__ norm,
                                                                      float world, float weight, float* __restrict__ partial,
                                                                      float* __restrict__ dlogits) {
  __shared__ float sh[GL_THREADS / 32];
  const int lane = threadIdx.x & 31, l = blockIdx.y;
  const long rows = (long)B * Q;
  const float gs = weight / num_boxes(norm, world);
  float acc = 0.f;
  for (long row = (long)blockIdx.x * (GL_THREADS / 32) + (threadIdx.x >> 5); row < rows; row += (long)gridDim.x * (GL_THREADS / 32)) {
    const long b = row / Q, lr = (long)l * rows + row;
    const int m = match[lr];
    const float* tok = m >= 0 ? gt_tokens + ((long)b * Gmax + m) * T : nullptr;
    if (tok) {
      float s = 0.f;
      for (int t = lane; t < T; t += 32) s += tok[t];
      if (warp_sum(s) == 0.f) tok = nullptr;
    }
    const float* tm = text_mask ? text_mask + b * T : nullptr;
    const float* x = logits + lr * T;
    float* dx = dlogits + lr * T;
    for (int t = lane; t < T; t += 32) {
      float e = 0.f, d = 0.f;
      if (!tm || tm[t] > 0.f) token_focal_elem(x[t], tok ? tok[t] : (t == T - 1 ? 1.f : 0.f), alpha, gamma, e, d);
      acc += e;
      dx[t] = d * gs;
    }
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) partial[(long)l * gridDim.x + blockIdx.x] = acc;
}

// One thread per query: L1 and 1 - GIoU of the matched pairs (loss.py:70-91) and d_boxes (0 for unmatched queries).
__global__ void __launch_bounds__(GL_THREADS) gdino_box_loss_kernel(const float* __restrict__ boxes, const int* __restrict__ match,
                                                                    const float* __restrict__ gt_boxes, int Gmax, int B, int Q,
                                                                    const float* __restrict__ norm, float world, float w_bbox,
                                                                    float w_giou, float* __restrict__ partial,
                                                                    float* __restrict__ dboxes) {
  __shared__ float sh[GL_THREADS / 32];
  const int l = blockIdx.y;
  const long rows = (long)B * Q, row = (long)blockIdx.x * GL_THREADS + threadIdx.x;
  float l1 = 0.f, lg = 0.f;
  if (row < rows) {
    const long lr = (long)l * rows + row;
    const int m = match[lr];
    float g[4] = {0.f, 0.f, 0.f, 0.f};
    if (m >= 0) {
      const float nb = num_boxes(norm, world);
      const float* pb = boxes + lr * 4;
      const float* gb = gt_boxes + ((row / Q) * Gmax + m) * 4;
      const float sb = w_bbox / nb;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float d = pb[k] - gb[k];
        l1 += fabsf(d);
        g[k] = d > 0.f ? sb : (d < 0.f ? -sb : 0.f);  // torch: sign(d), 0 at a tie
      }
      float gg[4];
      lg = giou_loss_grad(pb, gb, 1.f, gg);
      const float sg = w_giou / nb;
#pragma unroll
      for (int k = 0; k < 4; ++k) g[k] += sg * gg[k];
    }
    float* o = dboxes + lr * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = g[k];
  }
  l1 = block_sum(l1, sh);
  lg = block_sum(lg, sh);
  if (threadIdx.x == 0) {
    float* p = partial + ((long)l * gridDim.x + blockIdx.x) * 2;
    p[0] = l1;
    p[1] = lg;
  }
}

// losses[l] = (loss_ce, loss_bbox, loss_giou) of layer l, each (sum / num_boxes) * its weight (loss.py:166-171)
__global__ void __launch_bounds__(GL_THREADS) gdino_loss_finalize_kernel(const float* __restrict__ tok_partial, int ntok,
                                                                         const float* __restrict__ box_partial, int nbox, int L,
                                                                         const float* __restrict__ norm, float world, float w_ce,
                                                                         float w_bbox, float w_giou, float* __restrict__ losses) {
  __shared__ float sh[GL_THREADS / 32];
  const float nb = num_boxes(norm, world);
  for (int l = 0; l < L; ++l) {
    float t = 0.f, a = 0.f, g = 0.f;
    for (int i = threadIdx.x; i < ntok; i += GL_THREADS) t += tok_partial[(long)l * ntok + i];
    for (int i = threadIdx.x; i < nbox; i += GL_THREADS) {
      a += box_partial[((long)l * nbox + i) * 2];
      g += box_partial[((long)l * nbox + i) * 2 + 1];
    }
    t = block_sum(t, sh);
    a = block_sum(a, sh);
    g = block_sum(g, sh);
    if (threadIdx.x == 0) {
      losses[3 * l] = t / nb * w_ce;
      losses[3 * l + 1] = a / nb * w_bbox;
      losses[3 * l + 2] = g / nb * w_giou;
    }
  }
}

inline long gl_box_blocks(long rows) { return (rows + GL_THREADS - 1) / GL_THREADS; }
inline long gl_token_blocks(long rows) {
  const long warps = (rows + GL_THREADS / 32 - 1) / (GL_THREADS / 32);
  return warps < GL_TOKEN_BLOCKS ? warps : GL_TOKEN_BLOCKS;
}
inline size_t lsa_smem_bytes(long Q) { return (size_t)Q * (3 * sizeof(double) + 4 * sizeof(int) + 2); }

}  // namespace
}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_gdino_match_cost(const float* logits, const float* boxes, const float* gt_boxes, const int32_t* gt_count,
                                      const float* gt_tokens, int64_t L, int64_t B, int64_t Q, int64_t T, int64_t Gmax, float alpha,
                                      float cost_class, float cost_bbox, float cost_giou, float* cost, float* norm, void* stream) {
  MQ_REQUIRE(logits && boxes && gt_boxes && gt_count && gt_tokens && cost, "gdino_match_cost: null pointer");
  MQ_REQUIRE(L >= 1 && B >= 1 && L * B <= 65535, "gdino_match_cost: L*B=%ld out of range 1..65535", (long)(L * B));
  MQ_REQUIRE(Q >= 1 && Q <= (1l << 24), "gdino_match_cost: bad query count Q=%ld", (long)Q);
  MQ_REQUIRE(T >= 1 && T <= (1l << 20), "gdino_match_cost: bad token count T=%ld", (long)T);
  MQ_REQUIRE(Gmax >= 1 && Gmax <= Q, "gdino_match_cost: GT capacity Gmax=%ld must be in 1..Q=%ld", (long)Gmax, (long)Q);
  const dim3 grid((unsigned)((Q + GC_TQ - 1) / GC_TQ), (unsigned)((Gmax + GC_TG - 1) / GC_TG), (unsigned)(L * B));
  MQ_REQUIRE(grid.y <= 65535, "gdino_match_cost: Gmax=%ld too large", (long)Gmax);
  gdino_cost_kernel<<<grid, GC_THREADS, 0, (cudaStream_t)stream>>>(logits, boxes, gt_boxes, gt_count, gt_tokens, (int)B, (int)Q, (int)T,
                                                                  (int)Gmax, alpha, cost_class, cost_bbox, cost_giou, cost, norm);
  return check_launch("gdino_cost_kernel");
}

extern "C" int64_t mqdet_linear_sum_assignment_workspace_bytes(int64_t P, int64_t Q, int64_t Gmax) {
  if (P < 1 || Q < 1 || Gmax < 1) return 0;
  return P * Q * Gmax * (int64_t)sizeof(float);
}

extern "C" int mqdet_linear_sum_assignment(const float* cost, const int32_t* counts, int64_t ncounts, int64_t P, int64_t Q,
                                           int64_t Gmax, void* workspace, int32_t* match, void* stream) {
  MQ_REQUIRE(cost && counts && workspace && match, "linear_sum_assignment: null pointer");
  MQ_REQUIRE(P >= 1 && P <= (1l << 31) - 1 && ncounts >= 1, "linear_sum_assignment: bad problem count P=%ld / ncounts=%ld", (long)P,
             (long)ncounts);
  MQ_REQUIRE(Q >= 1 && Q <= LSA_MAX_Q, "linear_sum_assignment: Q=%ld out of range 1..%d", (long)Q, LSA_MAX_Q);
  MQ_REQUIRE(Gmax >= 1 && Gmax <= Q, "linear_sum_assignment: GT capacity Gmax=%ld must be in 1..Q=%ld", (long)Gmax, (long)Q);
  cudaStream_t st = (cudaStream_t)stream;
  float* cost_t = (float*)workspace;
  const dim3 tgrid((unsigned)((Q + 31) / 32), (unsigned)((Gmax + 31) / 32), (unsigned)P);
  MQ_REQUIRE(P <= 65535, "linear_sum_assignment: P=%ld problems per call at most 65535", (long)P);
  lsa_transpose_kernel<<<tgrid, dim3(32, 8), 0, st>>>(cost, (int)Q, (int)Gmax, cost_t);
  int rc = check_launch("lsa_transpose_kernel");
  if (rc) return rc;
  const size_t smem = lsa_smem_bytes(Q);
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(lsa_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return check_launch("linear_sum_assignment shared memory");
  lsa_kernel<<<(unsigned)P, 32, smem, st>>>(cost, cost_t, counts, (int)ncounts, (int)Q, (int)Gmax, match);
  return check_launch("lsa_kernel");
}

extern "C" int64_t mqdet_gdino_set_loss_workspace_floats(int64_t L, int64_t B, int64_t Q) {
  if (L < 1 || B < 1 || Q < 1) return 0;
  return L * gl_token_blocks(B * Q) + L * gl_box_blocks(B * Q) * 2;
}

extern "C" int mqdet_gdino_set_loss(const float* logits, const float* boxes, const int32_t* match, const float* gt_boxes,
                                    const float* gt_tokens, int64_t L, int64_t B, int64_t Q, int64_t T, int64_t Gmax,
                                    const float* text_mask, const float* norm, float world, float alpha, float gamma, float w_ce,
                                    float w_bbox, float w_giou, float* workspace, float* losses, float* d_logits, float* d_boxes,
                                    void* stream) {
  MQ_REQUIRE(logits && boxes && match && gt_boxes && gt_tokens && norm && workspace && losses && d_logits && d_boxes,
             "gdino_set_loss: null pointer");
  MQ_REQUIRE(L >= 1 && L <= 65535 && B >= 1, "gdino_set_loss: bad layer / image count L=%ld B=%ld", (long)L, (long)B);
  MQ_REQUIRE(Q >= 1 && B * Q <= (1l << 31) - 1, "gdino_set_loss: bad query count Q=%ld", (long)Q);
  MQ_REQUIRE(T >= 1 && T <= (1l << 20), "gdino_set_loss: bad token count T=%ld", (long)T);
  MQ_REQUIRE(Gmax >= 1 && Gmax <= Q, "gdino_set_loss: GT capacity Gmax=%ld must be in 1..Q=%ld", (long)Gmax, (long)Q);
  MQ_REQUIRE(world >= 1.f, "gdino_set_loss: world size %g < 1", (double)world);
  cudaStream_t st = (cudaStream_t)stream;
  const long rows = B * Q;
  const int ntok = (int)gl_token_blocks(rows), nbox = (int)gl_box_blocks(rows);
  float* tok_partial = workspace;
  float* box_partial = workspace + L * ntok;
  gdino_token_loss_kernel<<<dim3((unsigned)ntok, (unsigned)L), GL_THREADS, 0, st>>>(logits, match, gt_tokens, (int)Gmax, text_mask, (int)T,
                                                                                   (int)B, (int)Q, alpha, gamma, norm, world, w_ce,
                                                                                   tok_partial, d_logits);
  int rc = check_launch("gdino_token_loss_kernel");
  if (rc) return rc;
  gdino_box_loss_kernel<<<dim3((unsigned)nbox, (unsigned)L), GL_THREADS, 0, st>>>(boxes, match, gt_boxes, (int)Gmax, (int)B, (int)Q, norm,
                                                                                 world, w_bbox, w_giou, box_partial, d_boxes);
  rc = check_launch("gdino_box_loss_kernel");
  if (rc) return rc;
  gdino_loss_finalize_kernel<<<1, GL_THREADS, 0, st>>>(tok_partial, ntok, box_partial, nbox, (int)L, norm, world, w_ce, w_bbox, w_giou,
                                                       losses);
  return check_launch("gdino_loss_finalize_kernel");
}
