// mqdet_b200 — small device ops of the GroundingDINO variant (SURVEY.md §8 f1) next to ms_deform_attn (msda.cu):
//   * STABLE_SOFTMAX_2D of BiMultiHeadAttention (groundingdino_new/models/GroundingDINO/fuse_modules.py:177-187): the GLOBAL
//     maximum of the score tensor (of each batch element's, when prompt chunks share a batch) is subtracted before the +-5e4
//     clamps                                                                            -> global_max + shift_clamp
//   * two-stage query selection (transformer.py:288-318): max over the text tokens of the encoder class logits, top-900
//     proposals per image, gathers of the selected rows                                -> row_max, topk_desc, gather_rows
// All HBM-bound single-pass kernels; no host synchronisation.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int GMAX_BLOCKS = 1024;

__device__ __forceinline__ float block_max_256(float m, float* sh) {
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
  __syncthreads();
  float r = threadIdx.x < 8 ? sh[threadIdx.x] : -INFINITY;
  if (threadIdx.x < 32) r = warp_max(r);
  return r;  // valid in warp 0
}

// Segment s = x[s * seg_len, (s + 1) * seg_len): blockIdx.y = segment, gridDim.x blocks per segment -> partial[s][blockIdx.x].
// float4 loads where the segment starts 16-byte aligned (always for one segment, or seg_len % 4 == 0), scalar loads otherwise.
__global__ void __launch_bounds__(256) global_max_partial_kernel(const float* __restrict__ x, long seg_len, float* __restrict__ partial) {
  __shared__ float sh[8];
  float m = -INFINITY;
  const long s = blockIdx.y;
  const float* xs = x + s * seg_len;
  const long stride = (long)gridDim.x * 256;
  if (((s * seg_len) & 3) == 0) {
    const long n4 = seg_len >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(xs);
    for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n4; i += stride) {
      const float4 v = __ldg(x4 + i);
      m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
    }
    if (blockIdx.x == 0)
      for (long i = (n4 << 2) + threadIdx.x; i < seg_len; i += 256) m = fmaxf(m, xs[i]);
  } else {
    for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < seg_len; i += stride) m = fmaxf(m, __ldg(xs + i));
  }
  m = block_max_256(m, sh);
  if (threadIdx.x == 0) partial[s * gridDim.x + blockIdx.x] = m;
}

// out[s] = max of partial[s][0 .. np): one CTA per segment
__global__ void __launch_bounds__(256) global_max_final_kernel(const float* __restrict__ partial, int np, float* __restrict__ out) {
  __shared__ float sh[8];
  float m = -INFINITY;
  const float* p = partial + (long)blockIdx.x * np;
  for (int i = threadIdx.x; i < np; i += 256) m = fmaxf(m, p[i]);
  m = block_max_256(m, sh);
  if (threadIdx.x == 0) out[blockIdx.x] = m;
}

// x[i] = clamp(x[i] - shift[i / per_shift], lo, hi); per_shift = 0: shift[0] everywhere
__global__ void __launch_bounds__(256) shift_clamp_kernel(float* __restrict__ x, long n, const float* __restrict__ shift, long per_shift,
                                                          float lo, float hi) {
  const float s = __ldg(shift);
  auto sh = [&](long i) { return per_shift ? __ldg(shift + i / per_shift) : s; };
  const long n4 = n >> 2;
  float4* x4 = reinterpret_cast<float4*>(x);
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long)gridDim.x * 256) {
    float4 v = x4[i];
    v.x = fminf(fmaxf(v.x - sh(4 * i), lo), hi);
    v.y = fminf(fmaxf(v.y - sh(4 * i + 1), lo), hi);
    v.z = fminf(fmaxf(v.z - sh(4 * i + 2), lo), hi);
    v.w = fminf(fmaxf(v.w - sh(4 * i + 3), lo), hi);
    x4[i] = v;
  }
  if (blockIdx.x == 0)
    for (long i = (n4 << 2) + threadIdx.x; i < n; i += 256) x[i] = fminf(fmaxf(x[i] - sh(i), lo), hi);
}

// out[r] = max_j x[r][j], warp per row
__global__ void __launch_bounds__(256) row_max_kernel(const float* __restrict__ x, long rows, int D, long ld, float* __restrict__ out) {
  const long r = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int j = lane; j < D; j += 32) m = fmaxf(m, __ldg(x + r * ld + j));
  m = warp_max(m);
  if (lane == 0) out[r] = m;
}

// dst[b][i][:] = act(src[b][idx[b][i]][:]), warp per (b, i); act = identity or sigmoid
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ src, const long long* __restrict__ idx, long total,
                                                          long rows_src, long k, int D, int sigmoid, float* __restrict__ dst) {
  const long w = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (w >= total) return;
  const int lane = threadIdx.x & 31;
  const long b = w / k;
  const float* s = src + (b * rows_src + idx[w]) * D;
  float* d = dst + w * D;
  for (int j = lane; j < D; j += 32) {
    const float v = __ldg(s + j);
    d[j] = sigmoid ? 1.f / (1.f + expf(-v)) : v;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Top-k (k <= 1024) of n fp32 keys per image, result sorted by (value descending, index ascending): one CTA per image.
//   1. radix select (4 x 8 bits on the order-preserving integer image of the float) -> the k-th largest key T
//   2. every element > T, plus the lowest-index elements == T that fill up to k (an ordered block scan), into shared memory
//   3. bitonic sort of the <= 1024 collected (key, index) pairs
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ordered_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(1024) topk_desc_kernel(const float* __restrict__ keys, int n, int k, long long* __restrict__ out) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long sel[1024];  // (ordered key << 32) | (0xffffffff - index): descending sort of this = wanted order
  __shared__ unsigned int s_prefix, s_remaining, s_count, s_base;
  __shared__ unsigned int wsum[32];
  const float* x = keys + (long)blockIdx.x * n;
  const int tid = threadIdx.x;
  if (tid == 0) {
    s_prefix = 0;
    s_remaining = (unsigned)k;
  }
  __syncthreads();
  // -- 1. radix select, most significant byte first
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    const unsigned int prefix = s_prefix;
    const unsigned int pmask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    for (int i = tid; i < n; i += 1024) {
      const uint32_t u = ordered_key(x[i]);
      if ((u & pmask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      unsigned int rem = s_remaining;
      int b = 255;
      for (; b > 0; --b) {
        if (hist[b] >= rem) break;
        rem -= hist[b];
      }
      s_prefix = prefix | ((unsigned)b << shift);
      s_remaining = rem;  // how many elements of bin b (with this prefix) are still wanted
    }
    __syncthreads();
  }
  const uint32_t T = s_prefix;           // the k-th largest ordered key
  const unsigned int need_eq = s_remaining;  // elements == T to take (lowest indices first)
  if (tid == 0) {
    s_count = 0;
    s_base = 0;
  }
  __syncthreads();
  // -- 2. collect
  for (int i0 = 0; i0 < n; i0 += 1024) {
    const int i = i0 + tid;
    const uint32_t u = i < n ? ordered_key(x[i]) : 0u;
    const bool gt = i < n && u > T, eq = i < n && u == T;
    if (gt) sel[atomicAdd(&s_count, 1u)] = ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
    // ordered scan of the == T flags
    const unsigned int bal = __ballot_sync(0xffffffffu, eq);
    const int lane = tid & 31, w = tid >> 5;
    if (lane == 0) wsum[w] = __popc(bal);
    __syncthreads();
    unsigned int before = s_base;
    for (int j = 0; j < w; ++j) before += wsum[j];
    before += __popc(bal & ((1u << lane) - 1u));
    if (eq && before < need_eq) sel[atomicAdd(&s_count, 1u)] = ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
    __syncthreads();
    if (tid == 0) {
      unsigned int t = 0;
      for (int j = 0; j < 32; ++j) t += wsum[j];
      s_base += t;
    }
    __syncthreads();
  }
  const int cnt = (int)s_count;  // == min(k, n)
  if (tid >= cnt) sel[tid] = 0ull;
  __syncthreads();
  // -- 3. bitonic sort, descending
  for (int size = 2; size <= 1024; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const int j = tid ^ stride;
      if (j > tid) {
        const unsigned long long a = sel[tid], b = sel[j];
        const bool desc = (tid & size) == 0;
        if (desc ? a < b : a > b) {
          sel[tid] = b;
          sel[j] = a;
        }
      }
      __syncthreads();
    }
  }
  if (tid < k) out[(long)blockIdx.x * k + tid] = tid < cnt ? (long long)(0xffffffffu - (unsigned)(sel[tid] & 0xffffffffull)) : -1ll;
}

}  // namespace mqdet

using namespace mqdet;

// blocks per segment: GMAX_BLOCKS shared by the segments (at least one each), no more than the segment has float4 groups of 256
static long gmax_blocks_per_segment(long seg_len, long segments) {
  long cap = GMAX_BLOCKS / segments;
  if (cap < 1) cap = 1;
  long need = (seg_len / 4 + 255) / 256;
  if (need < 1) need = 1;
  return need < cap ? need : cap;
}

extern "C" int mqdet_global_max_f32(const float* x, int64_t n, int64_t segments, float* out, float* workspace, void* stream) {
  MQ_REQUIRE(x && out && workspace && n > 0, "global_max: null pointer / empty");
  MQ_REQUIRE(segments >= 1 && segments <= 65535 && (n % segments) == 0, "global_max: %ld elements do not split into %ld equal segments (1..65535)",
             (long)n, (long)segments);
  MQ_REQUIRE(((uintptr_t)x & 15) == 0, "global_max: x must be 16-byte aligned");
  const long seg_len = n / segments;
  const long blocks = gmax_blocks_per_segment(seg_len, segments);
  global_max_partial_kernel<<<dim3((unsigned)blocks, (unsigned)segments), 256, 0, (cudaStream_t)stream>>>(x, seg_len, workspace);
  global_max_final_kernel<<<(unsigned)segments, 256, 0, (cudaStream_t)stream>>>(workspace, (int)blocks, out);
  return check_launch("global_max");
}

extern "C" int64_t mqdet_global_max_workspace_floats(int64_t segments) {
  return segments < 1 ? 0 : segments * (GMAX_BLOCKS / segments > 0 ? GMAX_BLOCKS / segments : 1);
}

extern "C" int mqdet_shift_clamp_f32(float* x, int64_t n, const float* shift, int64_t elems_per_shift, float lo, float hi, void* stream) {
  MQ_REQUIRE(x && shift && n > 0 && elems_per_shift >= 0, "shift_clamp: null pointer / empty");
  MQ_REQUIRE(((uintptr_t)x & 15) == 0, "shift_clamp: x must be 16-byte aligned");
  const long blocks = (n / 4 + 255) / 256;
  shift_clamp_kernel<<<(unsigned)(blocks < 1 ? 1 : (blocks > 132 * 16 ? 132 * 16 : blocks)), 256, 0, (cudaStream_t)stream>>>(
      x, n, shift, elems_per_shift, lo, hi);
  return check_launch("shift_clamp_kernel");
}

extern "C" int mqdet_row_max_f32(const float* x, int64_t rows, int64_t D, int64_t ld, float* out, void* stream) {
  MQ_REQUIRE(x && out && rows > 0 && D > 0 && ld >= D, "row_max: bad arguments");
  row_max_kernel<<<cdiv(rows, 8), 256, 0, (cudaStream_t)stream>>>(x, rows, (int)D, ld, out);
  return check_launch("row_max_kernel");
}

extern "C" int mqdet_gather_rows_f32(const float* src, const int64_t* idx, int64_t B, int64_t rows_src, int64_t k, int64_t D,
                                     int sigmoid, float* dst, void* stream) {
  MQ_REQUIRE(src && idx && dst && B > 0 && rows_src > 0 && k > 0 && D > 0, "gather_rows: bad arguments");
  gather_rows_kernel<<<cdiv(B * k, 8), 256, 0, (cudaStream_t)stream>>>(src, (const long long*)idx, B * k, rows_src, k, (int)D, sigmoid, dst);
  return check_launch("gather_rows_kernel");
}

extern "C" int mqdet_topk_desc(const float* keys, int64_t B, int64_t n, int64_t k, int64_t* idx_out, void* stream) {
  MQ_REQUIRE(keys && idx_out, "topk_desc: null pointer");
  MQ_REQUIRE(B >= 1 && n >= 1 && k >= 1 && k <= 1024 && k <= n && n < (1L << 31), "topk_desc: need B >= 1 and 1 <= k <= min(n, 1024) (got B=%ld n=%ld k=%ld)",
             (long)B, (long)n, (long)k);
  topk_desc_kernel<<<(unsigned)B, 1024, 0, (cudaStream_t)stream>>>(keys, (int)n, (int)k, (long long*)idx_out);
  return check_launch("topk_desc_kernel");
}
