// mqdet_b200 — row-wise HBM-bound kernels: LayerNorm, add+LayerNorm, masked softmax, casts.
// One warp per row, fp32 statistics, coalesced strided-by-lane accesses.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

template <typename T>
__device__ __forceinline__ float ld_as_float(const T* p);
template <>
__device__ __forceinline__ float ld_as_float<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float ld_as_float<__half>(const __half* p) { return __half2float(*p); }

// LayerNorm: nn.LayerNorm semantics (biased variance, eps inside the sqrt), modeling_bert_new.py:150-153.
template <typename T>
__global__ void __launch_bounds__(256) layernorm_kernel(const T* __restrict__ x, long ldx, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, long rows, int D,
                                                        __half* __restrict__ out16, float* __restrict__ out32, long ldo,
                                                        long zero_row_period) {
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const bool zero_row = zero_row_period > 0 && (row % zero_row_period) == zero_row_period - 1;
  const T* xr = x + row * ldx;
  float mean = 0.f, rstd;
  if (zero_row) {
    rstd = rsqrtf(eps);
  } else {
    float s = 0.f;
    for (int i = lane; i < D; i += 32) s += ld_as_float(xr + i);
    mean = warp_sum(s) / D;
    float v = 0.f;
    for (int i = lane; i < D; i += 32) {
      float d = ld_as_float(xr + i) - mean;
      v += d * d;
    }
    rstd = rsqrtf(warp_sum(v) / D + eps);
  }
  for (int i = lane; i < D; i += 32) {
    float xv = zero_row ? 0.f : ld_as_float(xr + i);
    float y = (xv - mean) * rstd * gamma[i] + beta[i];
    if (out16) out16[row * ldo + i] = __float2half_rn(y);
    if (out32) out32[row * ldo + i] = y;
  }
}

// Register-cached variants: the row is read ONCE.
//   layernorm_reg_kernel<T, K>: D == 32 * K, element i of lane l is x[l + 32 i] (every load/store covers contiguous bytes)
//   layernorm_h256_kernel     : fp16 rows of 256 (the fused visual stream): one 16-byte vector per lane
// Same arithmetic as layernorm_kernel (two-pass mean / biased variance in fp32).
template <typename T, int K>
__global__ void __launch_bounds__(256) layernorm_reg_kernel(const T* __restrict__ x, long ldx, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float eps, long rows,
                                                            __half* __restrict__ out16, float* __restrict__ out32, long ldo,
                                                            long zero_row_period) {
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  constexpr int D = 32 * K;
  const bool zero_row = zero_row_period > 0 && (row % zero_row_period) == zero_row_period - 1;
  const T* xr = x + row * ldx;
  float v[K];
#pragma unroll
  for (int i = 0; i < K; ++i) v[i] = zero_row ? 0.f : ld_as_float(xr + lane + 32 * i);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < K; ++i) s += v[i];
  const float mean = zero_row ? 0.f : warp_sum(s) / D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < K; ++i) {
    const float d = v[i] - mean;
    q += d * d;
  }
  const float rstd = zero_row ? rsqrtf(eps) : rsqrtf(warp_sum(q) / D + eps);
#pragma unroll
  for (int i = 0; i < K; ++i) {
    const int c = lane + 32 * i;
    const float y = (v[i] - mean) * rstd * gamma[c] + beta[c];
    if (out16) out16[row * ldo + c] = __float2half_rn(y);
    if (out32) out32[row * ldo + c] = y;
  }
}

// Narrow rows (Swin stages 1 / 2: D = 96 / 192 over 537600 / 134400 tokens): R consecutive rows per warp, all R*K loads issued
// before the first reduction, so a warp keeps R x 384 bytes in flight instead of 384 (the one-row kernel sits at ~30 % of
// the HBM rate on these shapes).  Same arithmetic per row as layernorm_reg_kernel.
template <typename T, int K, int R>
__global__ void __launch_bounds__(256) layernorm_reg_rows_kernel(const T* __restrict__ x, long ldx,
                                                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                 float eps, long rows, __half* __restrict__ out16,
                                                                 float* __restrict__ out32, long ldo, long zero_row_period) {
  const long row0 = ((long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * R;
  const int lane = threadIdx.x & 31;
  if (row0 >= rows) return;
  constexpr int D = 32 * K;
  float v[R][K];
  bool zr[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const long row = row0 + r;
    zr[r] = row >= rows || (zero_row_period > 0 && (row % zero_row_period) == zero_row_period - 1);
#pragma unroll
    for (int i = 0; i < K; ++i) v[r][i] = zr[r] ? 0.f : ld_as_float(x + row * ldx + lane + 32 * i);
  }
  float g[K], bt[K];
#pragma unroll
  for (int i = 0; i < K; ++i) {
    g[i] = gamma[lane + 32 * i];
    bt[i] = beta[lane + 32 * i];
  }
  float mean[R], rstd[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) s += v[r][i];
    mean[r] = s;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int r = 0; r < R; ++r) mean[r] += __shfl_xor_sync(0xffffffffu, mean[r], o);
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    mean[r] = zr[r] ? 0.f : mean[r] / D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {
      const float d = v[r][i] - mean[r];
      q += d * d;
    }
    rstd[r] = q;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int r = 0; r < R; ++r) rstd[r] += __shfl_xor_sync(0xffffffffu, rstd[r], o);
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const long row = row0 + r;
    if (row >= rows) break;
    const float rs = zr[r] ? rsqrtf(eps) : rsqrtf(rstd[r] / D + eps);
#pragma unroll
    for (int i = 0; i < K; ++i) {
      const int c = lane + 32 * i;
      const float y = (v[r][i] - mean[r]) * rs * g[i] + bt[i];
      if (out16) out16[row * ldo + c] = __float2half_rn(y);
      if (out32) out32[row * ldo + c] = y;
    }
  }
}

__global__ void __launch_bounds__(256) layernorm_h256_kernel(const __half* __restrict__ x, long ldx,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             float eps, long rows, __half* __restrict__ out16,
                                                             float* __restrict__ out32, long ldo, long zero_row_period) {
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const bool zero_row = zero_row_period > 0 && (row % zero_row_period) == zero_row_period - 1;
  float v[8];
  {
    const uint4 u = zero_row ? make_uint4(0, 0, 0, 0) : *reinterpret_cast<const uint4*>(x + row * ldx + lane * 8);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      v[2 * i] = f.x;
      v[2 * i + 1] = f.y;
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += v[i];
  const float mean = zero_row ? 0.f : warp_sum(s) * (1.f / 256.f);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float d = v[i] - mean;
    q += d * d;
  }
  const float rstd = zero_row ? rsqrtf(eps) : rsqrtf(warp_sum(q) * (1.f / 256.f) + eps);
  const float4 g0 = *reinterpret_cast<const float4*>(gamma + lane * 8), g1 = *reinterpret_cast<const float4*>(gamma + lane * 8 + 4);
  const float4 b0 = *reinterpret_cast<const float4*>(beta + lane * 8), b1 = *reinterpret_cast<const float4*>(beta + lane * 8 + 4);
  const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
  const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
  float y[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) y[i] = (v[i] - mean) * rstd * gg[i] + bb[i];
  if (out16) {
    __half2 o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = __floats2half2_rn(y[2 * i], y[2 * i + 1]);
    *reinterpret_cast<uint4*>(out16 + row * ldo + lane * 8) = *reinterpret_cast<uint4*>(o);
  }
  if (out32) {
    float4* d = reinterpret_cast<float4*>(out32 + row * ldo + lane * 8);
    d[0] = make_float4(y[0], y[1], y[2], y[3]);
    d[1] = make_float4(y[4], y[5], y[6], y[7]);
  }
}

// y = LN(a + b) (BertSelfOutput / BertOutput, rpn/modeling_bert.py:175-188,258-270), optional clamp of the sum and result.
__global__ void __launch_bounds__(256) add_layernorm_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                            const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float eps, long rows, int D,
                                                            float* __restrict__ out32, __half* __restrict__ out16,
                                                            float clampv) {
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* ar = a + row * D;
  const float* br = b + row * D;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) s += ar[i] + br[i];
  const float mean = warp_sum(s) / D;
  float v = 0.f;
  for (int i = lane; i < D; i += 32) {
    float d = ar[i] + br[i] - mean;
    v += d * d;
  }
  const float rstd = rsqrtf(warp_sum(v) / D + eps);
  for (int i = lane; i < D; i += 32) {
    float y = (ar[i] + br[i] - mean) * rstd * gamma[i] + beta[i];
    if (clampv > 0.f) y = fminf(fmaxf(y, -clampv), clampv);
    if (out32) out32[row * D + i] = y;
    if (out16) out16[row * D + i] = __float2half_rn(y);
  }
}

// Masked row softmax, warp per row. x fp32 -> y fp16. Columns [n, n_pad) are written as 0.
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ x, long ldx, __half* __restrict__ y, long ldy,
                                                           long rows, int n, int n_pad, float scale,
                                                           const float* __restrict__ colmask, long rows_per_batch,
                                                           float mask_value, float keep_add) {
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + row * ldx;
  __half* yr = y + row * ldy;
  const float* cm = colmask ? colmask + (row / rows_per_batch) * n : nullptr;
  float mx = -INFINITY;
  for (int i = lane; i < n; i += 32) {
    float v = xr[i] * scale;
    if (cm) v += (cm[i] == 0.f) ? mask_value : keep_add;
    mx = fmaxf(mx, v);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int i = lane; i < n; i += 32) {
    float v = xr[i] * scale;
    if (cm) v += (cm[i] == 0.f) ? mask_value : keep_add;
    sum += expf(v - mx);
  }
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
  for (int i = lane; i < n_pad; i += 32) {
    float o = 0.f;
    if (i < n) {
      float v = xr[i] * scale;
      if (cm) v += (cm[i] == 0.f) ? mask_value : keep_add;
      o = expf(v - mx) * inv;
    }
    yr[i] = __float2half_rn(o);
  }
}

// fp32 scores (the BERT self-attention products, [B*12*256, 256]): same single-read scheme with two float4 per lane.
template <int RW>
__global__ void __launch_bounds__(256) softmax_rows256_f32_kernel(const float* __restrict__ x, long ldx, __half* __restrict__ y,
                                                                  long ldy, long rows, float scale,
                                                                  const float* __restrict__ colmask, long rows_per_batch,
                                                                  float mask_value, float keep_add,
                                                                  const float* __restrict__ shift = nullptr, float lo = -INFINITY,
                                                                  float hi = INFINITY) {
  const int lane = threadIdx.x & 31;
  const long r0 = ((long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RW;
  if (r0 >= rows) return;
  constexpr float L2E = 1.4426950408889634f;
  float4 u[RW][2];
#pragma unroll
  for (int j = 0; j < RW; ++j) {
    if (r0 + j < rows) {
      const float4* src = reinterpret_cast<const float4*>(x + (r0 + j) * ldx + lane * 8);
      u[j][0] = src[0];
      u[j][1] = src[1];
    } else {
      u[j][0] = u[j][1] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
#pragma unroll
  for (int j = 0; j < RW; ++j) {
    const long row = r0 + j;
    if (row >= rows) break;
    float v[8] = {u[j][0].x * scale, u[j][0].y * scale, u[j][0].z * scale, u[j][0].w * scale,
                  u[j][1].x * scale, u[j][1].y * scale, u[j][1].z * scale, u[j][1].w * scale};
    if (shift) {  // STABLE_SOFTMAX_2D: v = clamp(v - global max, lo, hi) fused here instead of a pass of its own over the scores
      const float sh = __ldg(shift);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = fminf(fmaxf(v[i] - sh, lo), hi);
    }
    if (colmask) {
      const float* cm = colmask + (row / rows_per_batch) * 256 + lane * 8;
      const float4 m0 = *reinterpret_cast<const float4*>(cm);
      const float4 m1 = *reinterpret_cast<const float4*>(cm + 4);
      const float mm[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] += (mm[i] == 0.f) ? mask_value : keep_add;
    }
    float mx = v[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) mx = fmaxf(mx, v[i]);
    mx = warp_max(mx);
    const float ms = -mx * L2E;
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] = exp2f(fmaf(v[i], L2E, ms));
      sum += v[i];
    }
    const float inv = 1.f / warp_sum(sum);
    __half2 o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = __floats2half2_rn(v[2 * i] * inv, v[2 * i + 1] * inv);
    *reinterpret_cast<uint4*>(y + row * ldy + lane * 8) = *reinterpret_cast<uint4*>(o);
  }
}

// Long fp32 rows (the text -> image side of the explicit BiAttention path: n = 22323 image tokens per (image, head, text token)): one
// CTA per row instead of one warp, so a few thousand rows still fill the machine; three passes (max, sum, write) over a row that
// stays in L2 (89 KB), float4 loads where the row is 16-byte aligned.
__global__ void __launch_bounds__(256) softmax_longrows_f32_kernel(const float* __restrict__ x, long ldx, __half* __restrict__ y, long ldy,
                                                                   int n, int n_pad, float scale, const float* __restrict__ colmask,
                                                                   long rows_per_batch, float mask_value, float keep_add,
                                                                   const float* __restrict__ shift = nullptr, float lo = -INFINITY,
                                                                   float hi = INFINITY) {
  __shared__ float red[8];
  __shared__ float bcast;
  const long row = blockIdx.x;
  const float* xr = x + row * ldx;
  __half* yr = y + row * ldy;
  const float* cm = colmask ? colmask + (row / rows_per_batch) * n : nullptr;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float sh = shift ? __ldg(shift) : 0.f;
  auto val = [&](int i) {
    float v = xr[i] * scale;
    if (shift) v = fminf(fmaxf(v - sh, lo), hi);
    if (cm) v += (cm[i] == 0.f) ? mask_value : keep_add;
    return v;
  };
  float mx = -INFINITY;
  for (int i = tid; i < n; i += 256) mx = fmaxf(mx, val(i));
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  if (tid < 32) {
    float m = tid < 8 ? red[tid] : -INFINITY;
    m = warp_max(m);
    if (tid == 0) bcast = m;
  }
  __syncthreads();
  mx = bcast;
  __syncthreads();
  float sum = 0.f;
  for (int i = tid; i < n; i += 256) sum += expf(val(i) - mx);
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  if (tid < 32) {
    float t = tid < 8 ? red[tid] : 0.f;
    t = warp_sum(t);
    if (tid == 0) bcast = t;
  }
  __syncthreads();
  const float inv = 1.f / bcast;
  for (int i = tid; i < n_pad; i += 256) yr[i] = __float2half_rn(i < n ? expf(val(i) - mx) * inv : 0.f);
}

// out16[z2][z1][r][c] (strides o_s2, o_s1, ldo) = sum_s part[z2][z1][s][r][c]: the reduction of a split-K product whose K slices ran as an
// extra batch dimension of mqdet_gemm_f16 (fp32 partials).  One thread per 4 output columns.
__global__ void __launch_bounds__(256) sum_splits_cast_kernel(const float4* __restrict__ part, int S, int R, int C4, int nb1, long o_s1, long o_s2,
                                                              long ldo, long total, __half* __restrict__ out) {
  const long i = (long)blockIdx.x * 256 + threadIdx.x;
  if (i >= total) return;
  const int c4 = (int)(i % C4);
  const int r = (int)((i / C4) % R);
  const long z = i / ((long)C4 * R);
  const float4* p = part + (z * S * R + r) * C4 + c4;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s = 0; s < S; ++s) {
    const float4 v = p[(long)s * R * C4];
    a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
  }
  const long z1 = z % nb1, z2 = z / nb1;
  __half* o = out + z2 * o_s2 + z1 * o_s1 + (long)r * ldo + c4 * 4;
  const __half2 h0 = __floats2half2_rn(a.x, a.y), h1 = __floats2half2_rn(a.z, a.w);
  uint2 u;
  u.x = *reinterpret_cast<const uint32_t*>(&h0);
  u.y = *reinterpret_cast<const uint32_t*>(&h1);
  *reinterpret_cast<uint2*>(o) = u;
}

// ContrastiveEmbed tail (groundingdino_new/models/GroundingDINO/utils.py:261-266): columns of padding tokens and the
// columns T .. Tmax-1 of the [B, Q, Tmax] logits become -inf; the first T columns were written by the x . y^T product.
__global__ void contrastive_mask_kernel(float* __restrict__ logits, const uint8_t* __restrict__ text_token_mask, long rows,
                                        int Q, int T, int Tmax) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * Tmax) return;
  const int t = (int)(i % Tmax);
  const long b = (i / Tmax) / Q;
  if (t >= T || !text_token_mask[b * T + t]) logits[i] = -INFINITY;
}

__global__ void cast_f32_f16_kernel(const float* __restrict__ x, __half* __restrict__ y, long n) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long stride = (long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) y[i] = __float2half_rn(x[i]);
}
__global__ void cast_f16_f32_kernel(const __half* __restrict__ x, float* __restrict__ y, long n) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long stride = (long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) y[i] = __half2float(x[i]);
}

// e = x / max(||x||_2, eps) (F.normalize, vldyhead.py:810) and beta = e . w + b0 (:818).  One warp per row.
__global__ void __launch_bounds__(256) l2norm_rowdot_kernel(const float* __restrict__ x, long rows, int D, float eps,
                                                            const float* __restrict__ w, const float* __restrict__ b0,
                                                            __half* __restrict__ e16, float* __restrict__ e32,
                                                            float* __restrict__ dot) {
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + row * D;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) s += xr[i] * xr[i];
  const float inv = 1.f / fmaxf(sqrtf(warp_sum(s)), eps);
  float d = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float e = xr[i] * inv;
    if (e16) e16[row * D + i] = __float2half_rn(e);
    if (e32) e32[row * D + i] = e;
    if (w) d = fmaf(e, w[i], d);
  }
  if (dot) {
    d = warp_sum(d);
    if (lane == 0) dot[row] = d + (b0 ? b0[0] : 0.f);
  }
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_l2norm_rowdot(const float* x, int64_t rows, int64_t D, float eps, const float* w, const float* b0,
                                   void* e16, float* e32, float* dot, void* stream) {
  MQ_REQUIRE(x && rows > 0 && D > 0 && (e16 || e32 || dot), "l2norm_rowdot: bad args");
  const int wpb = 8;
  l2norm_rowdot_kernel<<<cdiv(rows, wpb), wpb * 32, 0, (cudaStream_t)stream>>>(x, rows, (int)D, eps, w, b0, (__half*)e16, e32,
                                                                             dot);
  return check_launch("l2norm_rowdot_kernel");
}

extern "C" int mqdet_layernorm(const void* x, int in_dtype, int64_t ldx, const float* gamma, const float* beta, float eps,
                               int64_t rows, int64_t D, void* out16, void* out32, int64_t ldo, int64_t zero_row_period,
                               void* stream) {
  MQ_REQUIRE(x && gamma && beta && (out16 || out32), "layernorm: null pointer");
  MQ_REQUIRE(rows > 0 && D > 0, "layernorm: empty");
  cudaStream_t st = (cudaStream_t)stream;
  const int wpb = 8;
  dim3 grid(cdiv(rows, wpb));
  const bool al16 = ((uintptr_t)x % 16) == 0 && (ldx % 8) == 0 && (ldo % 8) == 0 && (!out16 || ((uintptr_t)out16 % 16) == 0) &&
                    (!out32 || ((uintptr_t)out32 % 16) == 0) && ((uintptr_t)gamma % 16) == 0 && ((uintptr_t)beta % 16) == 0;
  if (in_dtype == MQDET_F16 && D == 256 && al16) {
    layernorm_h256_kernel<<<grid, wpb * 32, 0, st>>>((const __half*)x, ldx, gamma, beta, eps, rows, (__half*)out16, (float*)out32,
                                                    ldo, zero_row_period);
    return check_launch("layernorm_h256_kernel");
  }
#define MQ_LN_REG(TT, KK)                                                                                                   \
  layernorm_reg_kernel<TT, KK><<<grid, wpb * 32, 0, st>>>((const TT*)x, ldx, gamma, beta, eps, rows, (__half*)out16,        \
                                                          (float*)out32, ldo, zero_row_period)
  if ((D == 96 || D == 192) && rows >= 4096) {  // narrow rows: several rows per warp (see layernorm_reg_rows_kernel)
#define MQ_LN_ROWS(TT, KK, RR)                                                                                               \
  layernorm_reg_rows_kernel<TT, KK, RR><<<cdiv(rows, wpb * RR), wpb * 32, 0, st>>>(                                         \
      (const TT*)x, ldx, gamma, beta, eps, rows, (__half*)out16, (float*)out32, ldo, zero_row_period)
    if (in_dtype == MQDET_F32) {
      if (D == 96) MQ_LN_ROWS(float, 3, 4);
      else MQ_LN_ROWS(float, 6, 2);
    } else {
      if (D == 96) MQ_LN_ROWS(__half, 3, 4);
      else MQ_LN_ROWS(__half, 6, 2);
    }
#undef MQ_LN_ROWS
    return check_launch("layernorm_reg_rows_kernel");
  }
  if ((D % 32) == 0 && D / 32 <= 24) {
    const int k = (int)(D / 32);
    bool done = true;
    if (in_dtype == MQDET_F32) {
      switch (k) {
        case 3: MQ_LN_REG(float, 3); break;
        case 6: MQ_LN_REG(float, 6); break;
        case 8: MQ_LN_REG(float, 8); break;
        case 12: MQ_LN_REG(float, 12); break;
        case 24: MQ_LN_REG(float, 24); break;
        default: done = false;
      }
    } else {
      switch (k) {
        case 3: MQ_LN_REG(__half, 3); break;
        case 6: MQ_LN_REG(__half, 6); break;
        case 8: MQ_LN_REG(__half, 8); break;
        case 12: MQ_LN_REG(__half, 12); break;
        case 24: MQ_LN_REG(__half, 24); break;
        default: done = false;
      }
    }
    if (done) return check_launch("layernorm_reg_kernel");
  }
#undef MQ_LN_REG
  if (in_dtype == MQDET_F32)
    layernorm_kernel<float><<<grid, wpb * 32, 0, st>>>((const float*)x, ldx, gamma, beta, eps, rows, (int)D,
                                                      (__half*)out16, (float*)out32, ldo, zero_row_period);
  else
    layernorm_kernel<__half><<<grid, wpb * 32, 0, st>>>((const __half*)x, ldx, gamma, beta, eps, rows, (int)D,
                                                       (__half*)out16, (float*)out32, ldo, zero_row_period);
  return check_launch("layernorm_kernel");
}

extern "C" int mqdet_add_layernorm(const float* a, const float* b, const float* gamma, const float* beta, float eps,
                                   int64_t rows, int64_t D, float* out32, void* out16, float clampv, void* stream) {
  MQ_REQUIRE(a && b && gamma && beta && (out16 || out32), "add_layernorm: null pointer");
  const int wpb = 8;
  add_layernorm_kernel<<<cdiv(rows, wpb), wpb * 32, 0, (cudaStream_t)stream>>>(a, b, gamma, beta, eps, rows, (int)D, out32,
                                                                             (__half*)out16, clampv);
  return check_launch("add_layernorm_kernel");
}

extern "C" int mqdet_softmax_rows(const void* x, int in_dtype, int64_t ldx, void* y, int64_t ldy, int64_t rows, int64_t n,
                                  int64_t n_pad, float scale, const float* colmask, int64_t rows_per_batch,
                                  float mask_value, float keep_add, void* stream) {
  MQ_REQUIRE(x && y && rows > 0 && n > 0 && n_pad >= n, "softmax_rows: bad args");
  MQ_REQUIRE(in_dtype == MQDET_F32, "softmax_rows: fp32 scores required (in_dtype %d)", in_dtype);
  if (rows_per_batch <= 0) rows_per_batch = rows;
  const int wpb = 8;
  cudaStream_t st = (cudaStream_t)stream;
  const float* xf = (const float*)x;
  if (n == 256 && n_pad == 256 && (ldx % 4) == 0 && (ldy % 8) == 0 && ((uintptr_t)x % 16) == 0 && ((uintptr_t)y % 16) == 0 &&
      (!colmask || ((uintptr_t)colmask % 16) == 0)) {
    constexpr int RW = 2;
    softmax_rows256_f32_kernel<RW><<<(unsigned)cdiv(rows, (long)wpb * RW), wpb * 32, 0, st>>>(
        xf, ldx, (__half*)y, ldy, rows, scale, colmask, rows_per_batch, mask_value, keep_add);
    return check_launch("softmax_rows256_f32_kernel");
  }
  if (n >= 4096 && rows <= 0x7fffffffL) {
    softmax_longrows_f32_kernel<<<(unsigned)rows, 256, 0, st>>>(xf, ldx, (__half*)y, ldy, (int)n, (int)n_pad, scale, colmask,
                                                                rows_per_batch, mask_value, keep_add);
    return check_launch("softmax_longrows_f32_kernel");
  }
  softmax_rows_kernel<<<cdiv(rows, wpb), wpb * 32, 0, st>>>(xf, ldx, (__half*)y, ldy, rows, (int)n, (int)n_pad, scale, colmask,
                                                           rows_per_batch, mask_value, keep_add);
  return check_launch("softmax_rows_kernel");
}

extern "C" int mqdet_softmax_rows_shifted_supported(int64_t n, int64_t n_pad) { return (n == 256 && n_pad == 256) || n >= 4096; }

extern "C" int mqdet_softmax_rows_shifted(const float* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int64_t n, int64_t n_pad,
                                          const float* shift_dev, float lo, float hi, const float* colmask, int64_t rows_per_batch,
                                          float mask_value, float keep_add, void* stream) {
  MQ_REQUIRE(x && y && shift_dev && rows > 0 && n > 0 && n_pad >= n, "softmax_rows_shifted: bad args");
  MQ_REQUIRE(mqdet_softmax_rows_shifted_supported(n, n_pad), "softmax_rows_shifted: n == n_pad == 256 or n >= 4096 only");
  if (rows_per_batch <= 0) rows_per_batch = rows;
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 256) {
    MQ_REQUIRE((ldx % 4) == 0 && (ldy % 8) == 0 && ((uintptr_t)x % 16) == 0 && ((uintptr_t)y % 16) == 0 &&
                   (!colmask || ((uintptr_t)colmask % 16) == 0), "softmax_rows_shifted: 16-byte aligned rows required for n = 256");
    constexpr int RW = 2;
    softmax_rows256_f32_kernel<RW><<<(unsigned)cdiv(rows, 8L * RW), 256, 0, st>>>(x, ldx, (__half*)y, ldy, rows, 1.f, colmask,
                                                                                  rows_per_batch, mask_value, keep_add, shift_dev, lo, hi);
    return check_launch("softmax_rows256_f32_kernel");
  }
  MQ_REQUIRE(rows <= 0x7fffffffL, "softmax_rows_shifted: too many rows");
  softmax_longrows_f32_kernel<<<(unsigned)rows, 256, 0, st>>>(x, ldx, (__half*)y, ldy, (int)n, (int)n_pad, 1.f, colmask, rows_per_batch,
                                                              mask_value, keep_add, shift_dev, lo, hi);
  return check_launch("softmax_longrows_f32_kernel");
}

extern "C" int mqdet_sum_splits_cast(const float* part, int64_t nb2, int64_t nb1, int64_t S, int64_t R, int64_t C, void* out16, int64_t o_s2,
                                     int64_t o_s1, int64_t ldo, void* stream) {
  MQ_REQUIRE(part && out16 && nb1 > 0 && nb2 > 0 && S > 0 && R > 0 && C > 0 && (C % 4) == 0, "sum_splits_cast: bad args (C %% 4 == 0)");
  MQ_REQUIRE(((uintptr_t)part & 15) == 0 && ((uintptr_t)out16 & 7) == 0 && (ldo % 4) == 0 && (o_s1 % 4) == 0 && (o_s2 % 4) == 0,
             "sum_splits_cast: 16-byte aligned partials, 8-byte aligned output rows required");
  const long total = nb1 * nb2 * R * (C / 4);
  sum_splits_cast_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const float4*)part, (int)S, (int)R, (int)(C / 4),
                                                                                          (int)nb1, o_s1, o_s2, ldo, total, (__half*)out16);
  return check_launch("sum_splits_cast_kernel");
}

extern "C" int mqdet_cast_f32_f16(const float* x, void* y, int64_t n, void* stream) {
  MQ_REQUIRE(x && y && n > 0, "cast: bad args");
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  cast_f32_f16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, (__half*)y, n);
  return check_launch("cast_f32_f16_kernel");
}
extern "C" int mqdet_contrastive_mask(float* logits, const uint8_t* text_token_mask, int64_t B, int64_t Q, int64_t T,
                                      int64_t Tmax, void* stream) {
  MQ_REQUIRE(logits && text_token_mask && B > 0 && Q > 0 && T > 0 && Tmax >= T, "contrastive_mask: bad args");
  const long n = B * Q * Tmax;
  contrastive_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(logits, text_token_mask, B * Q, (int)Q,
                                                                                       (int)T, (int)Tmax);
  return check_launch("contrastive_mask");
}

extern "C" int mqdet_cast_f16_f32(const void* x, float* y, int64_t n, void* stream) {
  MQ_REQUIRE(x && y && n > 0, "cast: bad args");
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  cast_f16_f32_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __half*)x, y, n);
  return check_launch("cast_f16_f32_kernel");
}
