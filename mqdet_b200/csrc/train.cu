// mqdet_b200 — training-side kernels of the modulated pre-training step (SURVEY.md §8 f2, BASELINE config 5): the backward of the
// Gated Class-scalable Perceiver block (the only trainable blocks besides PreSelect: tools/train_net.py:70-77), the token focal loss
// and the optimizer step.  The matrix products of the backward (activation gradients dX = dY W, weight gradients dW = dY^T X) are
// mqdet_gemm_f16 launches; this file holds everything around them:
//   * transpose_cast        : [R][C] (f16 | f32) -> f16 [C][R] (zero padded to a multiple of 8) — the K-major operands of dW = dY^T X
//   * layernorm_bwd         : dx, dgamma, dbeta of nn.LayerNorm (mean / rstd recomputed from the saved input)
//   * gelu_bwd              : dz = dh * gelu'(z), exact erf GELU (modeling_bert_new.py:115-126)
//   * gcp_gate_bwd          : x1 = s * tanh(h1 . w2) + x (modeling_bert_new.py:355-361) -> ds, d(pre-tanh gate), dh1
//   * colsum_weighted       : out[j] = sum_r w[r] h[r][j] (the gradient of the 384 -> 1 gate projection)
//   * gcp_sparse_attn_bwd   : backward of the sparse masked cross-attention (gcp.cu forward; modeling_bert_new.py:215-240):
//                             dq per token, dK / dV scattered onto the UNIQUE query rows (fp32 atomics)
//   * dot_sum, scale_cast   : d(ff_gate) = (1 - tanh^2) sum(dy . u); du = tanh(ff_gate) dy
//   * token_focal_loss      : token_sigmoid_binary_focal_loss (layers/sigmoid_focal_loss.py:127-162) — loss sum and d(logits)
//   * sqnorm_partials, clip_coef, adamw_step : global-norm clipping (solver CLIP_GRADIENTS full_model, NORM_TYPE 2) + AdamW
//                             (solver/build.py:8-57) with the clip coefficient read from the device (no host synchronisation)
// All HBM-bound; reductions are two-stage and deterministic except the dK / dV scatter.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int RED_BLOCKS = 64;  // blocks (x 8 warps) of the two-stage row reductions

template <typename T>
__device__ __forceinline__ float ldf(const T* p);
template <>
__device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float ldf<__half>(const __half* p) { return __half2float(*p); }

// ---------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) transpose_cast_kernel(const T* __restrict__ x, int R, int C, long ld, long s1, long s2, int nb1,
                                                             float scale, __half* __restrict__ out, long ldo) {
  __shared__ float tile[32][33];
  const int z = blockIdx.z, z1 = z % nb1, z2 = z / nb1;
  x += (long)z1 * s1 + (long)z2 * s2;
  out += (long)z * C * ldo;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + tx;
    tile[j][tx] = (r < R && c < C) ? ldf<T>(x + (long)r * ld + c) * scale : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, r = r0 + tx;  // out[c][r]
    if (c < C && r < ldo) out[(long)c * ldo + r] = __float2half_rn(tile[tx][j]);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// LayerNorm backward, warp per row (grid-stride).  Per-warp partial dgamma / dbeta rows go to the workspace
// [2][nwarps][D]; ln_bwd_reduce sums them per column.
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                            const float* __restrict__ x2, const float* __restrict__ gamma, float eps,
                                                            long rows, int D,
                                                            float* __restrict__ dx, int accumulate, float* __restrict__ ws) {
  extern __shared__ float lnb_sh[];  // [8 warps][2][D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long nw = (long)gridDim.x * 8, gw = (long)blockIdx.x * 8 + warp;
  float* pg = lnb_sh + (long)warp * 2 * D;
  float* pb = pg + D;
  for (int i = lane; i < D; i += 32) pg[i] = pb[i] = 0.f;
  for (long r = gw; r < rows; r += nw) {
    const float* xr = x + r * D;
    const float* x2r = x2 ? x2 + r * D : nullptr;  // LN input = x + x2 (post-norm residual blocks store the two addends)
    const float* dr = dy + r * D;
    float s = 0.f;
    for (int i = lane; i < D; i += 32) s += xr[i] + (x2r ? x2r[i] : 0.f);
    const float mean = warp_sum(s) / D;
    float v = 0.f;
    for (int i = lane; i < D; i += 32) {
      const float d = xr[i] + (x2r ? x2r[i] : 0.f) - mean;
      v = fmaf(d, d, v);
    }
    const float rstd = rsqrtf(warp_sum(v) / D + eps);
    float sg = 0.f, sgx = 0.f;
    for (int i = lane; i < D; i += 32) {
      const float xh = (xr[i] + (x2r ? x2r[i] : 0.f) - mean) * rstd, g = dr[i] * gamma[i];
      sg += g;
      sgx = fmaf(g, xh, sgx);
      pg[i] = fmaf(dr[i], xh, pg[i]);
      pb[i] += dr[i];
    }
    sg = warp_sum(sg) / D;
    sgx = warp_sum(sgx) / D;
    for (int i = lane; i < D; i += 32) {
      const float xh = (xr[i] + (x2r ? x2r[i] : 0.f) - mean) * rstd, g = dr[i] * gamma[i];
      const float o = rstd * (g - sg - xh * sgx);
      dx[r * D + i] = accumulate ? dx[r * D + i] + o : o;
    }
  }
  float* wg = ws + gw * D;
  float* wb = ws + (nw + gw) * D;
  for (int i = lane; i < D; i += 32) {
    wg[i] = pg[i];
    wb[i] = pb[i];
  }
}

// out[j] = sum_p partial[p][j]; used for dgamma / dbeta (two calls) and colsum_weighted
__global__ void __launch_bounds__(256) colsum_partials_kernel(const float* __restrict__ partial, int np, int C, float* __restrict__ out) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= C) return;
  float s = 0.f;
  for (int p = 0; p < np; ++p) s += partial[(long)p * C + j];
  out[j] = s;
}

// ---------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) gelu_bwd_kernel(const __half* __restrict__ z, const T* __restrict__ dh, long n,
                                                       __half* __restrict__ dz) {
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long)gridDim.x * 256) {
    const float x = __half2float(z[i]);
    const float cdf = 0.5f * (1.f + erff(x * 0.7071067811865476f));
    const float pdf = 0.3989422804014327f * expf(-0.5f * x * x);
    dz[i] = __float2half_rn(ldf<T>(dh + i) * (cdf + x * pdf));
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// softmax backward, warp per row: ds[j] = scale * p[j] * (dp[j] - sum_k p[k] dp[k]); columns n..n_pad-1 are written as zero
__global__ void __launch_bounds__(256) softmax_bwd_rows_kernel(const __half* __restrict__ p, long ldp, const float* __restrict__ dp, long ldd,
                                                               long rows, int n, int n_pad, float scale, __half* __restrict__ ds, long lds) {
  const long r = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float dot = 0.f;
  for (int j = lane; j < n; j += 32) dot = fmaf(__half2float(p[r * ldp + j]), dp[r * ldd + j], dot);
  dot = warp_sum(dot);
  for (int j = lane; j < n_pad; j += 32)
    ds[r * lds + j] = __float2half_rn(j < n ? scale * __half2float(p[r * ldp + j]) * (dp[r * ldd + j] - dot) : 0.f);
}

// ---------------------------------------------------------------------------------------------------------------------
// warp per row: ds = dx1 * g; dgpre = (sum_d dx1 * s) (1 - g^2); dh1 = dgpre * w2
__global__ void __launch_bounds__(256) gcp_gate_bwd_kernel(const float* __restrict__ dx1, const float* __restrict__ s,
                                                           const float* __restrict__ g, const float* __restrict__ w2, long rows,
                                                           int D, int Dg, float* __restrict__ ds, float* __restrict__ dgpre,
                                                           __half* __restrict__ dh1) {
  const long r = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const float gv = g[r];
  float acc = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float d = dx1[r * D + i];
    acc = fmaf(d, s[r * D + i], acc);
    ds[r * D + i] = d * gv;
  }
  const float dgp = warp_sum(acc) * (1.f - gv * gv);
  if (lane == 0) dgpre[r] = dgp;
  for (int j = lane; j < Dg; j += 32) dh1[r * Dg + j] = __float2half_rn(dgp * w2[j]);
}

// partial[block][j] = sum over the block's rows of w[r] * h[r][j]
__global__ void __launch_bounds__(256) colsum_weighted_kernel(const __half* __restrict__ h, const float* __restrict__ w, long rows,
                                                              int C, float* __restrict__ partial) {
  const long per = (rows + gridDim.x - 1) / gridDim.x;
  const long r0 = (long)blockIdx.x * per, r1 = min(rows, r0 + per);
  for (int j = threadIdx.x; j < C; j += 256) {
    float s = 0.f;
    for (long r = r0; r < r1; ++r) s = fmaf(w[r], __half2float(h[r * C + j]), s);
    partial[(long)blockIdx.x * C + j] = s;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
constexpr int GCPB_MAX_S = 16;

__device__ __forceinline__ void ld16hf(const __half* p, float (&f)[16]) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const uint4 b = *reinterpret_cast<const uint4*>(p + 8);
  const __half2* ha = reinterpret_cast<const __half2*>(&a);
  const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 x = __half22float2(ha[i]), y = __half22float2(hb[i]);
    f[2 * i] = x.x; f[2 * i + 1] = x.y;
    f[8 + 2 * i] = y.x; f[8 + 2 * i + 1] = y.y;
  }
}

// Same work split as the forward (gcp.cu): one warp per token, lane = 16 contiguous dims, lanes_per_head lanes per head.
__global__ void __launch_bounds__(256) gcp_sparse_attn_bwd_kernel(const __half* __restrict__ q, const __half* __restrict__ kv,
                                                                  const int* __restrict__ idx, const __half* __restrict__ dout,
                                                                  __half* __restrict__ dq, float* __restrict__ dkv, long BT, int T,
                                                                  int V, int S, int lanes_per_head) {
  const long tok = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (tok >= BT) return;
  const int b = (int)(tok / T);
  const int inner = 512;
  const __half* kvb = kv + (long)b * (V + 1) * (2 * inner);
  float* dkvb = dkv + (long)b * (V + 1) * (2 * inner);
  float qf[16], gof[16];
  ld16hf(q + tok * inner + lane * 16, qf);
  ld16hf(dout + tok * inner + lane * 16, gof);
  float sim[GCPB_MAX_S], dp[GCPB_MAX_S];
  int id[GCPB_MAX_S];
#pragma unroll
  for (int s = 0; s < GCPB_MAX_S; ++s) {
    if (s < S) {
      id[s] = idx[tok * S + s];
      float kf[16], vf[16];
      ld16hf(kvb + (long)id[s] * (2 * inner) + lane * 16, kf);
      ld16hf(kvb + (long)id[s] * (2 * inner) + inner + lane * 16, vf);
      float d = 0.f, e = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        d = fmaf(qf[i], kf[i], d);
        e = fmaf(gof[i], vf[i], e);
      }
      for (int o = 1; o < lanes_per_head; o <<= 1) {
        d += __shfl_xor_sync(0xffffffffu, d, o);
        e += __shfl_xor_sync(0xffffffffu, e, o);
      }
      sim[s] = d + (id[s] == V ? -1e4f : 0.f);
      dp[s] = (id[s] == V) ? 0.f : e;  // p = softmax * mask: the gradient reaches the softmax only through unmasked slots
    }
  }
  float mx = -INFINITY;
#pragma unroll
  for (int s = 0; s < GCPB_MAX_S; ++s)
    if (s < S) mx = fmaxf(mx, sim[s]);
  float den = 0.f;
#pragma unroll
  for (int s = 0; s < GCPB_MAX_S; ++s)
    if (s < S) {
      sim[s] = expf(sim[s] - mx);
      den += sim[s];
    }
  const float inv = 1.f / den;
  float dot = 0.f;
#pragma unroll
  for (int s = 0; s < GCPB_MAX_S; ++s)
    if (s < S) {
      sim[s] *= inv;  // softmax probability (before the mask)
      dot = fmaf(sim[s], dp[s], dot);
    }
  float dqa[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) dqa[i] = 0.f;
#pragma unroll
  for (int s = 0; s < GCPB_MAX_S; ++s) {
    if (s < S) {
      const float dsim = sim[s] * (dp[s] - dot);
      const float p = (id[s] == V) ? 0.f : sim[s];
      float kf[16];
      ld16hf(kvb + (long)id[s] * (2 * inner) + lane * 16, kf);
      float* dk = dkvb + (long)id[s] * (2 * inner) + lane * 16;
      float* dv = dk + inner;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        dqa[i] = fmaf(dsim, kf[i], dqa[i]);
        atomicAdd(dk + i, dsim * qf[i]);
        atomicAdd(dv + i, p * gof[i]);
      }
    }
  }
  __half2 h[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) h[i] = __floats2half2_rn(dqa[2 * i], dqa[2 * i + 1]);
  uint4* dst = reinterpret_cast<uint4*>(dq + tok * inner + lane * 16);
  dst[0] = *reinterpret_cast<uint4*>(&h[0]);
  dst[1] = *reinterpret_cast<uint4*>(&h[4]);
}

// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum_256(float v, float* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = threadIdx.x < 8 ? sh[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) r = warp_sum(r);
  __syncthreads();
  return r;  // valid in warp 0
}

__global__ void __launch_bounds__(256) dot_partial_kernel(const float* __restrict__ a, const float* __restrict__ b, long n,
                                                          float* __restrict__ partial) {
  __shared__ float sh[8];
  float s = 0.f;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long)gridDim.x * 256) s = fmaf(a[i], b ? b[i] : a[i], s);
  s = block_sum_256(s, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// out[0] = mul * sum(partial); with one_minus_tanh2 != null: out[0] *= 1 - tanh(*one_minus_tanh2)^2
__global__ void __launch_bounds__(256) sum_partials_kernel(const float* __restrict__ partial, int np, const float* __restrict__ one_minus_tanh2,
                                                           float mul, float* __restrict__ out) {
  __shared__ float sh[8];
  float s = 0.f;
  for (int i = threadIdx.x; i < np; i += 256) s += partial[i];
  s = block_sum_256(s, sh);
  if (threadIdx.x == 0) {
    float m = mul;
    if (one_minus_tanh2) {
      const float t = tanhf(*one_minus_tanh2);
      m *= 1.f - t * t;
    }
    out[0] = s * m;
  }
}

__global__ void __launch_bounds__(256) scale_cast_kernel(const float* __restrict__ x, const float* __restrict__ scalar, int tanh_scalar,
                                                         float alpha, long n, __half* __restrict__ o16, float* __restrict__ o32) {
  float a = alpha;
  if (scalar) a *= tanh_scalar ? tanhf(*scalar) : *scalar;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long)gridDim.x * 256) {
    const float v = x[i] * a;
    if (o16) o16[i] = __float2half_rn(v);
    if (o32) o32[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// token_sigmoid_binary_focal_loss: elements of masked text tokens are dropped (masked_select); loss summed.
__global__ void __launch_bounds__(256) token_focal_loss_kernel(const float* __restrict__ logits, const float* __restrict__ targets,
                                                               const float* __restrict__ text_mask, float alpha, float gamma, long NT,
                                                               int T, long total, float grad_scale, float* __restrict__ partial,
                                                               float* __restrict__ dlogits) {
  __shared__ float sh[8];
  float acc = 0.f;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const long b = i / NT;
    const int t = (int)(i % T);
    float l = 0.f, d = 0.f;
    if (!text_mask || text_mask[b * T + t] > 0.f) token_focal_elem(logits[i], targets[i], alpha, gamma, l, d);
    acc += l;
    if (dlogits) dlogits[i] = d * grad_scale;
  }
  acc = block_sum_256(acc, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}

// ---------------------------------------------------------------------------------------------------------------------
// coef[0] = min(1, max_norm / (sqrt(sum partial) + 1e-6)) (torch.nn.utils.clip_grad_norm_), coef[1] = the norm
__global__ void __launch_bounds__(256) clip_coef_kernel(const float* __restrict__ partial, int np, float max_norm, float* __restrict__ coef) {
  __shared__ float sh[8];
  float s = 0.f;
  for (int i = threadIdx.x; i < np; i += 256) s += partial[i];
  s = block_sum_256(s, sh);
  if (threadIdx.x == 0) {
    const float norm = sqrtf(s);
    coef[1] = norm;
    coef[0] = max_norm > 0.f ? fminf(1.f, max_norm / (norm + 1e-6f)) : 1.f;
  }
}

__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                    float* __restrict__ v, long n, float lr, float b1, float b2, float eps, float wd,
                                                    float bc1, float bc2_sqrt, const float* __restrict__ grad_scale) {
  const float gs = grad_scale ? *grad_scale : 1.f;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long)gridDim.x * 256) {
    const float gr = g[i] * gs;
    float pv = p[i] * (1.f - lr * wd);
    const float mv = b1 * m[i] + (1.f - b1) * gr;
    const float vv = b2 * v[i] + (1.f - b2) * gr * gr;
    m[i] = mv;
    v[i] = vv;
    const float denom = sqrtf(vv) / bc2_sqrt + eps;
    pv -= (lr / bc1) * (mv / denom);
    p[i] = pv;
  }
}

static inline unsigned ew_blocks(long n) {
  long b = (n + 255) / 256;
  if (b > 132 * 8) b = 132 * 8;
  return (unsigned)(b < 1 ? 1 : b);
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_transpose_cast_batched(const void* x, int x_dtype, int64_t nb1, int64_t nb2, int64_t x_s1, int64_t x_s2, int64_t R,
                                            int64_t C, int64_t ld, float scale, void* out16, int64_t ldo, void* stream) {
  MQ_REQUIRE(x && out16 && R > 0 && C > 0 && ldo >= R && nb1 > 0 && nb2 > 0 && nb1 * nb2 <= 65535, "transpose_cast: bad arguments");
  const dim3 grid((unsigned)((C + 31) / 32), (unsigned)((ldo + 31) / 32), (unsigned)(nb1 * nb2));
  if (x_dtype == MQDET_F16)
    transpose_cast_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)x, (int)R, (int)C, ld, x_s1, x_s2, (int)nb1, scale,
                                                                          (__half*)out16, ldo);
  else
    transpose_cast_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)x, (int)R, (int)C, ld, x_s1, x_s2, (int)nb1, scale,
                                                                         (__half*)out16, ldo);
  return check_launch("transpose_cast_kernel");
}

extern "C" int mqdet_transpose_cast(const void* x, int x_dtype, int64_t R, int64_t C, int64_t ld, float scale, void* out16,
                                    int64_t ldo, void* stream) {
  MQ_REQUIRE(ld >= C, "transpose_cast: ld < C");
  return mqdet_transpose_cast_batched(x, x_dtype, 1, 1, 0, 0, R, C, ld, scale, out16, ldo, stream);
}

extern "C" int mqdet_softmax_bwd_rows(const void* p16, int64_t ldp, const float* dp, int64_t ldd, int64_t rows, int64_t n, int64_t n_pad,
                                      float scale, void* ds16, int64_t lds, void* stream) {
  MQ_REQUIRE(p16 && dp && ds16 && rows > 0 && n > 0 && n_pad >= n && ldp >= n && ldd >= n && lds >= n_pad, "softmax_bwd_rows: bad arguments");
  softmax_bwd_rows_kernel<<<cdiv(rows, 8), 256, 0, (cudaStream_t)stream>>>((const __half*)p16, ldp, dp, ldd, rows, (int)n, (int)n_pad, scale,
                                                                          (__half*)ds16, lds);
  return check_launch("softmax_bwd_rows_kernel");
}

extern "C" int64_t mqdet_layernorm_bwd_workspace_floats(int64_t rows, int64_t D) { return 2 * (int64_t)RED_BLOCKS * 8 * D; }

extern "C" int mqdet_layernorm_bwd(const float* dy, const float* x, const float* x2, const float* gamma, float eps, int64_t rows, int64_t D,
                                   float* dx, int accumulate, float* dgamma, float* dbeta, float* workspace, void* stream) {
  MQ_REQUIRE(dy && x && gamma && dx && workspace && rows > 0 && D > 0, "layernorm_bwd: bad arguments");
  MQ_REQUIRE(D <= 2048, "layernorm_bwd: D <= 2048");
  const size_t sh = (size_t)8 * 2 * D * sizeof(float);
  int rc = ensure_dyn_smem((const void*)layernorm_bwd_kernel, (int)sh);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  layernorm_bwd_kernel<<<RED_BLOCKS, 256, sh, st>>>(dy, x, x2, gamma, eps, rows, (int)D, dx, accumulate, workspace);
  const int nw = RED_BLOCKS * 8;
  if (dgamma) colsum_partials_kernel<<<cdiv(D, 256), 256, 0, st>>>(workspace, nw, (int)D, dgamma);
  if (dbeta) colsum_partials_kernel<<<cdiv(D, 256), 256, 0, st>>>(workspace + (long)nw * D, nw, (int)D, dbeta);
  return check_launch("layernorm_bwd");
}

extern "C" int mqdet_gelu_bwd(const void* z16, const void* dh, int dh_dtype, int64_t n, void* dz16, void* stream) {
  MQ_REQUIRE(z16 && dh && dz16 && n > 0, "gelu_bwd: bad arguments");
  if (dh_dtype == MQDET_F16)
    gelu_bwd_kernel<__half><<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>((const __half*)z16, (const __half*)dh, n, (__half*)dz16);
  else
    gelu_bwd_kernel<float><<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>((const __half*)z16, (const float*)dh, n, (__half*)dz16);
  return check_launch("gelu_bwd_kernel");
}

extern "C" int mqdet_gcp_gate_bwd(const float* dx1, const float* s, const float* g, const float* w2, int64_t rows, int64_t D, int64_t Dg,
                                  float* ds, float* dgpre, void* dh1_16, void* stream) {
  MQ_REQUIRE(dx1 && s && g && w2 && ds && dgpre && dh1_16 && rows > 0 && D > 0 && Dg > 0, "gcp_gate_bwd: bad arguments");
  gcp_gate_bwd_kernel<<<cdiv(rows, 8), 256, 0, (cudaStream_t)stream>>>(dx1, s, g, w2, rows, (int)D, (int)Dg, ds, dgpre, (__half*)dh1_16);
  return check_launch("gcp_gate_bwd_kernel");
}

extern "C" int64_t mqdet_colsum_weighted_workspace_floats(int64_t C) { return (int64_t)RED_BLOCKS * C; }

extern "C" int mqdet_colsum_weighted(const void* h16, const float* w, int64_t rows, int64_t C, float* out, float* workspace, void* stream) {
  MQ_REQUIRE(h16 && w && out && workspace && rows > 0 && C > 0, "colsum_weighted: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  colsum_weighted_kernel<<<RED_BLOCKS, 256, 0, st>>>((const __half*)h16, w, rows, (int)C, workspace);
  colsum_partials_kernel<<<cdiv(C, 256), 256, 0, st>>>(workspace, RED_BLOCKS, (int)C, out);
  return check_launch("colsum_weighted");
}

extern "C" int mqdet_gcp_sparse_attn_bwd(const void* q16, const void* kv16, const int32_t* idx, const void* dout16, int64_t B, int64_t T,
                                         int64_t V, int64_t S, int64_t H, int64_t Dh, void* dq16, float* dkv, void* stream) {
  MQ_REQUIRE(q16 && kv16 && idx && dout16 && dq16 && dkv, "gcp_sparse_attn_bwd: null pointer");
  MQ_REQUIRE(H * Dh == 512 && (Dh % 16) == 0, "gcp_sparse_attn_bwd: H*Dh must be 512");
  MQ_REQUIRE(S >= 1 && S <= GCPB_MAX_S, "gcp_sparse_attn_bwd: S out of range");
  const int lph = (int)(Dh / 16);
  MQ_REQUIRE((lph & (lph - 1)) == 0, "gcp_sparse_attn_bwd: Dh/16 must be a power of two");
  const long BT = B * T;
  gcp_sparse_attn_bwd_kernel<<<cdiv(BT, 8), 256, 0, (cudaStream_t)stream>>>((const __half*)q16, (const __half*)kv16, idx,
                                                                           (const __half*)dout16, (__half*)dq16, dkv, BT, (int)T,
                                                                           (int)V, (int)S, lph);
  return check_launch("gcp_sparse_attn_bwd_kernel");
}

extern "C" int64_t mqdet_reduce_workspace_floats(void) { return 1024; }

extern "C" int mqdet_dot_sum(const float* a, const float* b, int64_t n, const float* one_minus_tanh2_of, float mul, float* out,
                             float* workspace, void* stream) {
  MQ_REQUIRE(a && out && workspace && n > 0, "dot_sum: bad arguments");
  const unsigned nb = ew_blocks(n) > 1024 ? 1024 : ew_blocks(n);
  cudaStream_t st = (cudaStream_t)stream;
  dot_partial_kernel<<<nb, 256, 0, st>>>(a, b, n, workspace);
  sum_partials_kernel<<<1, 256, 0, st>>>(workspace, (int)nb, one_minus_tanh2_of, mul, out);
  return check_launch("dot_sum");
}

extern "C" int mqdet_scale_cast(const float* x, const float* scalar_dev, int tanh_scalar, float alpha, int64_t n, void* out16,
                                float* out32, void* stream) {
  MQ_REQUIRE(x && (out16 || out32) && n > 0, "scale_cast: bad arguments");
  scale_cast_kernel<<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>(x, scalar_dev, tanh_scalar, alpha, n, (__half*)out16, out32);
  return check_launch("scale_cast_kernel");
}

extern "C" int mqdet_token_focal_loss(const float* logits, const float* targets, const float* text_mask, float alpha, float gamma,
                                      int64_t B, int64_t N, int64_t T, float grad_scale, float* loss_out, float* dlogits,
                                      float* workspace, void* stream) {
  MQ_REQUIRE(logits && targets && loss_out && workspace && B > 0 && N > 0 && T > 0, "token_focal_loss: bad arguments");
  const long total = B * N * T;
  const unsigned nb = ew_blocks(total) > 1024 ? 1024 : ew_blocks(total);
  cudaStream_t st = (cudaStream_t)stream;
  token_focal_loss_kernel<<<nb, 256, 0, st>>>(logits, targets, text_mask, alpha, gamma, N * T, (int)T, total, grad_scale, workspace, dlogits);
  sum_partials_kernel<<<1, 256, 0, st>>>(workspace, (int)nb, nullptr, 1.f, loss_out);
  return check_launch("token_focal_loss");
}

extern "C" int mqdet_sqnorm_partials(const float* x, int64_t n, float* partial_out, int64_t max_partials, int64_t* partials_written,
                                     void* stream) {
  MQ_REQUIRE(x && partial_out && n > 0 && max_partials > 0, "sqnorm_partials: bad arguments");
  unsigned nb = ew_blocks(n);
  if (nb > 64) nb = 64;
  if ((int64_t)nb > max_partials) nb = (unsigned)max_partials;
  dot_partial_kernel<<<nb, 256, 0, (cudaStream_t)stream>>>(x, nullptr, n, partial_out);
  if (partials_written) *partials_written = nb;
  return check_launch("sqnorm_partials");
}

extern "C" int mqdet_clip_coef(const float* partials, int64_t count, float max_norm, float* coef2, void* stream) {
  MQ_REQUIRE(partials && coef2 && count > 0, "clip_coef: bad arguments");
  clip_coef_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(partials, (int)count, max_norm, coef2);
  return check_launch("clip_coef_kernel");
}

extern "C" int mqdet_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float beta1,
                                float beta2, float eps, float weight_decay, int64_t step, const float* grad_scale_dev, void* stream) {
  MQ_REQUIRE(param && grad && exp_avg && exp_avg_sq && n > 0 && step >= 1, "adamw_step: bad arguments");
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2s = sqrtf(1.f - powf(beta2, (float)step));
  adamw_kernel<<<ew_blocks(n), 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay,
                                                              bc1, bc2s, grad_scale_dev);
  return check_launch("adamw_kernel");
}
