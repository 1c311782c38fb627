// mqdet_b200 — Gated Class-scalable Perceiver (GCP) kernels.
//
// Reference: maskrcnn_benchmark/modeling/language_backbone/modeling_bert_new.py
//   get_index_with_padding_batch :40-63, _construct_sparse_inputs :162-184,
//   MaskedCrossAttention.forward (sparse) :186-248, GatedCrossAttentionBlock.forward :347-374.
//
// The reference gathers the <=S vision queries of every text token and re-projects them to K/V per
// token (B*T*S rows).  K/V only depend on the unique query, so here they are projected ONCE for the
// V+1 rows (row V = the zero padding slot pushed through norm_kv) and the attention kernel gathers the
// projected rows: one warp per token, 8 heads x 64 dims = 16 contiguous dims per lane, 4 lanes per head,
// warp-shuffle reductions for q.k.  A token's S indices and H x S scores live in a warp-private slice of
// dynamic shared memory, so S (NUM_QUERY_PER_CLASS, summed over the classes a token belongs to) is open-ended
// up to GCP_MAX_S.
#include <algorithm>

#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

// Largest S whose one-warp slice, S x (H + 1) words, fits the 227 KB of opt-in shared memory of an sm_90 CTA for every
// supported head split (H <= 32).  Keep ops.GCP_MAX_S equal.
constexpr int GCP_MAX_S = 1760;
constexpr int GCP_SMEM_MAX = 227 * 1024;
constexpr int GCP_CHUNK = 16;  // slots whose K (or V) row loads are issued together
constexpr long gcp_slice_bytes(long S, long H) { return S * (H + 1) * 4; }
static_assert(gcp_slice_bytes(GCP_MAX_S, 32) <= GCP_SMEM_MAX, "GCP_MAX_S slice exceeds the shared-memory limit");

__device__ __forceinline__ void ld16h(const __half* p, float (&f)[16]) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const uint4 b = *reinterpret_cast<const uint4*>(p + 8);
  const __half2* ha = reinterpret_cast<const __half2*>(&a);
  const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 x = __half22float2(ha[i]);
    float2 y = __half22float2(hb[i]);
    f[2 * i] = x.x; f[2 * i + 1] = x.y;
    f[8 + 2 * i] = y.x; f[8 + 2 * i + 1] = y.y;
  }
}

// Generic in heads/dim as long as H*Dh == 32 * 16 (8x64 GCP) -- lanes_per_head = Dh/16, H = 32 / lanes_per_head.
// Per token: sim = q.k (+ -1e4 on padding slots), max, e = exp(sim - max) and den summed in slot order, p = e / den (0 on
// padding slots), sum p.v in slot order.  Every lane of a head holds the same score; the slice keeps one copy per head.
__global__ void __launch_bounds__(256) gcp_sparse_attn_kernel(const __half* __restrict__ q, const __half* __restrict__ kv,
                                                              const int* __restrict__ idx, __half* __restrict__ out,
                                                              long BT, int T, int V, int S, int lanes_per_head) {
  extern __shared__ float gcp_smem[];
  const int lg = __ffs(lanes_per_head) - 1;  // lanes_per_head is a power of two
  const int H = 32 >> lg;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int head = lane >> lg;
  const bool head_leader = (lane & (lanes_per_head - 1)) == 0;
  int* ids = reinterpret_cast<int*>(gcp_smem + (long)warp * S * (H + 1));  // [S]
  float* sim = reinterpret_cast<float*>(ids + S);                           // [S][H]
  const long tok = (long)blockIdx.x * (blockDim.x >> 5) + warp;
  if (tok >= BT) return;
  const int b = (int)(tok / T);
  const int inner = 32 * 16;  // H*Dh
  const __half* kvb = kv + (long)b * (V + 1) * (2 * inner);
  float qf[16];
  ld16h(q + tok * inner + lane * 16, qf);
  for (int s0 = 0; s0 < S; s0 += GCP_CHUNK) {
#pragma unroll
    for (int j = 0; j < GCP_CHUNK; ++j) {
      const int s = s0 + j;
      if (s < S) {
        const int id = idx[tok * S + s];
        float kf[16];
        ld16h(kvb + (long)id * (2 * inner) + lane * 16, kf);
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) d = fmaf(qf[i], kf[i], d);
        for (int o = 1; o < lanes_per_head; o <<= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (lane == 0) ids[s] = id;
        // additive -1e4 on padding slots (":219-223", "for half")
        if (head_leader) sim[s * H + head] = d + (id == V ? -1e4f : 0.f);
      }
    }
  }
  __syncwarp();
  float mx = -INFINITY;
  for (int s = 0; s < S; ++s) mx = fmaxf(mx, sim[s * H + head]);
  // e, den and p are rounded one operation at a time: never contracted with the last multiply of expf
  float den = 0.f;
  for (int s = 0; s < S; ++s) den = __fadd_rn(den, expf(sim[s * H + head] - mx));
  const float inv = 1.f / den;
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  for (int s0 = 0; s0 < S; s0 += GCP_CHUNK) {
#pragma unroll
    for (int j = 0; j < GCP_CHUNK; ++j) {
      const int s = s0 + j;
      if (s < S) {
        const int id = ids[s];
        // probabilities of padding slots are zeroed AFTER the softmax, without renormalisation (:227-231)
        const float p = (id == V) ? 0.f : __fmul_rn(expf(sim[s * H + head] - mx), inv);
        float vf[16];
        ld16h(kvb + (long)id * (2 * inner) + inner + lane * 16, vf);
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = fmaf(p, vf[i], acc[i]);
      }
    }
  }
  __half2 h[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) h[i] = __floats2half2_rn(acc[2 * i], acc[2 * i + 1]);
  uint4* dst = reinterpret_cast<uint4*>(out + tok * inner + lane * 16);
  dst[0] = *reinterpret_cast<uint4*>(&h[0]);
  dst[1] = *reinterpret_cast<uint4*>(&h[4]);
}

// g = tanh(h1 . w2); x1 = s*g + x; ln = LN(x1).  One warp per row.
__global__ void __launch_bounds__(256) gcp_gate_residual_ln_kernel(const __half* __restrict__ h1, const float* __restrict__ w2,
                                                                   int Dg, const float* __restrict__ s,
                                                                   const float* __restrict__ x,
                                                                   const float* __restrict__ gamma,
                                                                   const float* __restrict__ beta, float eps, long rows,
                                                                   int D, float* __restrict__ x1_out,
                                                                   __half* __restrict__ ln_out, float* __restrict__ gate_out) {
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float d = 0.f;
  for (int i = lane; i < Dg; i += 32) d = fmaf(__half2float(h1[row * Dg + i]), w2[i], d);
  const float g = tanhf(warp_sum(d));
  if (gate_out && lane == 0) gate_out[row] = g;
  const float* sr = s + row * D;
  const float* xr = x + row * D;
  float sum = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float v = fmaf(sr[i], g, xr[i]);
    x1_out[row * D + i] = v;
    sum += v;
  }
  const float mean = warp_sum(sum) / D;
  float var = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float v = fmaf(sr[i], g, xr[i]) - mean;
    var += v * v;
  }
  const float rstd = rsqrtf(warp_sum(var) / D + eps);
  for (int i = lane; i < D; i += 32) {
    const float v = fmaf(sr[i], g, xr[i]);
    ln_out[row * D + i] = __float2half_rn((v - mean) * rstd * gamma[i] + beta[i]);
  }
}

// idx[b,t,0:S] = ascending v with mask[b,v,t] != 0, padded with V.
__global__ void gcp_build_index_kernel(const float* __restrict__ mask, int B, int V, int T, int S, int* __restrict__ idx,
                                       int* __restrict__ counts) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T) return;
  const int b = (int)(i / T), t = (int)(i % T);
  const float* m = mask + (long)b * V * T + t;
  int n = 0, total = 0;
  for (int v = 0; v < V; ++v) {
    if (m[(long)v * T] != 0.f) {
      if (n < S) idx[i * S + n++] = v;
      ++total;
    }
  }
  for (; n < S; ++n) idx[i * S + n] = V;
  if (counts) counts[i] = total;
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_gcp_sparse_attn(const void* q, const void* kv, const int32_t* idx, void* out, int64_t B, int64_t T,
                                     int64_t V, int64_t S, int64_t H, int64_t Dh, void* stream) {
  MQ_REQUIRE(q && kv && idx && out, "gcp_sparse_attn: null pointer");
  MQ_REQUIRE(H * Dh == 512 && (Dh % 16) == 0 && Dh <= 512, "gcp_sparse_attn: H*Dh must be 512 (got %ld x %ld)", (long)H,
             (long)Dh);
  MQ_REQUIRE(S >= 1 && S <= GCP_MAX_S, "gcp_sparse_attn: S=%ld queries per token out of range [1,%d]", (long)S, GCP_MAX_S);
  const int lph = (int)(Dh / 16);
  MQ_REQUIRE((lph & (lph - 1)) == 0, "gcp_sparse_attn: Dh/16 must be a power of two");
  const long BT = B * T;
  const long slice = gcp_slice_bytes(S, H);
  const int wpb = (int)std::min<long>(8, GCP_SMEM_MAX / slice);
  const int smem = (int)(wpb * slice);
  if (smem > 48 * 1024) {
    const int rc = ensure_dyn_smem((const void*)gcp_sparse_attn_kernel, smem);
    if (rc != MQDET_OK) return rc;
  }
  gcp_sparse_attn_kernel<<<cdiv(BT, wpb), wpb * 32, smem, (cudaStream_t)stream>>>((const __half*)q, (const __half*)kv, idx,
                                                                                (__half*)out, BT, (int)T, (int)V, (int)S, lph);
  return check_launch("gcp_sparse_attn_kernel");
}

extern "C" int mqdet_gcp_gate_residual_ln(const void* h1, const float* w2, int64_t Dg, const float* s, const float* x,
                                          const float* gamma, const float* beta, float eps, int64_t rows, int64_t D,
                                          float* x1_out, void* ln_out16, float* gate_out, void* stream) {
  MQ_REQUIRE(h1 && w2 && s && x && gamma && beta && x1_out && ln_out16, "gcp_gate_residual_ln: null pointer");
  const int wpb = 8;
  gcp_gate_residual_ln_kernel<<<cdiv(rows, wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
      (const __half*)h1, w2, (int)Dg, s, x, gamma, beta, eps, rows, (int)D, x1_out, (__half*)ln_out16, gate_out);
  return check_launch("gcp_gate_residual_ln_kernel");
}

extern "C" int mqdet_gcp_build_index(const float* mask, int64_t B, int64_t V, int64_t T, int64_t S, int32_t* idx,
                                     int32_t* counts_out, void* stream) {
  MQ_REQUIRE(mask && idx && B > 0 && V > 0 && T > 0 && S > 0, "gcp_build_index: bad args");
  const long n = B * T;
  gcp_build_index_kernel<<<cdiv(n, 128), 128, 0, (cudaStream_t)stream>>>(mask, (int)B, (int)V, (int)T, (int)S, idx,
                                                                        counts_out);
  return check_launch("gcp_build_index_kernel");
}
