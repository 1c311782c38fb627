// mqdet_b200 — dense multi-head cross-attention with a small head dimension (PreSelect: 8 heads x 32, a few hundred vision
// queries attending to the 5577 pooled image tokens) as ONE flash-style kernel.
//
// Reference: MaskedCrossAttention.forward with spase_forward=False and no mask (maskrcnn_benchmark/modeling/language_backbone/
// modeling_bert_new.py:186-248), as used by PreSelectBlock (:398-409):  sim = q k^T (q already scaled), softmax over the image
// tokens, out = attn v.  Round 1 materialised the fp32 score tensor [B, 8, V, 5577] (571 MB at B = 8) twice per step.
//
// One CTA (4 warps) per (64 queries, head, image); a warp owns 16 queries.  Keys / values stream through shared memory in
// chunks of 64 tokens (16-byte global loads of the NEXT chunk are in flight while the current one is consumed; V is stored
// transposed because the B fragments of P.V need two consecutive KEYS per register).  S = Q K^T and O += P V run on
// mma.sync.m16n8k16 (a 16 x 64 x 32 problem per warp and chunk is far below a wgmma tile); the softmax is the online
// (running max / running sum) form in the accumulator fragments, fp32 throughout, P travels as fp16.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

__device__ __forceinline__ void xa_mma_16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

constexpr int XA_D = 32, XA_KC = 64, XA_KLD = 40, XA_VLD = 72;

// q [B][Tq][q_ld] (head h at column h*32), kv [B][I][kv_ld] (K of head h at column h*32, V at v_col0 + h*32), out [B][Tq][o_ld]
__global__ void __launch_bounds__(128) dense_cross_attn_kernel(const __half* __restrict__ q, long q_ld, long q_b,
                                                               const __half* __restrict__ kv, long kv_ld, long kv_b, int v_col0,
                                                               __half* __restrict__ out, long o_ld, long o_b, int Tq, int I) {
  __shared__ __align__(16) __half ks[XA_KC * XA_KLD];
  __shared__ __align__(16) __half vT[XA_D * XA_VLD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int h = blockIdx.y, b = blockIdx.z;
  const int row0 = blockIdx.x * 64 + warp * 16;
  const int r0 = row0 + g, r1 = r0 + 8;
  const __half* qb = q + (long)b * q_b + h * XA_D;
  const __half* kb = kv + (long)b * kv_b + h * XA_D;
  const __half* vb = kv + (long)b * kv_b + v_col0 + h * XA_D;
  // Q fragments of this warp's 16 queries (rows beyond Tq read row Tq-1: finite values, never stored)
  uint32_t qf[2][4];
  {
    const __half* q0 = qb + (long)min(r0, Tq - 1) * q_ld;
    const __half* q1 = qb + (long)min(r1, Tq - 1) * q_ld;
#pragma unroll
    for (int ki = 0; ki < 2; ++ki) {
      qf[ki][0] = *reinterpret_cast<const uint32_t*>(q0 + 16 * ki + 2 * t4);
      qf[ki][1] = *reinterpret_cast<const uint32_t*>(q1 + 16 * ki + 2 * t4);
      qf[ki][2] = *reinterpret_cast<const uint32_t*>(q0 + 16 * ki + 2 * t4 + 8);
      qf[ki][3] = *reinterpret_cast<const uint32_t*>(q1 + 16 * ki + 2 * t4 + 8);
    }
  }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float oacc[4][4];
#pragma unroll
  for (int ni = 0; ni < 4; ++ni)
#pragma unroll
    for (int e = 0; e < 4; ++e) oacc[ni][e] = 0.f;
  // staging: thread -> (key = tid / 2 within the chunk ... ) 64 keys x 4 pieces of 8 dims for K and for V = 512 pieces / 128 threads
  const int nchunks = (I + XA_KC - 1) / XA_KC;
  uint4 pk[2], pv[2];
  auto fetch = [&](int c) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int piece = threadIdx.x + u * 128, key = piece >> 2, d0 = (piece & 3) * 8;
      const int tok = c * XA_KC + key;
      if (tok < I) {
        pk[u] = __ldg(reinterpret_cast<const uint4*>(kb + (long)tok * kv_ld + d0));
        pv[u] = __ldg(reinterpret_cast<const uint4*>(vb + (long)tok * kv_ld + d0));
      } else {
        pk[u] = make_uint4(0, 0, 0, 0);
        pv[u] = make_uint4(0, 0, 0, 0);
      }
    }
  };
  fetch(0);
  for (int c = 0; c < nchunks; ++c) {
    __syncthreads();  // every warp has finished reading the previous chunk
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int piece = threadIdx.x + u * 128, key = piece >> 2, d0 = (piece & 3) * 8;
      *reinterpret_cast<uint4*>(ks + key * XA_KLD + d0) = pk[u];
      const __half* hv = reinterpret_cast<const __half*>(&pv[u]);
#pragma unroll
      for (int e = 0; e < 8; ++e) vT[(d0 + e) * XA_VLD + key] = hv[e];
    }
    __syncthreads();
    if (c + 1 < nchunks) fetch(c + 1);  // in flight while this chunk is consumed
    // ---- S = Q K^T for 64 keys ----
    float sacc[8][4];
#pragma unroll
    for (int nj = 0; nj < 8; ++nj) {
#pragma unroll
      for (int e = 0; e < 4; ++e) sacc[nj][e] = 0.f;
      uint32_t kf0[2], kf1[2];
      kf0[0] = *reinterpret_cast<const uint32_t*>(ks + (8 * nj + g) * XA_KLD + 2 * t4);
      kf0[1] = *reinterpret_cast<const uint32_t*>(ks + (8 * nj + g) * XA_KLD + 2 * t4 + 8);
      kf1[0] = *reinterpret_cast<const uint32_t*>(ks + (8 * nj + g) * XA_KLD + 16 + 2 * t4);
      kf1[1] = *reinterpret_cast<const uint32_t*>(ks + (8 * nj + g) * XA_KLD + 16 + 2 * t4 + 8);
      xa_mma_16816(sacc[nj], qf[0], kf0);
      xa_mma_16816(sacc[nj], qf[1], kf1);
    }
    // ---- online softmax ----
    const int kbase = c * XA_KC;
    float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
    for (int nj = 0; nj < 8; ++nj)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kbase + 8 * nj + 2 * t4 + (e & 1);
        if (key >= I) sacc[nj][e] = -INFINITY;
        if (e < 2) cm0 = fmaxf(cm0, sacc[nj][e]); else cm1 = fmaxf(cm1, sacc[nj][e]);
      }
    cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 1));
    cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 2));
    cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 1));
    cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 2));
    const float mn0 = fmaxf(m0, cm0), mn1 = fmaxf(m1, cm1);  // finite: every chunk holds at least one real key
    const float sc0 = __expf(m0 - mn0), sc1 = __expf(m1 - mn1);  // exp(-inf) = 0 on the first chunk
    m0 = mn0;
    m1 = mn1;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int nj = 0; nj < 8; ++nj)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pvv = __expf(sacc[nj][e] - ((e < 2) ? mn0 : mn1));
        sacc[nj][e] = pvv;
        if (e < 2) s0 += pvv; else s1 += pvv;
      }
    s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
    s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
    l0 = l0 * sc0 + s0;
    l1 = l1 * sc1 + s1;
#pragma unroll
    for (int ni = 0; ni < 4; ++ni) {
      oacc[ni][0] *= sc0; oacc[ni][1] *= sc0;
      oacc[ni][2] *= sc1; oacc[ni][3] *= sc1;
    }
    // ---- O += P V ----
#pragma unroll
    for (int kj = 0; kj < 4; ++kj) {
      uint32_t pf[4];
      pf[0] = pack_half2(sacc[2 * kj][0], sacc[2 * kj][1]);
      pf[1] = pack_half2(sacc[2 * kj][2], sacc[2 * kj][3]);
      pf[2] = pack_half2(sacc[2 * kj + 1][0], sacc[2 * kj + 1][1]);
      pf[3] = pack_half2(sacc[2 * kj + 1][2], sacc[2 * kj + 1][3]);
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        uint32_t vf[2];
        vf[0] = *reinterpret_cast<const uint32_t*>(vT + (8 * ni + g) * XA_VLD + 16 * kj + 2 * t4);
        vf[1] = *reinterpret_cast<const uint32_t*>(vT + (8 * ni + g) * XA_VLD + 16 * kj + 2 * t4 + 8);
        xa_mma_16816(oacc[ni], pf, vf);
      }
    }
  }
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
  __half* ob = out + (long)b * o_b + h * XA_D;
#pragma unroll
  for (int ni = 0; ni < 4; ++ni) {
    const int d = 8 * ni + 2 * t4;
    if (r0 < Tq) *reinterpret_cast<uint32_t*>(ob + (long)r0 * o_ld + d) = pack_half2(oacc[ni][0] * inv0, oacc[ni][1] * inv0);
    if (r1 < Tq) *reinterpret_cast<uint32_t*>(ob + (long)r1 * o_ld + d) = pack_half2(oacc[ni][2] * inv1, oacc[ni][3] * inv1);
  }
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_dense_cross_attn(const void* q, int64_t q_ld, int64_t q_b, const void* kv, int64_t kv_ld, int64_t kv_b,
                                      int64_t v_col0, void* out, int64_t o_ld, int64_t o_b, int64_t B, int64_t Tq, int64_t I,
                                      int64_t heads, int64_t head_dim, void* stream) {
  MQ_REQUIRE(q && kv && out, "dense_cross_attn: null pointer");
  MQ_REQUIRE(head_dim == 32, "dense_cross_attn: head dim must be 32 (PreSelect dim_head_v, modeling_bert_new.py:643-660), got %ld",
             (long)head_dim);
  MQ_REQUIRE(B >= 1 && Tq >= 1 && I >= 1 && heads >= 1 && heads <= 65535 && B <= 65535, "dense_cross_attn: empty problem");
  MQ_REQUIRE((q_ld % 2) == 0 && (kv_ld % 8) == 0 && (v_col0 % 8) == 0 && (o_ld % 2) == 0 && (kv_b % 8) == 0 &&
                 ((uintptr_t)kv % 16) == 0 && ((uintptr_t)q % 4) == 0 && ((uintptr_t)out % 4) == 0,
             "dense_cross_attn: kv rows must take 16-byte loads, q / out rows 4-byte accesses");
  dim3 grid((unsigned)((Tq + 63) / 64), (unsigned)heads, (unsigned)B);
  dense_cross_attn_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const __half*)q, q_ld, q_b, (const __half*)kv, kv_ld, kv_b,
                                                                  (int)v_col0, (__half*)out, o_ld, o_b, (int)Tq, (int)I);
  return check_launch("dense_cross_attn_kernel");
}
