// mqdet_b200 — fp16 x fp16 -> fp32-accumulate GEMM with fused epilogue, hand-written for sm_90a.
//
//   D[z][m,n] = epi( sum_k A[z][m,k] * B[z][n,k] )      (both operands K-contiguous: "TN")
//
// Product kernel (gemm_wg_kernel): warp-specialised, one 128 x BN output tile per CTA (BN = 64 or 128).
//   warpgroup 0    : TMA producer — one thread issues cp.async.bulk.tensor (4-D maps, 128B swizzle) into a STAGES-deep ring
//   warpgroups 1-2 : consumers    — rows 0-63 / 64-127 of the tile: wgmma.m64nBNk16 from the swizzled ring (fp32
//                                   accumulators in registers, one commit group per k-block, the previous k-block's slot
//                                   released as soon as its group retires), then the epilogue straight from the fragments
// The grid runs n-tiles fastest so the A row-panel is shared through L2.
//
// Validation kernel (gemm_simt_kernel): plain 64x64 shared-memory tiled FMA kernel with the same
// epilogue, used by the tests to cross-check the tensor-core path (never by the product path).
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

struct GemmP {
  const __half* A;
  const __half* B;
  long M, N, K, lda, ldb;
  int nb1, nb2;
  long a_b1, a_b2, b_b1, b_b2;
  void* C;
  int c_dtype;
  long ldc, c_b1, c_b2;
  float alpha;
  int scale_after_bias;
  const float* bias;
  int bias_mode;
  long bias_b1, bias_b2;
  int act;
  float clamp;
  const float* gate;
  int gate_mode, gate_tanh;
  const void* R;
  int r_dtype;
  long ldr, r_b1, r_b2;
  int a_bcast1, a_bcast2, b_bcast1, b_bcast2;  // 1 -> TMA coordinate pinned to 0
  int vec2;                                    // output pairs (col, col + 1) may be written with one aligned store
};

// One output element's epilogue:
//   epi_pre : alpha / bias / activation / clamp / gate      epi_one = epi_pre + residual
__device__ __forceinline__ float epi_pre(const GemmP& p, float acc, long row, long col, int z1, int z2,
                                         float gate_scalar) {
  float v = acc;
  float b = 0.f;
  if (p.bias_mode == MQDET_VEC_PER_COL)
    b = p.bias[z1 * p.bias_b1 + z2 * p.bias_b2 + col];
  else if (p.bias_mode == MQDET_VEC_PER_ROW)
    b = p.bias[z1 * p.bias_b1 + z2 * p.bias_b2 + row];
  v = p.scale_after_bias ? p.alpha * (v + b) : p.alpha * v + b;
  if (p.act == MQDET_ACT_GELU)
    v = gelu_erf(v);
  else if (p.act == MQDET_ACT_RELU)
    v = fmaxf(v, 0.f);
  if (p.clamp > 0.f) v = fminf(fmaxf(v, -p.clamp), p.clamp);
  if (p.gate_mode == MQDET_VEC_SCALAR) {
    v *= gate_scalar;
  } else if (p.gate_mode == MQDET_VEC_PER_COL) {
    float g = p.gate[col];
    v *= p.gate_tanh ? tanhf(g) : g;
  } else if (p.gate_mode == MQDET_VEC_PER_ROW) {
    float g = p.gate[row];
    v *= p.gate_tanh ? tanhf(g) : g;
  }
  return v;
}
__device__ __forceinline__ float ld_residual(const GemmP& p, long row, long col, int z1, int z2) {
  const long off = z1 * p.r_b1 + z2 * p.r_b2 + row * p.ldr + col;
  return (p.r_dtype == MQDET_F32) ? reinterpret_cast<const float*>(p.R)[off]
                                  : __half2float(reinterpret_cast<const __half*>(p.R)[off]);
}
__device__ __forceinline__ float epi_one(const GemmP& p, float acc, long row, long col, int z1, int z2,
                                         float gate_scalar) {
  float v = epi_pre(p, acc, row, col, z1, z2, gate_scalar);
  if (p.R) v += ld_residual(p, row, col, z1, z2);
  return v;
}

__device__ __forceinline__ void store_one(const GemmP& p, float v, long row, long col, int z1, int z2) {
  long off = z1 * p.c_b1 + z2 * p.c_b2 + row * p.ldc + col;
  if (p.c_dtype == MQDET_F32)
    reinterpret_cast<float*>(p.C)[off] = v;
  else
    reinterpret_cast<__half*>(p.C)[off] = __float2half_rn(v);
}

// ---------------------------------------------------------------------------------------------
// wgmma kernel
// ---------------------------------------------------------------------------------------------
constexpr int BM = 128;
constexpr int BK = 64;  // 64 fp16 = 128 B = one swizzle row

template <int BN, int STAGES>
struct WgCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 128)
    wgmma_ss_m64n128_kk(acc, da, db, 1);
  else
    wgmma_ss_m64n64_kk(acc, da, db, 1);
}

// 128 x 64 tiles: two CTAs per SM (96 KB of shared memory each), so one CTA's epilogue overlaps the other's main loop
template <int BN, int STAGES>
__global__ void __launch_bounds__(384, BN == 128 ? 1 : 2) gemm_wg_kernel(const __grid_constant__ CUtensorMap tma_a,
                                                                        const __grid_constant__ CUtensorMap tma_b, const GemmP p) {
  using Cfg = WgCfg<BN, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled tiles need 1024-byte alignment.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * Cfg::A_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int n_tile = blockIdx.x, m_tile = blockIdx.y;
  const int z1 = blockIdx.z % p.nb1, z2 = blockIdx.z / p.nb1;
  const int num_kb = (int)((p.K + BK - 1) / BK);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 256);  // every consumer thread arrives once its wgmma group has read the slot
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (tid == 0) {
      const int az1 = p.a_bcast1 ? 0 : z1, az2 = p.a_bcast2 ? 0 : z2;
      const int bz1 = p.b_bcast1 ? 0 : z1, bz2 = p.b_bcast2 ? 0 : z2;
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        mbar_wait(&empty_bar[s], ((kb / STAGES) & 1) ^ 1);
        mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
        tma_load_4d(smem_a + s * Cfg::A_BYTES, &tma_a, &full_bar[s], kb * BK, m_tile * BM, az1, az2);
        tma_load_4d(smem_b + s * Cfg::B_BYTES, &tma_b, &full_bar[s], kb * BK, n_tile * BN, bz1, bz2);
      }
    }
    return;
  }
  const int g = wg - 1;  // rows 64 g .. 64 g + 63 of the tile
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(&full_bar[s], (kb / STAGES) & 1);
    const uint32_t a_addr = smem_u32(smem_a + s * Cfg::A_BYTES) + g * (64 * 128);
    const uint32_t b_addr = smem_u32(smem_b + s * Cfg::B_BYTES);
    wgmma_fence_acc(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) wgmma_tile<BN>(acc, wg_desc_k_sw128(a_addr + k * 32), wg_desc_k_sw128(b_addr + k * 32));
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's group has retired: its slot may be refilled
    wgmma_fence_acc(acc);
    if (kb > 0) mbar_arrive(&empty_bar[(kb - 1) % STAGES]);
  }
  wgmma_wait<0>();
  wgmma_fence_acc(acc);

  // ---- epilogue from the accumulator fragments: bias / act / clamp / gate / residual, column pairs per store ----
  float gate_s = 1.f;
  if (p.gate_mode == MQDET_VEC_SCALAR) gate_s = p.gate_tanh ? tanhf(p.gate[0]) : p.gate[0];
  const long row0 = (long)m_tile * BM + g * 64, col0 = (long)n_tile * BN;
#pragma unroll
  for (int i = 0; i < BN / 2; i += 2) {
    const long row = row0 + wg_row(tid, i), col = col0 + wg_col(tid, i);
    if (row >= p.M || col >= p.N) continue;
    const float v0 = epi_one(p, acc[i], row, col, z1, z2, gate_s);
    if (col + 1 < p.N) {
      const float v1 = epi_one(p, acc[i + 1], row, col + 1, z1, z2, gate_s);
      if (p.vec2) {
        const long off = z1 * p.c_b1 + z2 * p.c_b2 + row * p.ldc + col;
        if (p.c_dtype == MQDET_F32)
          *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.C) + off) = make_float2(v0, v1);
        else
          *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.C) + off) = __floats2half2_rn(v0, v1);
        continue;
      }
      store_one(p, v1, row, col + 1, z1, z2);
    }
    store_one(p, v0, row, col, z1, z2);
  }
}

// ---------------------------------------------------------------------------------------------
// SIMT validation kernel: 64x64 tile, 16x16 threads, 4x4 micro-tile.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gemm_simt_kernel(const GemmP p) {
  __shared__ float sa[16][64 + 1];
  __shared__ float sb[16][64 + 1];
  const int z1 = blockIdx.z % p.nb1, z2 = blockIdx.z / p.nb1;
  const __half* A = p.A + z1 * p.a_b1 + z2 * p.a_b2;
  const __half* B = p.B + z1 * p.b_b1 + z2 * p.b_b2;
  const long m0 = (long)blockIdx.y * 64, n0 = (long)blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  for (long k0 = 0; k0 < p.K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int r = i >> 4, k = i & 15;
      const long gm = m0 + r, gn = n0 + r, gk = k0 + k;
      sa[k][r] = (gm < p.M && gk < p.K) ? __half2float(A[gm * p.lda + gk]) : 0.f;
      sb[k][r] = (gn < p.N && gk < p.K) ? __half2float(B[gn * p.ldb + gk]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = sa[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = sb[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  float gate_scalar = 1.f;
  if (p.gate_mode == MQDET_VEC_SCALAR) {
    gate_scalar = p.gate[0];
    if (p.gate_tanh) gate_scalar = tanhf(gate_scalar);
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      const long row = m0 + ty * 4 + i, col = n0 + tx * 4 + j;
      if (row < p.M && col < p.N) store_one(p, epi_one(p, acc[i][j], row, col, z1, z2, gate_scalar), row, col, z1, z2);
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// make_operand_map / num_sms / ensure_dyn_smem: capi.cu (shared with the other TMA kernels; tensor maps are cached)
template <int BN, int STAGES>
static int launch_wg(const GemmP& p0, cudaStream_t st) {
  using Cfg = WgCfg<BN, STAGES>;
  GemmP p = p0;
  CUtensorMap ma, mb;
  int rc = make_operand_map(&ma, p.A, p.M, p.K, p.lda, p.nb1, p.a_b1, p.nb2, p.a_b2, BM, &p.a_bcast1, &p.a_bcast2);
  if (rc) return rc;
  rc = make_operand_map(&mb, p.B, p.N, p.K, p.ldb, p.nb1, p.b_b1, p.nb2, p.b_b2, BN, &p.b_bcast1, &p.b_bcast2);
  if (rc) return rc;
  const long al = p.c_dtype == MQDET_F16 ? 2 : 1;  // pair stores: 4-byte (fp16) / 8-byte (fp32) aligned
  p.vec2 = (p.ldc % 2 == 0) && (p.nb1 == 1 || p.c_b1 % 2 == 0) && (p.nb2 == 1 || p.c_b2 % 2 == 0) &&
           (reinterpret_cast<uintptr_t>(p.C) % (4 * (3 - al))) == 0;
  rc = ensure_dyn_smem(reinterpret_cast<const void*>(&gemm_wg_kernel<BN, STAGES>), Cfg::SMEM_BYTES);
  if (rc) return rc;
  dim3 grid(cdiv(p.N, BN), cdiv(p.M, BM), p.nb1 * p.nb2);
  gemm_wg_kernel<BN, STAGES><<<grid, 384, Cfg::SMEM_BYTES, st>>>(ma, mb, p);
  return check_launch("gemm_wg_kernel");
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_gemm_f16(const mqdet_gemm_args* a, int impl, void* stream) {
  MQ_REQUIRE(a && a->A && a->B && a->C, "gemm: null pointer");
  MQ_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "gemm: empty problem M=%ld N=%ld K=%ld", (long)a->M, (long)a->N,
             (long)a->K);
  MQ_REQUIRE(a->nb1 >= 1 && a->nb2 >= 1 && a->nb1 * a->nb2 <= 65535, "gemm: bad batch %ld x %ld", (long)a->nb1,
             (long)a->nb2);
  MQ_REQUIRE(a->c_dtype == MQDET_F16 || a->c_dtype == MQDET_F32, "gemm: bad c_dtype");
  GemmP p;
  memset(&p, 0, sizeof(p));
  p.A = (const __half*)a->A;
  p.B = (const __half*)a->B;
  p.M = a->M; p.N = a->N; p.K = a->K; p.lda = a->lda; p.ldb = a->ldb;
  p.nb1 = (int)a->nb1; p.nb2 = (int)a->nb2;
  p.a_b1 = a->a_b1; p.a_b2 = a->a_b2; p.b_b1 = a->b_b1; p.b_b2 = a->b_b2;
  p.C = a->C; p.c_dtype = a->c_dtype; p.ldc = a->ldc; p.c_b1 = a->c_b1; p.c_b2 = a->c_b2;
  p.alpha = a->alpha; p.scale_after_bias = a->scale_after_bias;
  p.bias = a->bias; p.bias_mode = a->bias ? a->bias_mode : MQDET_VEC_NONE;
  p.bias_b1 = a->bias_b1; p.bias_b2 = a->bias_b2;
  p.act = a->act; p.clamp = a->clamp;
  p.gate = a->gate; p.gate_mode = a->gate ? a->gate_mode : MQDET_VEC_NONE; p.gate_tanh = a->gate_tanh;
  p.R = a->R; p.r_dtype = a->r_dtype; p.ldr = a->ldr; p.r_b1 = a->r_b1; p.r_b2 = a->r_b2;
  cudaStream_t st = (cudaStream_t)stream;

  if (impl == MQDET_GEMM_IMPL_SIMT) {
    dim3 grid(cdiv(p.N, 64), cdiv(p.M, 64), p.nb1 * p.nb2);
    gemm_simt_kernel<<<grid, 256, 0, st>>>(p);
    return check_launch("gemm_simt_kernel");
  }
  MQ_REQUIRE(impl == MQDET_GEMM_IMPL_TC || impl == MQDET_GEMM_IMPL_TC_ONESHOT, "gemm: unknown impl %d", impl);
  MQ_REQUIRE((a->K % 8) == 0 && (a->lda % 8) == 0 && (a->ldb % 8) == 0, "gemm: K/lda/ldb must be multiples of 8");
  MQ_REQUIRE((a->a_b1 % 8) == 0 && (a->a_b2 % 8) == 0 && (a->b_b1 % 8) == 0 && (a->b_b2 % 8) == 0,
             "gemm: batch strides must be multiples of 8");
  MQ_REQUIRE(((uintptr_t)a->A % 16) == 0 && ((uintptr_t)a->B % 16) == 0, "gemm: A/B must be 16-byte aligned");
  // 128-wide tiles when they still give every SM a tile, 64-wide ones (two CTAs per SM) otherwise
  const long tiles128 = (long)cdiv(p.M, BM) * cdiv(p.N, 128) * p.nb1 * p.nb2;
  if (p.N > 64 && tiles128 >= num_sms()) return launch_wg<128, 4>(p, st);
  return launch_wg<64, 4>(p, st);
}
