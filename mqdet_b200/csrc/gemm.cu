// mqdet_b200 — fp16 x fp16 -> fp32-accumulate GEMM with fused epilogue, hand-written for sm_90a.
//
//   D[z][m,n] = epi( sum_k A[z][m,k] * B[z][n,k] )      (both operands K-contiguous: "TN")
//
// Product kernel (gemm_wg_kernel): warp-specialised and persistent, 128 x BN output tiles (BN = 64 or 128), one CTA per SM
// walking a static tile schedule (n-tiles fastest, so the CTAs running side by side share the A row-panel through L2).
//   warpgroup 0    : TMA producer — one thread issues cp.async.bulk.tensor (4-D maps, 128B swizzle) into a STAGES-deep ring,
//                                   running ahead into the next tile's k-blocks while the consumers finish the current one
//                                   (setmaxnreg hands its registers to the consumers)
//   warpgroups 1-2 : consumers    — ping-pong over the CTA's tiles: each takes every other tile whole (two wgmma.m64nBNk16
//                                   rows from the swizzled ring, fp32 accumulators in registers, one commit group per k-block,
//                                   the previous k-block's slot released as soon as its group retires) and runs its epilogue
//                                   while the other runs the next tile's main loop.  Epilogue: for the hot variants (none /
//                                   bias / bias + GELU in fp16, bias + fp32 residual in fp32) on the fragments into a swizzled
//                                   shared box, then a TMA store; otherwise fragments -> fp32 shared staging -> a rolled loop
//                                   over rows (consecutive threads on consecutive columns: coalesced residual loads and stores)
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

// Epilogue variants compiled as their own kernels: the Swin / FPN / FFN products use the four specialised ones, which run on
// the accumulator fragments and leave the tile by TMA store; everything else (alpha, row bias, ReLU, clamp, gates, fp16
// residual, outputs TMA cannot address) takes the generic rolled loop with pointer stores.
enum GemmEpi : int {
  EPI_GENERIC = 0,
  EPI_NONE_F16,       // fp16 out
  EPI_BIAS_F16,       // per-column bias, fp16 out
  EPI_BIAS_GELU_F16,  // per-column bias + erf-GELU, fp16 out
  EPI_BIAS_RES_F32,   // per-column bias + fp32 residual, fp32 out
};

template <int BN, int STAGES, int EPI>
struct WgCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int PITCH = BN + 8;  // fp32 staging row pitch: fragment writes (8 rows x 32 B per warp) are conflict-free
  // TMA-store staging: 128-byte-wide column boxes of BM rows (128B swizzle), BM x BN x 2 bytes per consumer warpgroup.  An fp32
  // tile takes two passes of BN / 2 columns through it.
  static constexpr bool OUT_F32 = EPI == EPI_BIAS_RES_F32;
  static constexpr int ES = OUT_F32 ? 4 : 2;
  static constexpr int PASSES = OUT_F32 ? 2 : 1;
  static constexpr int PASS_COLS = BN / PASSES;
  static constexpr int BOX_COLS = 128 / ES;
  static constexpr int BOXES = PASS_COLS / BOX_COLS;
  // generic: 64 rows of fp32 accumulators at a time (the tile's two halves in turn)
  static constexpr int EPI_BYTES = EPI == EPI_GENERIC ? 64 * PITCH * 4 : BM * BN * 2;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * EPI_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(EPI_BYTES % 1024 == 0, "swizzled boxes need 1024-byte alignment");
};

// Byte address of element (r, c) in the TMA-store staging: box c / BOX_COLS, 128-byte rows, 16-byte chunks XOR-swizzled by
// r % 8 (the layout CU_TENSOR_MAP_SWIZZLE_128B reads).  A warp's fragment writes (8 rows x 4 threads) hit 8 distinct chunks.
template <int ES>
__device__ __forceinline__ uint32_t box_addr(uint32_t base, int r, int c) {
  const int byte = c * ES;
  return base + (byte >> 7) * (BM * 128) + r * 128 + ((((byte >> 4) & 7) ^ (r & 7)) << 4) + (byte & 15);
}

// Static persistent schedule: tile t -> (batch z, m-tile, n-tile), n-tiles fastest so the CTAs running side by side share
// their A row-panels through L2.
struct TileIdx {
  int n_tile, m_tile, z1, z2;
};
__device__ __forceinline__ TileIdx tile_idx(int t, int n_tiles, int m_tiles, int nb1) {
  TileIdx r;
  const int per_z = n_tiles * m_tiles;
  const int z = t / per_z, rem = t - z * per_z;
  r.m_tile = rem / n_tiles;
  r.n_tile = rem - r.m_tile * n_tiles;
  r.z1 = z % nb1;
  r.z2 = z / nb1;
  return r;
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 128)
    wgmma_ss_m64n128_kk(acc, da, db, 1);
  else
    wgmma_ss_m64n64_kk(acc, da, db, 1);
}

// Persistent: CTA c computes tiles c, c + gridDim.x, ... (static schedule, no device-side counters, so a captured graph
// replays without resets).  The producer thread fills the ring with every tile's k-blocks in schedule order.  The two
// consumer warpgroups ping-pong: warpgroup g takes the CTA's tiles 2 j + g, each a whole 128 x BN tile (two m64 wgmma rows),
// and skips the other's k-blocks in its ring counter.  A pair of named barriers hands the MMA turn from one warpgroup to the
// other once its tile's wgmma groups have retired, so one warpgroup's main loop runs while the other runs its epilogue; the
// strict turn order also keeps every full-barrier wait within one phase of the barrier's state.  gridDim.x = number of tiles
// gives one tile per CTA (MQDET_GEMM_IMPL_TC_ONESHOT).
template <int BN, int STAGES, int EPI>
__global__ void __launch_bounds__(384, 1) gemm_wg_kernel(const __grid_constant__ CUtensorMap tma_a,
                                                         const __grid_constant__ CUtensorMap tma_b,
                                                         const __grid_constant__ CUtensorMap tma_c, const GemmP p) {
  using Cfg = WgCfg<BN, STAGES, EPI>;
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled tiles need 1024-byte alignment.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * Cfg::A_BYTES;
  uint8_t* smem_c = smem + STAGES * Cfg::STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_c + 2 * Cfg::EPI_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int n_tiles = (int)((p.N + BN - 1) / BN), m_tiles = (int)((p.M + BM - 1) / BM);
  const int tiles = n_tiles * m_tiles * p.nb1 * p.nb2;
  const int num_kb = (int)((p.K + BK - 1) / BK);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    if constexpr (EPI != EPI_GENERIC) tma_prefetch_desc(&tma_c);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 128);  // every thread of the consuming warpgroup arrives once its wgmma group has read the slot
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (tid == 0) {
      int it = 0;  // k-blocks issued by this CTA, over all its tiles
      for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        const TileIdx ti = tile_idx(t, n_tiles, m_tiles, p.nb1);
        const int az1 = p.a_bcast1 ? 0 : ti.z1, az2 = p.a_bcast2 ? 0 : ti.z2;
        const int bz1 = p.b_bcast1 ? 0 : ti.z1, bz2 = p.b_bcast2 ? 0 : ti.z2;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
          mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
          tma_load_4d(smem_a + s * Cfg::A_BYTES, &tma_a, &full_bar[s], kb * BK, ti.m_tile * BM, az1, az2);
          tma_load_4d(smem_b + s * Cfg::B_BYTES, &tma_b, &full_bar[s], kb * BK, ti.n_tile * BN, bz1, bz2);
        }
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int g = wg - 1;
  const int my_tiles = (int)blockIdx.x < tiles ? (tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  float gate_s = 1.f;
  if (EPI == EPI_GENERIC && p.gate_mode == MQDET_VEC_SCALAR) gate_s = p.gate_tanh ? tanhf(p.gate[0]) : p.gate[0];
  const uint32_t stage_c = smem_u32(smem_c + g * Cfg::EPI_BYTES);
  const int fr = wg_row(tid, 0), fc = wg_col(tid, 0);  // fragment row / column of acc[.][0]

  for (int lt = g; lt < my_tiles; lt += 2) {
    const TileIdx ti = tile_idx(blockIdx.x + lt * gridDim.x, n_tiles, m_tiles, p.nb1);
    const int z1 = ti.z1, z2 = ti.z2;
    const long row0 = (long)ti.m_tile * BM, col0 = (long)ti.n_tile * BN;

    // per-column bias of the thread's BN / 4 columns, loaded once per tile (the loads retire under the main loop; the
    // residual variant, whose residual needs the registers, loads each pass's bias next to its residual)
    constexpr bool HAS_BIAS = EPI == EPI_BIAS_F16 || EPI == EPI_BIAS_GELU_F16 || EPI == EPI_BIAS_RES_F32;
    const float* bp = p.bias + z1 * p.bias_b1 + z2 * p.bias_b2;
    float bv[BN / 4];
    if constexpr (HAS_BIAS && EPI != EPI_BIAS_RES_F32) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const long col = col0 + 8 * j + fc + e;
          bv[2 * j + e] = col < p.N ? __ldg(bp + col) : 0.f;
        }
    }

    float acc[2][BN / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
    if (lt > 0) named_bar_sync(3 + g, 256);  // the other warpgroup's MMA of tile lt - 1 has retired
    int it = lt * num_kb;
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
      const int s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1);
      const uint32_t a_addr = smem_u32(smem_a + s * Cfg::A_BYTES);
      const uint32_t b_addr = smem_u32(smem_b + s * Cfg::B_BYTES);
      wgmma_fence_acc(acc[0]);
      wgmma_fence_acc(acc[1]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t db = wg_desc_k_sw128(b_addr + k * 32);
        wgmma_tile<BN>(acc[0], wg_desc_k_sw128(a_addr + k * 32), db);
        wgmma_tile<BN>(acc[1], wg_desc_k_sw128(a_addr + 64 * 128 + k * 32), db);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's group has retired: its slot may be refilled
      wgmma_fence_acc(acc[0]);
      wgmma_fence_acc(acc[1]);
      if (kb > 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc[0]);
    wgmma_fence_acc(acc[1]);
    mbar_arrive(&empty_bar[(it - 1) % STAGES]);       // the tile's last slot: the producer is already filling the next tile's
    if (lt + 1 < my_tiles) named_bar_arrive(3 + (g ^ 1), 256);  // the other warpgroup's turn

    if constexpr (EPI != EPI_GENERIC) {
      // ---- specialised epilogue: fragments -> the op -> swizzled staging in the output dtype -> TMA store (clipped at the
      // M / N edges by the TMA unit).  The epilogue arithmetic and its order are epi_one's, so the results are bit-identical
      // to the generic path's.
      constexpr int ES = Cfg::ES, JP = Cfg::PASS_COLS / 8;  // 8-column fragment groups per pass
#pragma unroll
      for (int ps = 0; ps < Cfg::PASSES; ++ps) {
        if constexpr (EPI == EPI_BIAS_RES_F32) {
#pragma unroll
          for (int jj = 0; jj < JP; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int j = ps * JP + jj;
              const long col = col0 + 8 * j + fc + e;
              bv[2 * j + e] = col < p.N ? __ldg(bp + col) : 0.f;
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float2 rv[JP][2];
          if constexpr (EPI == EPI_BIAS_RES_F32) {  // issued before the staging wait: the loads overlap it
            const float* rp = reinterpret_cast<const float*>(p.R) + z1 * p.r_b1 + z2 * p.r_b2;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const long row = row0 + 64 * h + fr + 8 * q;
#pragma unroll
              for (int jj = 0; jj < JP; ++jj) {
                const long col = col0 + ps * Cfg::PASS_COLS + 8 * jj + fc;  // even; N is even on this path
                rv[jj][q] = (row < p.M && col < p.N) ? __ldg(reinterpret_cast<const float2*>(rp + row * p.ldr + col))
                                                     : make_float2(0.f, 0.f);
              }
            }
          }
          if (h == 0) {
            if (tid == 0) tma_store_wait_read_all();  // the staging's previous store has been read out
            named_bar_sync(1 + g, 128);
          }
#pragma unroll
          for (int jj = 0; jj < JP; ++jj) {
            const int j = ps * JP + jj;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              float v0 = acc[h][4 * j + 2 * q], v1 = acc[h][4 * j + 2 * q + 1];
              if constexpr (HAS_BIAS) {
                v0 = v0 + bv[2 * j];
                v1 = v1 + bv[2 * j + 1];
              }
              if constexpr (EPI == EPI_BIAS_GELU_F16) {
                v0 = gelu_erf(v0);
                v1 = gelu_erf(v1);
              }
              const uint32_t addr = box_addr<ES>(stage_c, 64 * h + fr + 8 * q, 8 * jj + fc);
              if constexpr (EPI == EPI_BIAS_RES_F32)
                sts64f(addr, v0 + rv[jj][q].x, v1 + rv[jj][q].y);
              else
                sts32(addr, pack_half2(v0, v1));
            }
          }
        }
        fence_proxy_async();  // the staging writes are visible to the TMA unit
        named_bar_sync(1 + g, 128);
        if (tid == 0) {
#pragma unroll
          for (int b = 0; b < Cfg::BOXES; ++b) {
            const long c = col0 + ps * Cfg::PASS_COLS + b * Cfg::BOX_COLS;
            if (c < p.N) tma_store_4d(&tma_c, reinterpret_cast<const void*>(smem_c + g * Cfg::EPI_BYTES + b * BM * 128),
                                      (int)c, (int)row0, z1, z2);
          }
          tma_store_commit();
        }
      }
    } else {
      // ---- generic epilogue, one 64-row half at a time: fragments -> fp32 staging -> rows walked by consecutive threads
      // (coalesced residual loads and stores).  The per-element epilogue is not unrolled over the fragments: 64 inlined
      // copies of it (erff, tanhf, every option's branch) made the kernel's code far larger than the instruction cache.
      constexpr int TPR = BN / 2, RPI = 128 / TPR, U = 4;  // threads per row (two columns each), rows per pass, passes per batch
      const int cc = 2 * (tid % TPR);
      const long col = col0 + cc;
      const bool two = col + 1 < p.N;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        named_bar_sync(1 + g, 128);  // the previous half's staging reads are done
        if (h == 0) {
#pragma unroll
          for (int i = 0; i < BN / 2; i += 2)
            sts64f(stage_c + (wg_row(tid, i) * Cfg::PITCH + wg_col(tid, i)) * 4, acc[0][i], acc[0][i + 1]);
        } else {
#pragma unroll
          for (int i = 0; i < BN / 2; i += 2)
            sts64f(stage_c + (wg_row(tid, i) * Cfg::PITCH + wg_col(tid, i)) * 4, acc[1][i], acc[1][i + 1]);
        }
        named_bar_sync(1 + g, 128);
        const long rowh = row0 + 64 * h;
        if (col >= p.N) continue;
#pragma unroll 1
        for (int r0 = tid / TPR; r0 < 64; r0 += RPI * U) {
          float2 a[U], rv[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {  // every load of the batch is issued before the first store
            const int r = r0 + u * RPI;
            const long row = rowh + r;
            a[u] = lds64f(stage_c + (r * Cfg::PITCH + cc) * 4);
            rv[u] = make_float2(0.f, 0.f);
            if (p.R && row < p.M) {
              rv[u].x = ld_residual(p, row, col, z1, z2);
              if (two) rv[u].y = ld_residual(p, row, col + 1, z1, z2);
            }
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const long row = rowh + r0 + u * RPI;
            if (row >= p.M) break;
            float v0 = epi_pre(p, a[u].x, row, col, z1, z2, gate_s);
            if (p.R) v0 += rv[u].x;
            if (two) {
              float v1 = epi_pre(p, a[u].y, row, col + 1, z1, z2, gate_s);
              if (p.R) v1 += rv[u].y;
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
      }
    }
  }
  if constexpr (EPI != EPI_GENERIC)
    if (tid == 0) tma_store_wait_all();  // the staging stays allocated until the last store has completed
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
// The specialised epilogue that computes exactly what the generic one would for these arguments, or EPI_GENERIC.  The
// specialised kernels store through a TMA map, so C's base must be 16-byte aligned and its row / batch strides multiples of
// 16 bytes.
static int pick_epi(const GemmP& p) {
  const long es = p.c_dtype == MQDET_F32 ? 4 : 2;
  const bool tma_c = (reinterpret_cast<uintptr_t>(p.C) % 16) == 0 && (p.ldc * es) % 16 == 0 &&
                     (p.nb1 == 1 || (p.c_b1 > 0 && (p.c_b1 * es) % 16 == 0)) &&
                     (p.nb2 == 1 || (p.c_b2 > 0 && (p.c_b2 * es) % 16 == 0));
  if (!tma_c || p.alpha != 1.f || p.clamp > 0.f || p.gate_mode != MQDET_VEC_NONE) return EPI_GENERIC;
  if (p.bias_mode == MQDET_VEC_NONE)
    return (p.act == MQDET_ACT_NONE && !p.R && p.c_dtype == MQDET_F16) ? EPI_NONE_F16 : EPI_GENERIC;
  if (p.bias_mode != MQDET_VEC_PER_COL) return EPI_GENERIC;
  if (!p.R && p.c_dtype == MQDET_F16) {
    if (p.act == MQDET_ACT_NONE) return EPI_BIAS_F16;
    if (p.act == MQDET_ACT_GELU) return EPI_BIAS_GELU_F16;
    return EPI_GENERIC;
  }
  // fp32 residual read as 8-byte column pairs
  if (p.R && p.r_dtype == MQDET_F32 && p.c_dtype == MQDET_F32 && p.act == MQDET_ACT_NONE && p.N % 2 == 0 &&
      (reinterpret_cast<uintptr_t>(p.R) % 8) == 0 && p.ldr % 2 == 0 && p.r_b1 % 2 == 0 && p.r_b2 % 2 == 0)
    return EPI_BIAS_RES_F32;
  return EPI_GENERIC;
}

// make_operand_map / make_store_map / num_sms / ensure_dyn_smem: capi.cu (shared with the other TMA kernels; tensor maps are
// cached)
template <int BN, int STAGES, int EPI>
static int launch_wg(const GemmP& p0, bool persistent, cudaStream_t st) {
  using Cfg = WgCfg<BN, STAGES, EPI>;
  GemmP p = p0;
  CUtensorMap ma, mb, mc;
  int rc = make_operand_map(&ma, p.A, p.M, p.K, p.lda, p.nb1, p.a_b1, p.nb2, p.a_b2, BM, &p.a_bcast1, &p.a_bcast2);
  if (rc) return rc;
  rc = make_operand_map(&mb, p.B, p.N, p.K, p.ldb, p.nb1, p.b_b1, p.nb2, p.b_b2, BN, &p.b_bcast1, &p.b_bcast2);
  if (rc) return rc;
  if constexpr (EPI != EPI_GENERIC) {
    rc = make_store_map(&mc, p.C, p.c_dtype, p.M, p.N, p.ldc, p.nb1, p.c_b1, p.nb2, p.c_b2);
    if (rc) return rc;
  } else {
    memset(&mc, 0, sizeof(mc));
    const long al = p.c_dtype == MQDET_F16 ? 2 : 1;  // pair stores: 4-byte (fp16) / 8-byte (fp32) aligned
    p.vec2 = (p.ldc % 2 == 0) && (p.nb1 == 1 || p.c_b1 % 2 == 0) && (p.nb2 == 1 || p.c_b2 % 2 == 0) &&
             (reinterpret_cast<uintptr_t>(p.C) % (4 * (3 - al))) == 0;
  }
  rc = ensure_dyn_smem(reinterpret_cast<const void*>(&gemm_wg_kernel<BN, STAGES, EPI>), Cfg::SMEM_BYTES);
  if (rc) return rc;
  const long tiles = (long)cdiv(p.N, BN) * cdiv(p.M, BM) * p.nb1 * p.nb2;
  MQ_REQUIRE(tiles < (1l << 31), "gemm: %ld tiles", tiles);
  const int grid = persistent ? (int)(tiles < num_sms() ? tiles : num_sms()) : (int)tiles;
  gemm_wg_kernel<BN, STAGES, EPI><<<grid, 384, Cfg::SMEM_BYTES, st>>>(ma, mb, mc, p);
  return check_launch("gemm_wg_kernel");
}

template <int BN, int STAGES>
static int launch_wg_epi(const GemmP& p, bool persistent, cudaStream_t st) {
  switch (pick_epi(p)) {
    case EPI_NONE_F16: return launch_wg<BN, STAGES, EPI_NONE_F16>(p, persistent, st);
    case EPI_BIAS_F16: return launch_wg<BN, STAGES, EPI_BIAS_F16>(p, persistent, st);
    case EPI_BIAS_GELU_F16: return launch_wg<BN, STAGES, EPI_BIAS_GELU_F16>(p, persistent, st);
    case EPI_BIAS_RES_F32: return launch_wg<BN, STAGES, EPI_BIAS_RES_F32>(p, persistent, st);
    default: return launch_wg<BN, STAGES, EPI_GENERIC>(p, persistent, st);
  }
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
  const bool persistent = impl == MQDET_GEMM_IMPL_TC;
  if (p.N > 64 && tiles128 >= num_sms()) return launch_wg_epi<128, 4>(p, persistent, st);
  return launch_wg_epi<64, 6>(p, persistent, st);
}
