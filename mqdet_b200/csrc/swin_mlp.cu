// mqdet_b200 — the MLP half of a Swin block in one sm_90a kernel, for the narrow stages (C = 96 / 192, hidden 4C):
//
//   out[r] = x[r] + fc2(GELU(fc1(LN2(x[r]))))          x, out: fp32 [rows][C]; fc1 / fc2: fp16 nn.Linear weights, fp32 biases
//
// It computes exactly what the three-launch chain computes (layernorm_reg_rows_kernel -> fc1 GEMM with the bias + GELU epilogue
// -> fc2 GEMM with the bias + fp32 residual epilogue) without the fp16 LN output and the 4C-wide hidden activation ever
// leaving the SM: only the fp32 residual stream goes in and out.
//
// Persistent, one CTA per SM on a static schedule of 64-row tiles (no device-side counters: a captured graph replays as is).
//   warpgroup 0    : TMA producer — one thread streams 64-hidden-column chunks of W1 ([64][C]) and W2 ([C][64]) through a
//                                   STAGES-deep ring (128B swizzle).  At C = 96 the ring holds all six chunks, so the weights are
//                                   loaded once and stay resident; at C = 192 (12 chunks, 48 KB each) three stages stream them
//                                   from L2.  setmaxnreg hands the producer's registers to the consumers.
//   warpgroups 1-2 : consumers    — each takes every other tile of the CTA (both walk the same chunk sequence, so each ring slot
//                                   is released by both).  Per tile:
//       LN2 prologue: a warp per 16 rows reads the fp32 rows and normalises them with layernorm_reg_rows_kernel's arithmetic
//                     (lane owns columns lane + 32 i, sequential per-lane sums, xor butterfly, two-pass mean / biased variance,
//                     rsqrtf(var / D + eps)), writing fp16 straight into the 128B-swizzled A tile.
//       per chunk j:  fc1 = wgmma.m64n64 (A tile x W1 chunk, k16 steps in increasing k) -> + bias1 -> gelu_erf -> fp16 fragments,
//                     which are fc2's register A operand (wgmma.m64nC ... rs over the W2 chunk); the 64 x C fp32 fc2 accumulator
//                     stays live across the chunks, which run in increasing hidden order: the fc2 k16 chain is the GEMM's own.
//       epilogue:     (acc + bias2) + x in fp32 (the GEMM's bias + residual order; x re-read, from L2) -> swizzled 64-row boxes
//                     -> TMA store (make_store_map; the unit clips ragged rows).
//   The two consumer warpgroups run independently, so one's erff GELU and LN issue under the other's wgmma.
//
// Shared memory: ring (C = 96: 6 x 28 KB; C = 192: 3 x 48 KB) + per consumer warpgroup one 24 KB buffer that holds the fp16 A tile
// and, once the tile's MMAs have retired, the fp32 output staging (C = 192: two passes of 96 columns).  Keeping the fp32 input
// rows for the residual as well (24 / 48 KB per warpgroup) would exceed the 227 KB limit at C = 96 and leave a single weight stage
// at C = 192, so the epilogue re-reads them; the tile was read moments before and is served by L2.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int TM = 64;  // rows per tile: one m64 wgmma row per consumer warpgroup
constexpr int NC = 64;  // hidden columns per chunk

template <int C>
struct MlpCfg {
  static constexpr int NCH = 4 * C / NC;                // chunks: 6 / 12
  static constexpr int KB1 = (C + 63) / 64;             // fc1 k-blocks of 64 (TMA zero-fills past C; only C / 16 k16 steps run)
  static constexpr int W1_BYTES = NC * 128 * KB1;       // [kb][64 hidden][64 c]
  static constexpr int W2_BYTES = C * 128;              // [C][64 hidden]
  static constexpr int STAGE_BYTES = W1_BYTES + W2_BYTES;
  static constexpr int STAGES = C == 96 ? NCH : 3;
  static constexpr bool RESIDENT = STAGES >= NCH;       // every chunk has its own slot: loaded once, never released
  static constexpr int A_BYTES = TM * 128 * KB1;        // [kb][64 rows][64 c] fp16
  static constexpr int PASSES = C == 96 ? 1 : 2;
  static constexpr int PASS_COLS = C / PASSES;          // 96
  static constexpr int BOXES = PASS_COLS / 32;          // fp32 store boxes of 32 columns x 64 rows
  static constexpr int OUT_BYTES = TM * PASS_COLS * 4;
  static constexpr int WG_BYTES = A_BYTES > OUT_BYTES ? A_BYTES : OUT_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * WG_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(W1_BYTES % 1024 == 0 && W2_BYTES % 1024 == 0 && WG_BYTES % 1024 == 0, "swizzled tiles need 1024-byte alignment");
  static_assert(SMEM_BYTES <= 232448, "shared memory");
};

struct MlpP {
  const float* x;
  long rows;
  const float* ln_w;
  const float* ln_b;
  float eps;
  const float* b1;
  const float* b2;
};

// byte address of fp16 element (r, c) of the A tile: 64-column k-blocks of 64 rows x 128 B, 16-byte chunks XOR-swizzled by r % 8
__device__ __forceinline__ uint32_t a_addr(uint32_t base, int r, int c) {
  const int byte = (c & 63) * 2;
  return base + (c >> 6) * (TM * 128) + r * 128 + ((((byte >> 4) & 7) ^ (r & 7)) << 4) + (byte & 15);
}
// byte address of fp32 element (r, c) of the output staging: 32-column boxes of 64 rows x 128 B, same swizzle
__device__ __forceinline__ uint32_t out_addr(uint32_t base, int r, int c) {
  const int byte = c * 4;
  return base + (byte >> 7) * (TM * 128) + r * 128 + ((((byte >> 4) & 7) ^ (r & 7)) << 4) + (byte & 15);
}

template <int C>
__device__ __forceinline__ void wgmma_fc2(float (&d)[C / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (C == 96)
    wgmma_rs_m64n96_kk(d, a, db, 1);
  else
    wgmma_rs_m64n192_kk(d, a, db, 1);
}

// fc1 of one chunk: acc1 = A tile x W1 chunk, k16 steps in increasing k (the GEMM's chain), as one commit group
template <int C>
__device__ __forceinline__ void fc1_issue(float (&acc1)[NC / 2], uint32_t buf_a, uint32_t w1a) {
#pragma unroll
  for (int i = 0; i < NC / 2; ++i) acc1[i] = 0.f;
  wgmma_fence_acc(acc1);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < C / 16; ++k)
    wgmma_ss_m64n64_kk(acc1, wg_desc_k_sw128(buf_a + (k >> 2) * TM * 128 + (k & 3) * 32),
                       wg_desc_k_sw128(w1a + (k >> 2) * NC * 128 + (k & 3) * 32), 1);
  wgmma_commit();
}

// LN2 of the tile's 64 rows into the A tile: warp w normalises rows 16 w .. 16 w + 15, R rows at a time with all their loads
// issued first.  Per row this is layernorm_reg_rows_kernel's arithmetic, operation for operation.
template <int C>
__device__ __forceinline__ void ln_tile(const MlpP& p, long row0, uint32_t a_base, int warp, int lane, const float (&g)[C / 32],
                                        const float (&bt)[C / 32]) {
  constexpr int K = C / 32, D = C, R = 4;
#pragma unroll 1
  for (int rb = 0; rb < 16; rb += R) {
    float v[R][K];
    bool zr[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const long row = row0 + 16 * warp + rb + r;
      zr[r] = row >= p.rows;
#pragma unroll
      for (int i = 0; i < K; ++i) v[r][i] = zr[r] ? 0.f : __ldg(p.x + row * C + lane + 32 * i);
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
      const float rs = zr[r] ? rsqrtf(p.eps) : rsqrtf(rstd[r] / D + p.eps);
#pragma unroll
      for (int i = 0; i < K; ++i) {
        const float y = (v[r][i] - mean[r]) * rs * g[i] + bt[i];
        sts16(a_addr(a_base, 16 * warp + rb + r, lane + 32 * i), __float2half_rn(y));
      }
    }
  }
}

template <int C>
__global__ void __launch_bounds__(384, 1) swin_mlp_kernel(const __grid_constant__ CUtensorMap tma_w1,
                                                          const __grid_constant__ CUtensorMap tma_w2,
                                                          const __grid_constant__ CUtensorMap tma_out, const MlpP p) {
  using Cfg = MlpCfg<C>;
  constexpr int STAGES = Cfg::STAGES, NCH = Cfg::NCH;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem;
  uint8_t* wg_buf = smem + STAGES * Cfg::STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(wg_buf + 2 * Cfg::WG_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int tiles = (int)((p.rows + TM - 1) / TM);
  const int my_tiles = (int)blockIdx.x < tiles ? (tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const int rounds = (my_tiles + 1) / 2;  // round r: consumer warpgroup g takes the CTA's tile 2 r + g

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_w1);
    tma_prefetch_desc(&tma_w2);
    tma_prefetch_desc(&tma_out);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 256);  // both consumer warpgroups release every slot
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (tid == 0) {
      const int total = Cfg::RESIDENT ? NCH : rounds * NCH;
      for (int it = 0; it < total; ++it) {
        const int s = it % STAGES, j = it % NCH;
        if (!Cfg::RESIDENT) mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
        mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
        uint8_t* w1s = ring + s * Cfg::STAGE_BYTES;
#pragma unroll
        for (int kb = 0; kb < Cfg::KB1; ++kb) tma_load_4d(w1s + kb * NC * 128, &tma_w1, &full_bar[s], kb * 64, j * NC, 0, 0);
        tma_load_4d(w1s + Cfg::W1_BYTES, &tma_w2, &full_bar[s], j * NC, 0, 0, 0);
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int g = wg - 1, warp = tid >> 5, lane = tid & 31;
  const int fr = wg_row(tid, 0), fc = wg_col(tid, 0);  // fragment row / column of acc[.][0]
  uint8_t* buf = wg_buf + g * Cfg::WG_BYTES;
  const uint32_t buf_a = smem_u32(buf);
  float ln_g[C / 32], ln_b[C / 32];
#pragma unroll
  for (int i = 0; i < C / 32; ++i) {
    ln_g[i] = __ldg(p.ln_w + lane + 32 * i);
    ln_b[i] = __ldg(p.ln_b + lane + 32 * i);
  }

  for (int r = 0; r < rounds; ++r) {
    const int lt = 2 * r + g;
    if (lt >= my_tiles) {  // the other warpgroup's last tile: release this warpgroup's share of its ring slots
      if constexpr (!Cfg::RESIDENT) {
        for (int j = 0; j < NCH; ++j) {
          const int it = r * NCH + j;
          mbar_wait(&full_bar[it % STAGES], (it / STAGES) & 1);
          mbar_arrive(&empty_bar[it % STAGES]);
        }
      }
      continue;
    }
    const long row0 = (long)((int)blockIdx.x + lt * (int)gridDim.x) * TM;

    // the previous tile's output staging (which aliases the A tile) has been read out by the TMA unit
    if (tid == 0) tma_store_wait_read_all();
    named_bar_sync(1 + g, 128);
    ln_tile<C>(p, row0, buf_a, warp, lane, ln_g, ln_b);
    fence_proxy_async();  // the A tile's generic-proxy writes are visible to wgmma
    named_bar_sync(1 + g, 128);

    float acc2[C / 2];
#pragma unroll
    for (int i = 0; i < C / 2; ++i) acc2[i] = 0.f;
#pragma unroll 1
    for (int j = 0; j < NCH; ++j) {
      const int it = r * NCH + j, s = it % STAGES;
      float b1v[NC / 4];  // per-column bias of the thread's 16 hidden columns of this chunk
#pragma unroll
      for (int t = 0; t < NC / 8; ++t)
#pragma unroll
        for (int e = 0; e < 2; ++e) b1v[2 * t + e] = __ldg(p.b1 + j * NC + 8 * t + fc + e);
      mbar_wait(&full_bar[s], Cfg::RESIDENT ? 0u : (uint32_t)((it / STAGES) & 1));
      const uint32_t w1a = smem_u32(ring + s * Cfg::STAGE_BYTES), w2a = w1a + Cfg::W1_BYTES;
      float acc1[NC / 2];
      fc1_issue<C>(acc1, buf_a, w1a);
      wgmma_wait<0>();  // fc1 of chunk j and fc2 of chunk j - 1 have retired
      wgmma_fence_acc(acc1);
      wgmma_fence_acc(acc2);
      if (!Cfg::RESIDENT && j > 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);

      // bias + erf-GELU (the GEMM's EPI_BIAS_GELU_F16 order) -> fp16 A fragments of fc2: the layouts coincide
      uint32_t pa[NC / 16][4];
#pragma unroll
      for (int kk = 0; kk < NC / 16; ++kk)
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const int i = 8 * kk + 2 * h;
          const float v0 = gelu_erf(acc1[i] + b1v[2 * (i >> 2)]);
          const float v1 = gelu_erf(acc1[i + 1] + b1v[2 * (i >> 2) + 1]);
          pa[kk][h] = pack_half2(v0, v1);
        }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < NC / 16; ++kk) wgmma_fc2<C>(acc2, pa[kk], wg_desc_k_sw128(w2a + kk * 32));
      wgmma_commit();
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc2);
    if constexpr (!Cfg::RESIDENT) mbar_arrive(&empty_bar[(r * NCH + NCH - 1) % STAGES]);
    named_bar_sync(1 + g, 128);  // every warp's MMAs have read the A tile: the staging may overwrite it

    // ---- epilogue: (acc + bias2) + x -> swizzled fp32 boxes -> TMA store
    constexpr int JP = Cfg::PASS_COLS / 8;  // 8-column fragment groups per pass
#pragma unroll
    for (int ps = 0; ps < Cfg::PASSES; ++ps) {
      float bv[2 * JP];
      float2 rv[JP][2];
#pragma unroll
      for (int jj = 0; jj < JP; ++jj) {
        const int col = ps * Cfg::PASS_COLS + 8 * jj + fc;
        bv[2 * jj] = __ldg(p.b2 + col);
        bv[2 * jj + 1] = __ldg(p.b2 + col + 1);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const long row = row0 + fr + 8 * q;
          rv[jj][q] = row < p.rows ? __ldg(reinterpret_cast<const float2*>(p.x + row * C + col)) : make_float2(0.f, 0.f);
        }
      }
      if (ps > 0) {
        if (tid == 0) tma_store_wait_read_all();  // the previous pass's boxes have been read out
        named_bar_sync(1 + g, 128);
      }
#pragma unroll
      for (int jj = 0; jj < JP; ++jj) {
        const int j = ps * JP + jj;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const float v0 = acc2[4 * j + 2 * q] + bv[2 * jj], v1 = acc2[4 * j + 2 * q + 1] + bv[2 * jj + 1];
          sts64f(out_addr(buf_a, fr + 8 * q, 8 * jj + fc), v0 + rv[jj][q].x, v1 + rv[jj][q].y);
        }
      }
      fence_proxy_async();  // the staging writes are visible to the TMA unit
      named_bar_sync(1 + g, 128);
      if (tid == 0) {
#pragma unroll
        for (int b = 0; b < Cfg::BOXES; ++b)
          tma_store_4d(&tma_out, buf + b * TM * 128, ps * Cfg::PASS_COLS + b * 32, (int)row0, 0, 0);
        tma_store_commit();
      }
    }
  }
  if (tid == 0) tma_store_wait_all();  // the staging stays allocated until the last store has completed
}

template <int C>
static int launch_swin_mlp(const float* x, long rows, const float* ln_w, const float* ln_b, float eps, const void* w1, const float* b1,
           const void* w2, const float* b2, float* out, cudaStream_t st) {
  using Cfg = MlpCfg<C>;
  CUtensorMap m1, m2, mo;
  int bc1, bc2;
  int rc = make_operand_map(&m1, w1, 4 * C, C, C, 1, 0, 1, 0, NC, &bc1, &bc2);
  if (rc) return rc;
  rc = make_operand_map(&m2, w2, C, 4 * C, 4 * C, 1, 0, 1, 0, C, &bc1, &bc2);
  if (rc) return rc;
  rc = make_store_map(&mo, out, MQDET_F32, rows, C, C, 1, 0, 1, 0, TM);
  if (rc) return rc;
  rc = ensure_dyn_smem(reinterpret_cast<const void*>(&swin_mlp_kernel<C>), Cfg::SMEM_BYTES);
  if (rc) return rc;
  MlpP p;
  p.x = x;
  p.rows = rows;
  p.ln_w = ln_w;
  p.ln_b = ln_b;
  p.eps = eps;
  p.b1 = b1;
  p.b2 = b2;
  const long tiles = (rows + TM - 1) / TM;
  const int grid = (int)(tiles < num_sms() ? tiles : num_sms());
  swin_mlp_kernel<C><<<grid, 384, Cfg::SMEM_BYTES, st>>>(m1, m2, mo, p);
  return check_launch("swin_mlp_kernel");
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_swin_mlp_f16(const float* x, int64_t rows, int64_t C, const float* ln_w, const float* ln_b, float eps,
                                  const void* w1, const float* b1, const void* w2, const float* b2, float* out, void* stream) {
  MQ_REQUIRE(x && ln_w && ln_b && w1 && b1 && w2 && b2 && out, "swin_mlp: null pointer");
  MQ_REQUIRE(C == 96 || C == 192, "swin_mlp: C must be 96 or 192 (got %ld)", (long)C);
  MQ_REQUIRE(rows > 0 && rows < (1l << 31) / 64 * 64, "swin_mlp: bad rows %ld", (long)rows);
  MQ_REQUIRE(((uintptr_t)x % 16) == 0 && ((uintptr_t)out % 16) == 0 && ((uintptr_t)w1 % 16) == 0 && ((uintptr_t)w2 % 16) == 0,
             "swin_mlp: x, out, w1 and w2 must be 16-byte aligned");
  MQ_REQUIRE((const char*)out + rows * C * 4 <= (const char*)x || (const char*)x + rows * C * 4 <= (const char*)out,
             "swin_mlp: out must not overlap x");
  cudaStream_t st = (cudaStream_t)stream;
  if (C == 96) return launch_swin_mlp<96>(x, rows, ln_w, ln_b, eps, w1, b1, w2, b2, out, st);
  return launch_swin_mlp<192>(x, rows, ln_w, ln_b, eps, w1, b1, w2, b2, out, st);
}
