// mqdet_b200 — DyConv's DCNv2 3x3 convolutions as ONE implicit GEMM on the sm_90a tensor cores (no column matrix in HBM).
//
// Reference: maskrcnn_benchmark/modeling/rpn/vldyhead.py DyConv.forward :205-247 (three ModulatedDeformConv per layer);
//            maskrcnn_benchmark/csrc/cuda/deform_conv_kernel_cuda.cu :473-505 (bilinear), :578-641 (modulated im2col),
//            deform_conv_cuda.cu modulated_deform_conv_cuda_forward (im2col + GEMM per image).
//
//   y_j[rows_j, 256] = A_j[rows_j, 2304] * W_j[256, 2304]^T + bias_j        (k = tap*256 + c; j = one of the three branches)
//
// A_j is the bilinearly sampled, mask-modulated column matrix of dyhead.cu's dcn_cols_kernel — here it only ever exists as
// 64x64 fp16 tiles in shared memory.  Persistent, one CTA (384 threads) per SM walks the 64-row tiles of ALL jobs of the launch:
//   * warps 8-11 (gather): per tile, every (pixel, tap) gets ONE sampling record in shared memory (four corner offsets, four
//     corner weights with the modulation mask folded in; 18 KB); then, per k-block (tap, 64 channels), two threads per pixel
//     fetch 64 contiguous bytes of each corner row (four 128-bit loads), blend in fp32, round once to fp16 and store straight
//     into the 128B-swizzled K-major A stage; the loads of k-block kb+1 are issued before k-block kb is stored;
//   * warp 0: the [256 x 64] weight tile of the k-block by TMA;
//   * warps 4-7 (one warpgroup): four wgmma.m64n256k16 per k-block, fp32 accumulator in registers (128 per thread), then
//     +bias -> fp16 -> global stores straight from the accumulator fragments.
// 64-row tiles keep the 64 x 256 accumulator in one warpgroup's registers next to the gather warps.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int DC_BM = 64, DC_BN = 256, DC_BK = 64, DC_C = 256, DC_TAPS = 9;
constexpr int DC_STAGES = 4;
constexpr int DC_A_BYTES = DC_BM * DC_BK * 2;  // 8 KB
constexpr int DC_B_BYTES = DC_BN * DC_BK * 2;  // 32 KB
constexpr int DC_KB = DC_TAPS * DC_C / DC_BK;  // 36 k-blocks: tap = kb / 4, channels (kb % 4) * 64 ..
constexpr int DC_GATHER_WARPS = 4;
constexpr int DC_GATHER_THREADS = DC_GATHER_WARPS * 32;  // two per pixel
constexpr int DC_THREADS = 256 + DC_GATHER_THREADS;      // warp 0 TMA, warps 4-7 MMA + epilogue, warps 8-11 gather
constexpr int DC_COORD_BYTES = DC_TAPS * DC_BM * 32;     // per (tap, row): 4 corner offsets + 4 corner weights
constexpr int DC_SMEM_BYTES = DC_STAGES * (DC_A_BYTES + DC_B_BYTES) + DC_COORD_BYTES + 1024 /*align*/ + 256 /*barriers*/ +
                              DC_BN * 4 /*bias row*/;
static_assert(DC_SMEM_BYTES <= 232448, "dcn_conv: shared memory budget");

struct DcnP {
  CUtensorMap map_w[MQDET_DCN_MAX_JOBS];  // weights  [256][2304] fp16, box 64 x 256
  __half* y[MQDET_DCN_MAX_JOBS];          // outputs  [rows][256]  fp16
  const __half* x;
  const float* om;
  const float* bias[MQDET_DCN_MAX_JOBS];
  long rows[MQDET_DCN_MAX_JOBS];
  int rows_per_img[MQDET_DCN_MAX_JOBS];
  int branch[MQDET_DCN_MAX_JOBS];
  int tile_begin[MQDET_DCN_MAX_JOBS + 1];
  int njobs, om_ld, N;
  LevelTable lt;
};

__device__ __forceinline__ uint4 lds128u(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

// (w1 v1 + w2 v2 + w3 v3 + w4 v4) of 8 fp16 channels, fp32 math, rounded once to fp16.
__device__ __forceinline__ uint4 blend8(const uint4& v1, const uint4& v2, const uint4& v3, const uint4& v4, float w1, float w2,
                                        float w3, float w4) {
  const __half2* h1 = reinterpret_cast<const __half2*>(&v1);
  const __half2* h2 = reinterpret_cast<const __half2*>(&v2);
  const __half2* h3 = reinterpret_cast<const __half2*>(&v3);
  const __half2* h4 = reinterpret_cast<const __half2*>(&v4);
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 a = __half22float2(h1[i]), b = __half22float2(h2[i]), c = __half22float2(h3[i]), d = __half22float2(h4[i]);
    float s0 = w1 * a.x, s1 = w1 * a.y;
    ffma2(s0, s1, b.x, b.y, w2, s0, s1);
    ffma2(s0, s1, c.x, c.y, w3, s0, s1);
    ffma2(s0, s1, d.x, d.y, w4, s0, s1);
    o[i] = pack_half2(s0, s1);
  }
  return make_uint4(o[0], o[1], o[2], o[3]);
}

__global__ void __launch_bounds__(DC_THREADS, 1) dcn_conv_kernel(const __grid_constant__ DcnP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + DC_STAGES * DC_A_BYTES;
  uint8_t* coords = smem_b + DC_STAGES * DC_B_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(coords + DC_COORD_BYTES);
  uint64_t* a_full = bars;                       // [S] one arrival per gather warp
  uint64_t* b_full = bars + DC_STAGES;           // [S] TMA bytes of the weight tile
  uint64_t* empty = bars + 2 * DC_STAGES;        // [S] every MMA thread: the stage's wgmma group has read it
  float* s_bias = reinterpret_cast<float*>(bars + 32);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_tiles = p.tile_begin[p.njobs];

  if (threadIdx.x == 0) {
    for (int j = 0; j < p.njobs; ++j) tma_prefetch_desc(&p.map_w[j]);
    for (int s = 0; s < DC_STAGES; ++s) {
      mbar_init(&a_full[s], DC_GATHER_WARPS);
      mbar_init(&b_full[s], 1);
      mbar_init(&empty[s], 128);
    }
    fence_mbar_init();
  }
  __syncthreads();

  auto job_of = [&](int tile) {
    int j = 0;
    while (j + 1 < p.njobs && tile >= p.tile_begin[j + 1]) ++j;
    return j;
  };

  if (warp == 0) {
    // ---- weight tiles by TMA ------------------------------------------------------------------------------------------
    if (lane == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int j = job_of(tile);
        for (int kb = 0; kb < DC_KB; ++kb, ++it) {
          const int s = it % DC_STAGES;
          mbar_wait(&empty[s], ((it / DC_STAGES) & 1) ^ 1);
          mbar_expect_tx(&b_full[s], DC_B_BYTES);
          tma_load_4d(smem_b + s * DC_B_BYTES, &p.map_w[j], &b_full[s], kb * DC_BK, 0, 0, 0);
        }
      }
    }
  } else if (warp >= 4 && warp < 8) {
    // ---- MMA + epilogue: registers -> (+bias) -> fp16 -> global ---------------------------------------------------------
    const int tid = threadIdx.x - 128;
    uint32_t it = 0;
    int cur_job = -1;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int j = job_of(tile);
      if (j != cur_job) {  // uniform over the 128 MMA threads
        asm volatile("bar.sync 1, 128;" ::: "memory");
        s_bias[tid] = p.bias[j] ? p.bias[j][tid] : 0.f;
        s_bias[tid + 128] = p.bias[j] ? p.bias[j][tid + 128] : 0.f;
        cur_job = j;
        asm volatile("bar.sync 1, 128;" ::: "memory");
      }
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < DC_KB; ++kb, ++it) {
        const int s = it % DC_STAGES;
        const uint32_t ph = (it / DC_STAGES) & 1;
        mbar_wait(&b_full[s], ph);
        mbar_wait(&a_full[s], ph);
        const uint32_t a_addr = smem_u32(smem_a + s * DC_A_BYTES);
        const uint32_t b_addr = smem_u32(smem_b + s * DC_B_BYTES);
        wgmma_fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < DC_BK / 16; ++k)
          wgmma_ss_m64n256_kk(acc, wg_desc_k_sw128(a_addr + k * 32), wg_desc_k_sw128(b_addr + k * 32), 1);
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_fence_acc(acc);
        if (kb > 0) mbar_arrive(&empty[(it - 1) % DC_STAGES]);
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      mbar_arrive(&empty[(it - 1) % DC_STAGES]);
      const long row0 = (long)(tile - p.tile_begin[j]) * DC_BM;
      __half* const y = p.y[j];
#pragma unroll
      for (int i = 0; i < 128; i += 2) {
        const long row = row0 + wg_row(tid, i);
        const int col = wg_col(tid, i);
        if (row < p.rows[j])
          *reinterpret_cast<__half2*>(y + row * DC_BN + col) = __floats2half2_rn(acc[i] + s_bias[col], acc[i + 1] + s_bias[col + 1]);
      }
    }
  } else if (warp >= 8) {
    // ---- gather: 2 threads per output pixel, 4 x 8 channels each per k-block -------------------------------------------
    const int pt = threadIdx.x - 256, rl = pt >> 1, q = pt & 1;
    const int sw = rl & 7;
    // thread q of a row owns the adjacent 16-byte chunks 4q .. 4q+3 of the 128-byte swizzled row
    const uint32_t a_row = smem_u32(smem_a) + rl * 128;
    const uint32_t my_coords = smem_u32(coords) + rl * 32;
    const LevelTable& L = p.lt;
    const __half* const xa = p.x + q * 32;
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int j = job_of(tile);
      // -- sampling records of the tile: thread pt works out (row pt % 64, taps pt / 64 + 2 i): four corner offsets
      //    (elements from x) and four corner weights with the modulation mask folded in
      {
        const int branch = p.branch[j];
        const int row = pt & (DC_BM - 1);
        const long r = (long)(tile - p.tile_begin[j]) * DC_BM + row;
        const bool valid = r < p.rows[j];
        int b = 0, qq = 0;
        if (valid) {
          b = (int)(r / p.rows_per_img[j]);
          qq = (int)(r - (long)b * p.rows_per_img[j]);
        }
        int lo, li, Ho, Wo, stride;
        if (branch == 1) {
          int l = 0;
          while (l + 1 < L.n && qq >= L.off[l + 1]) ++l;
          qq -= L.off[l];
          lo = l; li = l; Ho = L.H[l]; Wo = L.W[l]; stride = 1;
        } else {
          int l = 1;
          const int base = L.off[1];
          while (l + 1 < L.n && qq + base >= L.off[l + 1]) ++l;
          qq -= L.off[l] - base;
          Ho = L.H[l]; Wo = L.W[l];
          if (branch == 2) { lo = l; li = l - 1; stride = 2; }
          else { lo = l - 1; li = l; stride = 1; }
        }
        const int ho = qq / Wo, wo = qq - ho * Wo;
        const int Hi = L.H[li], Wi = L.W[li];
        const int HWl = L.H[lo] * L.W[lo], HWo = Ho * Wo, pix = ho * Wo + wo;
        const float* omb = p.om ? p.om + ((long)b * p.N + L.off[lo]) * p.om_ld : nullptr;
        const int xrow0 = b * p.N + L.off[li];
        for (int tap = pt / DC_BM; tap < DC_TAPS; tap += DC_GATHER_THREADS / DC_BM) {
          float off_h = 0.f, off_w = 0.f, m = 1.f;
          if (omb && valid) {
            // flat NCHW index c*HWo + pix re-read through the strides of the level the record was produced at
            // (deform_conv_kernel_cuda.cu:605-618; identical to dcn_cols_kernel)
            const int f0 = (2 * tap) * HWo + pix, f1 = f0 + HWo, f2 = tap * HWo + pix;
            off_h = __ldg(omb + (long)(f0 % HWl) * p.om_ld + f0 / HWl);
            off_w = __ldg(omb + (long)(f1 % HWl) * p.om_ld + f1 / HWl);
            const float ml = __ldg(omb + (long)(f2 % HWl) * p.om_ld + 18 + f2 / HWl);
            m = 1.f / (1.f + expf(-ml));
          }
          const float h_im = (float)(ho * stride - 1 + tap / 3) + off_h;
          const float w_im = (float)(wo * stride - 1 + tap % 3) + off_w;
          const bool inside = valid && h_im > -1.f && w_im > -1.f && h_im < (float)Hi && w_im < (float)Wi;
          const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
          const int h_high = h_low + 1, w_high = w_low + 1;
          const float lh = h_im - h_low, lw = w_im - w_low, hh = 1.f - lh, hw = 1.f - lw;
          const bool hl_ok = inside && h_low >= 0, hh_ok = inside && h_high <= Hi - 1;
          const bool wl_ok = w_low >= 0, wh_ok = w_high <= Wi - 1;
          const float w1 = (hl_ok && wl_ok) ? hh * hw * m : 0.f, w2 = (hl_ok && wh_ok) ? hh * lw * m : 0.f;
          const float w3 = (hh_ok && wl_ok) ? lh * hw * m : 0.f, w4 = (hh_ok && wh_ok) ? lh * lw * m : 0.f;
          // corner rows are always in-bounds (clamped); a zero weight removes an invalid corner
          const int hl = min(max(h_low, 0), Hi - 1), hh_i = min(max(h_high, 0), Hi - 1);
          const int wl = min(max(w_low, 0), Wi - 1), wh_i = min(max(w_high, 0), Wi - 1);
          const uint32_t rec = smem_u32(coords) + (uint32_t)((tap * DC_BM + row) * 32);
          sts128(rec, (uint32_t)((xrow0 + hl * Wi + wl) * DC_C), (uint32_t)((xrow0 + hl * Wi + wh_i) * DC_C),
                 (uint32_t)((xrow0 + hh_i * Wi + wl) * DC_C), (uint32_t)((xrow0 + hh_i * Wi + wh_i) * DC_C));
          sts128(rec + 16, __float_as_uint(w1), __float_as_uint(w2), __float_as_uint(w3), __float_as_uint(w4));
        }
      }
      asm volatile("bar.sync 2, %0;" ::"n"(DC_GATHER_THREADS) : "memory");
      // -- 36 k-blocks (tap = kb / 4, channels (kb % 4) * 64 ..): the corner rows of k-block kb+1 are in flight while
      //    k-block kb is stored
      uint4 o = lds128u(my_coords);
      float4 w = lds128f(my_coords + 16);
      uint4 c[4][4];
      auto load = [&](int ch) {
        const uint32_t off[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
        for (int cr = 0; cr < 4; ++cr)
#pragma unroll
          for (int h = 0; h < 4; ++h) c[cr][h] = __ldg(reinterpret_cast<const uint4*>(xa + off[cr] + ch) + h);
      };
      load(0);
#pragma unroll 1
      for (int kb = 0; kb < DC_KB; ++kb, ++it) {
        const int s = it % DC_STAGES;
        const float4 wc = w;
        const int nk = kb + 1;
        if ((nk & 3) == 0 && nk < DC_KB) {  // next k-block starts a new tap
          const uint32_t rec = my_coords + (uint32_t)((nk >> 2) * DC_BM * 32);
          o = lds128u(rec);
          w = lds128f(rec + 16);
        }
        uint4 ob[4];
#pragma unroll
        for (int h = 0; h < 4; ++h) ob[h] = blend8(c[0][h], c[1][h], c[2][h], c[3][h], wc.x, wc.y, wc.z, wc.w);
        if (nk < DC_KB) load((nk & 3) * DC_BK);
        mbar_wait(&empty[s], ((it / DC_STAGES) & 1) ^ 1);
        const uint32_t dst = a_row + s * DC_A_BYTES;
#pragma unroll
        for (int h = 0; h < 4; ++h) sts128(dst + (uint32_t)(((4 * q + h) ^ sw) << 4), ob[h].x, ob[h].y, ob[h].z, ob[h].w);
        fence_proxy_async();  // generic-proxy writes -> visible to the tensor core (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(&a_full[s]);
      }
      asm volatile("bar.sync 2, %0;" ::"n"(DC_GATHER_THREADS) : "memory");  // every record of this tile has been read
    }
  }
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_dcn_conv(const void* x, const float* om, int64_t om_ld, const int32_t* level_hw, int64_t nlev, int64_t B,
                              int64_t C, int64_t njobs, const int32_t* branch, const void* const* weight,
                              const float* const* bias, void* const* y, void* stream) {
  MQ_REQUIRE(x && level_hw && branch && weight && bias && y, "dcn_conv: null pointer");
  MQ_REQUIRE(C == DC_C, "dcn_conv: C must be 256 (got %ld)", (long)C);
  MQ_REQUIRE(njobs >= 1 && njobs <= MQDET_DCN_MAX_JOBS, "dcn_conv: 1..%d jobs (got %ld)", MQDET_DCN_MAX_JOBS, (long)njobs);
  MQ_REQUIRE(B >= 1, "dcn_conv: empty batch");
  MQ_REQUIRE(((uintptr_t)x & 15) == 0, "dcn_conv: x must be 16-byte aligned (128-bit loads)");
  MQ_REQUIRE(om == nullptr || om_ld >= 27, "dcn_conv: om_ld must hold the 27 offset/mask channels");
  MQ_REQUIRE(nlev >= 1 && nlev <= MQDET_MAX_LEVELS, "dcn_conv: 1..%d levels", MQDET_MAX_LEVELS);
  DcnP q;
  memset(&q, 0, sizeof(q));
  const int N = fill_levels(&q.lt, level_hw, nlev);
  MQ_REQUIRE(N > 0, "dcn_conv: bad level table");
  MQ_REQUIRE((long)B * N * DC_C < (1L << 31), "dcn_conv: x has more than 2^31 elements (32-bit corner offsets)");
  q.x = (const __half*)x;
  q.om = om;
  q.om_ld = (int)om_ld;
  q.N = N;
  q.njobs = (int)njobs;
  int tiles = 0;
  for (int j = 0; j < njobs; ++j) {
    MQ_REQUIRE(branch[j] >= 0 && branch[j] <= 2, "dcn_conv: branch must be 0, 1 or 2");
    MQ_REQUIRE(branch[j] == 1 || nlev >= 2, "dcn_conv: branches 0/2 need at least two levels");
    MQ_REQUIRE(weight[j] && y[j], "dcn_conv: null weight / output of job %d", j);
    const long rpi = branch[j] == 1 ? N : N - q.lt.H[0] * q.lt.W[0];
    q.branch[j] = branch[j];
    q.rows_per_img[j] = (int)rpi;
    q.rows[j] = rpi * B;
    q.bias[j] = bias[j];
    q.tile_begin[j] = tiles;
    tiles += cdiv(q.rows[j], DC_BM);
    int bc1, bc2;
    int rc = make_operand_map(&q.map_w[j], weight[j], DC_BN, DC_TAPS * DC_C, DC_TAPS * DC_C, 1, 0, 1, 0, DC_BN, &bc1, &bc2);
    if (rc != MQDET_OK) return rc;
    q.y[j] = (__half*)y[j];
  }
  q.tile_begin[njobs] = tiles;
  int rc = ensure_dyn_smem((const void*)dcn_conv_kernel, DC_SMEM_BYTES);
  if (rc != MQDET_OK) return rc;
  const int grid = min(tiles, num_sms());
  dcn_conv_kernel<<<grid, DC_THREADS, DC_SMEM_BYTES, (cudaStream_t)stream>>>(q);
  return check_launch("dcn_conv_kernel");
}
