// mqdet_b200 — the bi-directional image <-> text attention of the VL fusion tower (BiMultiHeadAttention,
// maskrcnn_benchmark/utils/fuse_helper.py:218-303) as two wgmma kernels that never materialise the score matrix:
//
//   biattn_image_kernel : image -> text side.  Per 64 image tokens and head: S = Q K^T (fp32, registers) -> +-5e4 clamp ->
//                         column-max partials (for the text side) -> masked row softmax over the T tokens in the accumulator
//                         fragments -> P (fp16, registers: the A operand of the next wgmma) -> P . mT_h, summed over the heads
//                         -> v' = residual + gamma * (acc + bias).  Neither the scores nor the per-head context reach HBM.
//   biattn_text_kernel  : text -> image side (one CTA per (image, head, 64 text tokens), streams all image tokens):
//                         S^T recomputed on the tensor cores, exp(S^T - column max), P . V accumulated in registers.
//                         VN variant: V = the layer-normed image tokens themselves (read MN-major from the same [n x c] tile),
//                         the value projection is applied AFTER the token reduction (sum_n p[n] = 1), and the column sums are
//                         accumulated in-kernel, so the [B, E, N] value tensor of the image side is never built.
// Each CTA is one warpgroup; a 64-row tile keeps a 64 x 256 fp32 accumulator in its registers (128 per thread).  Operands arrive
// by TMA (128B swizzle) through a two-stage ring; accumulator fragment: row / column of element i of thread t = wg_row / wg_col.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int BM = 64;  // rows (text tokens / image tokens) per CTA
constexpr int BK = 64;  // 64 fp16 = 128 B = one swizzle row
constexpr int KB_BYTES = 64 * BK * 2;  // one [64 x 64] k-block

// A-operand fragment of k-step kk (16 columns) from a 64 x N accumulator fragment: the register layouts coincide
template <int R>
__device__ __forceinline__ void acc_to_a(const float (&e)[R], int kk, uint32_t (&a)[4]) {
  a[0] = pack_half2(e[8 * kk + 0], e[8 * kk + 1]);
  a[1] = pack_half2(e[8 * kk + 2], e[8 * kk + 3]);
  a[2] = pack_half2(e[8 * kk + 4], e[8 * kk + 5]);
  a[3] = pack_half2(e[8 * kk + 6], e[8 * kk + 7]);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// =====================================================================================================================
// Fused text -> image side of the bi-directional attention (BiMultiHeadAttention, fuse_helper.py:257-275, 289-291):
//     out[t, :] = sum_n softmax_n(clamp(k_t . q_n)) * Vv[n, :]        per (image, head), t = text token, n = image token
// One CTA per (z, 64 text tokens).  The transposed probabilities [T, N] never reach HBM.  Per step of 64 image tokens:
//     S^T   = K_tile (64 x 256, resident) . Q_step^T           16 wgmma 64x64x16
//     P     = exp(fp16(clamp(S^T)) - colmax_t)                  in the accumulator fragments -> fp16 A operand (registers)
//     O    += P . Vv_step                                        4 wgmma 64x256x16, O (64 x 256) in registers
//     out   = O / colsum_t  -> fp16
// colmax / colsum come from mqdet_colsoftmax_stats / mqdet_colstats_rowsoftmax over the SAME fp16 scores the image -> text
// side uses, so no online rescaling is needed.
// =====================================================================================================================
constexpr int BT_STEP = 64;  // image tokens per step
struct BtCfg {
  static constexpr int KT_BYTES = 4 * KB_BYTES;       // resident K tile: 4 k-blocks of [64 x 64]
  static constexpr int Q_BYTES = 4 * KB_BYTES;        // Q step [64 n x 256 d]
  static constexpr int V_BYTES = 256 * BT_STEP * 2;   // Vv^T tile [256 d x 64 n]  /  VN: image-token tile [64 n x 256 c]
  static constexpr int STAGE_BYTES = Q_BYTES + V_BYTES;
  static constexpr int SMEM_BYTES = KT_BYTES + 2 * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};
static_assert(BtCfg::SMEM_BYTES <= 232448, "biattn_text: dynamic shared memory above the 227 KB per-CTA limit");
struct BtP {
  const float* stat;  // [Z][2][T]: column max, 1 / column sum   (VN: [Z][T] column max only)
  float clamp;
  int nb1, T, N, n_steps;
  int k_bc1, k_bc2, q_bc1, q_bc2, v_bc1, v_bc2;  // 1 -> batch coordinate pinned to 0
  const float* rowbias;                           // VN: optional [Z][T * rb_ld] additive score bias per text token (folded q bias)
  int rb_ld;
  __half* out;                                    // [nb2][nb1][T][256]
  long o_ld, o_b1, o_b2;
};

template <bool VN>
__global__ void __launch_bounds__(128, 1) biattn_text_kernel(const __grid_constant__ CUtensorMap tma_k,
                                                             const __grid_constant__ CUtensorMap tma_q,
                                                             const __grid_constant__ CUtensorMap tma_v, const BtP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* kt = smem;
  uint8_t* ring = kt + BtCfg::KT_BYTES;  // 2 x [Q step | V step]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + 2 * BtCfg::STAGE_BYTES);
  uint64_t* kt_full = bars;
  uint64_t* full = bars + 1;  // [2]

  const int tid = threadIdx.x;
  const int mt = blockIdx.x, z = blockIdx.y;
  const int z1 = z % p.nb1, z2 = z / p.nb1;
  const int NS = p.n_steps;
  const int qz1 = p.q_bc1 ? 0 : z1, qz2 = p.q_bc2 ? 0 : z2, vz1 = p.v_bc1 ? 0 : z1, vz2 = p.v_bc2 ? 0 : z2;

  auto issue = [&](int i) {  // Q and V of step i into stage i & 1
    uint8_t* st = ring + (i & 1) * BtCfg::STAGE_BYTES;
    uint64_t* bar = &full[i & 1];
    mbar_expect_tx(bar, BtCfg::STAGE_BYTES);
    for (int kb = 0; kb < 4; ++kb) tma_load_4d(st + kb * KB_BYTES, &tma_q, bar, kb * BK, i * BT_STEP, qz1, qz2);
    if (VN)  // image tokens themselves, [64 n x 256 c] as four [64 n x 64 c] blocks: the B operand of P.vn is read MN-major
      for (int cb = 0; cb < 4; ++cb) tma_load_4d(st + BtCfg::Q_BYTES + cb * KB_BYTES, &tma_v, bar, cb * BK, i * BT_STEP, vz1, vz2);
    else
      tma_load_4d(st + BtCfg::Q_BYTES, &tma_v, bar, i * BT_STEP, 0, vz1, vz2);
  };
  if (tid == 0) {
    tma_prefetch_desc(&tma_k);
    tma_prefetch_desc(&tma_q);
    tma_prefetch_desc(&tma_v);
    mbar_init(kt_full, 1);
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_mbar_init();
    mbar_expect_tx(kt_full, BtCfg::KT_BYTES);
    for (int kb = 0; kb < 4; ++kb)
      tma_load_4d(kt + kb * KB_BYTES, &tma_k, kt_full, kb * BK, mt * BM, p.k_bc1 ? 0 : z1, p.k_bc2 ? 0 : z2);
    issue(0);
    if (NS > 1) issue(1);
  }
  __syncthreads();

  // the two text tokens (rows) of this thread
  constexpr float L2E = 1.4426950408889634f;
  float m_l2[2] = {0.f, 0.f}, inv[2] = {0.f, 0.f}, gb[2] = {0.f, 0.f}, lsum[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = mt * BM + wg_row(tid, 2 * h);
    if (t < p.T) {
      if (VN) {
        m_l2[h] = -p.stat[(long)z * p.T + t] * L2E;
        if (p.rowbias) gb[h] = p.rowbias[((long)z * p.T + t) * p.rb_ld];
      } else {
        m_l2[h] = -p.stat[((long)z * 2) * p.T + t] * L2E;
        inv[h] = p.stat[((long)z * 2 + 1) * p.T + t];
      }
    }
  }
  const float clampv = p.clamp > 0.f ? p.clamp : 3.0e38f;
  const uint32_t kt_addr = smem_u32(kt);
  float o[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) o[i] = 0.f;
  mbar_wait(kt_full, 0);
  for (int i = 0; i < NS; ++i) {
    const int s = i & 1;
    mbar_wait(&full[s], (i >> 1) & 1);
    const uint32_t q0 = smem_u32(ring + s * BtCfg::STAGE_BYTES), v0 = q0 + BtCfg::Q_BYTES;
    float sc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) sc[j] = 0.f;
    wgmma_fence_acc(sc);
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss_m64n64_kk(sc, wg_desc_k_sw128(kt_addr + kb * KB_BYTES + k * 32), wg_desc_k_sw128(q0 + kb * KB_BYTES + k * 32), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(sc);
    const int nrem = p.N - i * BT_STEP;  // valid image tokens of this step
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int h = (j >> 1) & 1;
      const float a = fminf(fmaxf(sc[j] + gb[h], -clampv), clampv);
      // !VN: the score as the fp16 matrix A holds it (the statistics were taken from those values);
      //  VN: the fp32 score itself (the column maxima come from the fp32 scores of the image-side kernel)
      const float f = VN ? a : __half2float(__float2half_rn(a));
      float e = ex2_approx(fmaf(f, L2E, m_l2[h]));
      if (wg_col(tid, j) >= nrem) e = 0.f;  // image tokens beyond N (zero-filled q rows) must not contribute exp(-max)
      if (VN) lsum[h] += e;
      sc[j] = e;
    }
    uint32_t pa[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) acc_to_a(sc, kk, pa[kk]);
    wgmma_fence_acc(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      // VN: B = vn tile read MN-major (N = channel contiguous): 16 image tokens per MMA = 2 KB further down the block,
      // next 8 tokens (SBO) 1 KB apart, next 64 channels (LBO) one [64 n x 64 c] block = 8 KB apart
      if (VN)
        wgmma_rs_m64n256_kmn(o, pa[kk], wg_desc_mn_sw128(v0 + kk * 2048, KB_BYTES, 1024), 1);
      else
        wgmma_rs_m64n256_kk(o, pa[kk], wg_desc_k_sw128(v0 + kk * 32), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
    __syncthreads();  // every wgmma of the warpgroup has read stage s
    if (tid == 0 && i + 2 < NS) issue(i + 2);
  }
  if (VN) {  // total column sum of this text token: the four threads of a quad hold its columns
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float tot = quad_sum(lsum[h]);
      inv[h] = tot > 0.f ? 1.f / tot : 0.f;
    }
  }
  // ---- epilogue: O / colsum -> fp16 ----
  __half* out = p.out + z1 * p.o_b1 + z2 * p.o_b2;
#pragma unroll
  for (int j = 0; j < 128; j += 2) {
    const int h = (j >> 1) & 1;
    const int t = mt * BM + wg_row(tid, j);
    if (t < p.T)
      *reinterpret_cast<__half2*>(out + (long)t * p.o_ld + wg_col(tid, j)) = __floats2half2_rn(o[j] * inv[h], o[j + 1] * inv[h]);
  }
}

// =====================================================================================================================
// Image -> text side, fused with the out-projection, layer scale and residual.
//   vn [B][N][256] fp16 = the layer-normed image tokens
//   gT [B][H][T][256 c] fp16 = K_h (d^-1/2 Wv_h): the query projection of head h folded into the key operand —
//                              S = (vn Wv_h^T + bv) d^-1/2 K_h^T == vn gT_h^T + gbias_h[t] — so q is never built and ONE image-token
//                              tile serves all heads;  gbias [B*H][T] fp32 = d^-1/2 bv_h . K_h[t]
//   mT [B][H][256 o][T] fp16 = (W_h V_l,h^T): the value AND output projections of head h folded into one [T x 256] operand per
//                              (image, head) by a tiny GEMM — (P V_l,h) W_h^T == P (V_l,h W_h^T), so the per-head context O never
//                              exists and a head costs two tensor-core products instead of three
//   out[B][N][256] fp16
// One CTA per (image, 64-token tile); per tile the heads run back to back:
//   S (64 x 256 t)   = vn . gT_h^T (+ gbias_h)   16 wgmma 64x256x16, gT_h streamed as [256 x 64] k-blocks
//   P                = softmax_t(clamp(S) + mask) in the fragments (a row lives in one quad of threads); the column maxima of
//                      the clamped scores over the tile's valid rows go to colmax_part[b][h][tile][t] (reduced by
//                      colmax_reduce_kernel) — the text side needs them as the softmax shift
//   D (64 x 256 o)  += P . mT_h^T                 P from registers; the head sum is kept in thread-private shared memory
//   out              = res + gamma * (D + bias)
// =====================================================================================================================
struct BiCfg {
  static constexpr int VN_BYTES = 4 * KB_BYTES;     // image-token tile [64 x 256 c]
  static constexpr int STAGE_BYTES = 256 * BK * 2;  // one [256 x 64] k-block of gT_h or mT_h
  static constexpr int MAX_HEADS = 8;
  static constexpr int D_BYTES = 128 * 128 * 4;     // head sum: [128 fragment elements][128 threads] fp32
  static constexpr int EXTRA_BYTES = (4 * 256 + MAX_HEADS * 256) * 4;  // cmx, gk
  static constexpr int SMEM_BYTES = VN_BYTES + 2 * STAGE_BYTES + D_BYTES + EXTRA_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};
static_assert(BiCfg::SMEM_BYTES <= 232448, "biattn_image: dynamic shared memory above the 227 KB per-CTA limit");
struct BiP {
  const float* mask;   // [B][T] 1 keep / 0 padding, or nullptr
  const float* bias;   // [256] out-projection bias
  const float* gamma;  // [256] layer scale, or nullptr (1)
  const __half* res;   // residual [B][N][256] (row stride res_ld, batch stride res_b) or nullptr
  long res_ld, res_b;
  __half* out;         // [B][N][256] (row stride o_ld, batch stride o_b)
  long o_ld, o_b;
  float* colmax_part;  // [B][H][tiles_per_img][T]
  const float* gbias;  // [B*H][T * gb_ld] additive score bias per (head, token): the folded query-projection bias, or nullptr
  int gb_ld;
  float clamp;
  int B, H, T, N, tiles_per_img;
};

__global__ void __launch_bounds__(128, 1) biattn_image_kernel(const __grid_constant__ CUtensorMap tma_q,
                                                              const __grid_constant__ CUtensorMap tma_k,
                                                              const __grid_constant__ CUtensorMap tma_m, const BiP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* vnt = smem;
  uint8_t* ring = vnt + BiCfg::VN_BYTES;
  float* dsum = reinterpret_cast<float*>(ring + 2 * BiCfg::STAGE_BYTES);
  float* cmx = dsum + 128 * 128;  // [4 warps][256 tokens] column maxima
  float* gk = cmx + 4 * 256;      // [H][256] additive row-softmax term per (head, token): folded query bias + mask (0 / -inf)
  uint64_t* bars = reinterpret_cast<uint64_t*>(gk + BiCfg::MAX_HEADS * 256);
  uint64_t* vn_full = bars;
  uint64_t* full = bars + 1;  // [2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = p.H;
  const int b = blockIdx.x / p.tiles_per_img, ti = blockIdx.x - b * p.tiles_per_img, m0 = ti * BM;
  const int nq = 8 * H;  // ring sequence: per head 4 k-blocks of gT_h, then 4 of mT_h
  auto issue = [&](int q) {
    const int h = q >> 3, kb = q & 3;
    uint64_t* bar = &full[q & 1];
    mbar_expect_tx(bar, BiCfg::STAGE_BYTES);
    tma_load_4d(ring + (q & 1) * BiCfg::STAGE_BYTES, (q & 4) ? &tma_m : &tma_k, bar, kb * BK, 0, h, b);
  };
  if (tid == 0) {
    tma_prefetch_desc(&tma_q);
    tma_prefetch_desc(&tma_k);
    tma_prefetch_desc(&tma_m);
    mbar_init(vn_full, 1);
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_mbar_init();
    mbar_expect_tx(vn_full, BiCfg::VN_BYTES);
    for (int kb = 0; kb < 4; ++kb) tma_load_4d(vnt + kb * KB_BYTES, &tma_q, vn_full, kb * BK, m0, b, 0);
    issue(0);
    issue(1);
  }
  constexpr float L2E = 1.4426950408889634f;
  const float NEG_INF = __int_as_float(0xff800000);
  const float clampv = p.clamp > 0.f ? p.clamp : 3.0e38f;
  for (int t = tid; t < 256; t += 128) {
    const bool kept = t < p.T && (!p.mask || p.mask[(long)b * p.T + t] != 0.f);
    for (int hh = 0; hh < H; ++hh)
      gk[hh * 256 + t] = !kept ? NEG_INF : (p.gbias ? p.gbias[(((long)b * H + hh) * p.T + t) * p.gb_ld] : 0.f);
  }
  __syncthreads();
  bool valid[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) valid[h] = m0 + wg_row(tid, 2 * h) < p.N;
  const uint32_t vn_addr = smem_u32(vnt);
  int q = 0;
  auto ring_wait = [&](int qq) { mbar_wait(&full[qq & 1], (qq >> 1) & 1); };
  auto ring_release = [&](int qq) {  // every wgmma of the warpgroup has read stage qq & 1
    __syncthreads();
    if (tid == 0 && qq + 2 < nq) issue(qq + 2);
  };
  mbar_wait(vn_full, 0);
  for (int h = 0; h < H; ++h) {
    // ================= S = vn . gT_h^T =================
    float sc[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) sc[j] = 0.f;
    for (int kb = 0; kb < 4; ++kb, ++q) {
      ring_wait(q);
      const uint32_t b0 = smem_u32(ring + (q & 1) * BiCfg::STAGE_BYTES);
      wgmma_fence_acc(sc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss_m64n256_kk(sc, wg_desc_k_sw128(vn_addr + kb * KB_BYTES + k * 32), wg_desc_k_sw128(b0 + k * 32), 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(sc);
      ring_release(q);
    }
    // ---- column maxima over the tile's valid rows (for the text side): two rows per thread, then the 8 row groups of the warp,
    //      then the 4 warps through shared memory.  The +-5e4 clamp (fuse_helper.py:245-252) is applied to the REDUCED values
    //      (clamp is monotonic) ----
#pragma unroll
    for (int j = 0; j < 128; j += 4) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        float m = fmaxf(valid[0] ? sc[j + c] : NEG_INF, valid[1] ? sc[j + 2 + c] : NEG_INF);
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
        if (lane < 4) cmx[warp * 256 + wg_col(tid, j + c)] = m;
      }
    }
    __syncthreads();
    for (int t = tid; t < p.T; t += 128) {
      float c4 = fmaxf(fmaxf(cmx[t], cmx[256 + t]), fmaxf(cmx[512 + t], cmx[768 + t]));
      if (p.gbias) c4 += p.gbias[(((long)b * H + h) * p.T + t) * p.gb_ld];  // the text side sees the full score, no mask
      c4 = fminf(fmaxf(c4, -clampv), clampv);
      p.colmax_part[(((long)b * H + h) * p.tiles_per_img + ti) * p.T + t] = c4;
    }
    // ---- row softmax over the T tokens; `kk` carries the folded query bias and the token mask as an additive 0 / -inf ----
    const float* kl = gk + h * 256;
    float mr[2] = {NEG_INF, NEG_INF};
#pragma unroll
    for (int j = 0; j < 128; ++j) mr[(j >> 1) & 1] = fmaxf(mr[(j >> 1) & 1], sc[j] + kl[wg_col(tid, j)]);
    float ml2[2];
    bool uniform[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m_raw = quad_max(mr[r]);
      // every token masked: the reference's fp32 sum A + (-9e15) swallows A and the softmax is uniform over the T tokens
      uniform[r] = (m_raw == NEG_INF);
      ml2[r] = uniform[r] ? 0.f : fminf(fmaxf(m_raw, -clampv), clampv) * L2E;  // max over the kept tokens of the CLAMPED scores
    }
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 128; ++j) {
      const int r = (j >> 1) & 1, c = wg_col(tid, j);
      const float kk = kl[c];
      float ev = (kk == NEG_INF) ? 0.f : ex2_approx(fmaf(fminf(fmaxf(sc[j] + kk, -clampv), clampv), L2E, -ml2[r]));
      if (uniform[r]) ev = (c < p.T) ? 1.f : 0.f;
      sc[j] = ev;
      ls[r] += ev;
    }
    const float inv[2] = {1.f / quad_sum(ls[0]), 1.f / quad_sum(ls[1])};
#pragma unroll
    for (int j = 0; j < 128; ++j) sc[j] *= inv[(j >> 1) & 1];
    uint32_t pa[16][4];
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) acc_to_a(sc, kk, pa[kk]);
    // ================= D_h = P . mT_h^T, added to the head sum =================
    float d[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) d[j] = 0.f;
    for (int kb = 0; kb < 4; ++kb, ++q) {
      ring_wait(q);
      const uint32_t b0 = smem_u32(ring + (q & 1) * BiCfg::STAGE_BYTES);
      wgmma_fence_acc(d);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_rs_m64n256_kk(d, pa[kb * 4 + k], wg_desc_k_sw128(b0 + k * 32), 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(d);
      ring_release(q);
    }
#pragma unroll
    for (int j = 0; j < 128; ++j) dsum[j * 128 + tid] = (h == 0 ? 0.f : dsum[j * 128 + tid]) + d[j];
  }
  // ================= epilogue: out = res + gamma * (D + bias) =================
#pragma unroll 4
  for (int j = 0; j < 128; j += 2) {
    const long row = m0 + wg_row(tid, j);
    const int c = wg_col(tid, j);
    if (row >= p.N) continue;
    float o0 = dsum[j * 128 + tid], o1 = dsum[(j + 1) * 128 + tid];
    const float g0 = p.gamma ? p.gamma[c] : 1.f, g1 = p.gamma ? p.gamma[c + 1] : 1.f;
    const float b0 = p.bias ? p.bias[c] : 0.f, b1 = p.bias ? p.bias[c + 1] : 0.f;
    o0 = (o0 + b0) * g0;  // gamma * (D + bias)
    o1 = (o1 + b1) * g1;
    if (p.res) {
      const float2 r = __half22float2(*reinterpret_cast<const __half2*>(p.res + (long)b * p.res_b + row * p.res_ld + c));
      o0 += r.x;
      o1 += r.y;
    }
    *reinterpret_cast<__half2*>(p.out + (long)b * p.o_b + row * p.o_ld + c) = __floats2half2_rn(o0, o1);
  }
}

// colmax[z][t] = max over the tiles of colmax_part[z][tile][t]
__global__ void colmax_reduce_kernel(const float* __restrict__ part, int tiles, int T, float* __restrict__ out) {
  const int z = blockIdx.x;
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    float m = __int_as_float(0xff800000);
    const float* src = part + (long)z * tiles * T + t;
    for (int i = 0; i < tiles; ++i) m = fmaxf(m, src[(long)i * T]);
    out[(long)z * T + t] = m;
  }
}

}  // namespace mqdet

using namespace mqdet;

static int text_launch(bool vn, const float* rowbias, int64_t rb_ld, const void* k, int64_t k_ld, int64_t k_b1, int64_t k_b2, const void* q, int64_t q_ld, int64_t q_b1,
                       int64_t q_b2, const void* v, int64_t v_ld, int64_t v_b1, int64_t v_b2, const float* stat, float clamp,
                       void* out, int64_t o_ld, int64_t o_b1, int64_t o_b2, int64_t nb1, int64_t nb2, int64_t T, int64_t N,
                       int64_t Np, int64_t d, void* stream) {
  MQ_REQUIRE(k && q && v && stat && out, "biattn_text: null pointer");
  MQ_REQUIRE(d == 256, "biattn_text: head dim must be 256 (embed 2048 / 8 heads, fuse_helper.py:186-189), got %ld", (long)d);
  MQ_REQUIRE(T >= 1 && T <= 256 && N >= 1 && Np >= N && (Np % 8) == 0, "biattn_text: need 1 <= T <= 256, Np >= N, Np %% 8 == 0");
  MQ_REQUIRE(nb1 >= 1 && nb2 >= 1 && nb1 * nb2 <= 65535, "biattn_text: bad batch");
  const int64_t lds[] = {k_ld, k_b1, k_b2, q_ld, q_b1, q_b2, v_ld, v_b1, v_b2, o_ld, o_b1, o_b2};
  for (int64_t x : lds) MQ_REQUIRE((x % 8) == 0, "biattn_text: strides must be multiples of 8 elements");
  MQ_REQUIRE(((uintptr_t)k % 16) == 0 && ((uintptr_t)q % 16) == 0 && ((uintptr_t)v % 16) == 0 && ((uintptr_t)out % 16) == 0,
             "biattn_text: operands must be 16-byte aligned");
  CUtensorMap mk, mq, mv;
  BtP p;
  memset(&p, 0, sizeof(p));
  int rc = make_operand_map(&mk, k, T, d, k_ld, (int)nb1, k_b1, (int)nb2, k_b2, BM, &p.k_bc1, &p.k_bc2);
  if (rc) return rc;
  rc = make_operand_map(&mq, q, N, d, q_ld, (int)nb1, q_b1, (int)nb2, q_b2, BT_STEP, &p.q_bc1, &p.q_bc2);
  if (rc) return rc;
  if (vn)  // image tokens [N][256 c]: box [64 n x 64 c]
    rc = make_operand_map(&mv, v, N, 256, v_ld, (int)nb1, v_b1, (int)nb2, v_b2, BT_STEP, &p.v_bc1, &p.v_bc2);
  else     // Vv^T [256 d][Np]: box [256 d x 64 n]
    rc = make_operand_map(&mv, v, d, Np, v_ld, (int)nb1, v_b1, (int)nb2, v_b2, 256, &p.v_bc1, &p.v_bc2);
  if (rc) return rc;
  MQ_REQUIRE((nb1 == 1 || o_b1 != 0) && (nb2 == 1 || o_b2 != 0), "biattn_text: output batch strides must be non-zero");
  p.out = (__half*)out;
  p.o_ld = o_ld;
  p.o_b1 = o_b1;
  p.o_b2 = o_b2;
  p.stat = stat;
  p.clamp = clamp;
  p.nb1 = (int)nb1;
  p.T = (int)T;
  p.N = (int)N;
  p.n_steps = (int)((N + BT_STEP - 1) / BT_STEP);
  p.rowbias = rowbias;
  p.rb_ld = (int)(rb_ld > 0 ? rb_ld : 1);
  dim3 grid((unsigned)((T + BM - 1) / BM), (unsigned)(nb1 * nb2));
  if (vn) {
    rc = ensure_dyn_smem(reinterpret_cast<const void*>(&biattn_text_kernel<true>), BtCfg::SMEM_BYTES);
    if (rc) return rc;
    biattn_text_kernel<true><<<grid, 128, BtCfg::SMEM_BYTES, (cudaStream_t)stream>>>(mk, mq, mv, p);
  } else {
    rc = ensure_dyn_smem(reinterpret_cast<const void*>(&biattn_text_kernel<false>), BtCfg::SMEM_BYTES);
    if (rc) return rc;
    biattn_text_kernel<false><<<grid, 128, BtCfg::SMEM_BYTES, (cudaStream_t)stream>>>(mk, mq, mv, p);
  }
  return check_launch("biattn_text_kernel");
}

extern "C" int mqdet_biattn_text(const void* k, int64_t k_ld, int64_t k_b1, int64_t k_b2, const void* q, int64_t q_ld,
                                 int64_t q_b1, int64_t q_b2, const void* vvT, int64_t v_ld, int64_t v_b1, int64_t v_b2,
                                 const float* stat, float clamp, void* out, int64_t o_ld, int64_t o_b1, int64_t o_b2,
                                 int64_t nb1, int64_t nb2, int64_t T, int64_t N, int64_t Np, int64_t d, void* stream) {
  return text_launch(false, nullptr, 0, k, k_ld, k_b1, k_b2, q, q_ld, q_b1, q_b2, vvT, v_ld, v_b1, v_b2, stat, clamp, out, o_ld, o_b1, o_b2,
                     nb1, nb2, T, N, Np, d, stream);
}

extern "C" int mqdet_biattn_text_vn(const void* k, int64_t k_ld, int64_t k_b1, int64_t k_b2, const void* q, int64_t q_ld,
                                    int64_t q_b1, int64_t q_b2, const void* vn, int64_t vn_ld, int64_t vn_b1, int64_t vn_b2,
                                    const float* colmax, const float* rowbias, int64_t rb_ld, float clamp, void* out, int64_t o_ld,
                                    int64_t o_b1, int64_t o_b2, int64_t nb1, int64_t nb2, int64_t T, int64_t N, void* stream) {
  return text_launch(true, rowbias, rb_ld, k, k_ld, k_b1, k_b2, q, q_ld, q_b1, q_b2, vn, vn_ld, vn_b1, vn_b2, colmax, clamp, out, o_ld, o_b1,
                     o_b2, nb1, nb2, T, N, (N + 7) / 8 * 8, 256, stream);
}

extern "C" int64_t mqdet_biattn_image_workspace_floats(int64_t B, int64_t H, int64_t N, int64_t T) {
  return B * H * ((N + BM - 1) / BM) * T;
}

extern "C" int mqdet_biattn_image(const void* vn, int64_t vn_ld, int64_t vn_b, const void* gT, int64_t g_ld, int64_t g_bh,
                                  int64_t g_b, const float* gbias, int64_t gb_ld, const void* mT, int64_t m_ld, int64_t m_bh,
                                  int64_t m_b, const float* bias, const float* gamma, const void* res, int64_t res_ld,
                                  int64_t res_b, const float* mask, float clamp, void* out, int64_t o_ld, int64_t o_b,
                                  float* colmax, float* workspace, int64_t B, int64_t H, int64_t N, int64_t T, void* stream) {
  MQ_REQUIRE(vn && gT && mT && out && colmax && workspace, "biattn_image: null pointer");
  MQ_REQUIRE(B >= 1 && H >= 1 && H <= BiCfg::MAX_HEADS && N >= 1 && T >= 8 && T <= 256 && (T % 8) == 0,
             "biattn_image: need B, N >= 1, 1 <= H <= 8, 8 <= T <= 256, T %% 8 == 0 (got B=%ld H=%ld N=%ld T=%ld)", (long)B, (long)H, (long)N, (long)T);
  const int64_t lds[] = {vn_ld, vn_b, g_ld, g_bh, g_b, m_ld, m_bh, m_b, o_ld, o_b, res ? res_ld : 0, res ? res_b : 0};
  for (int64_t x : lds) MQ_REQUIRE((x % 8) == 0, "biattn_image: strides must be multiples of 8 elements");
  MQ_REQUIRE(((uintptr_t)vn % 16) == 0 && ((uintptr_t)gT % 16) == 0 && ((uintptr_t)mT % 16) == 0 && ((uintptr_t)out % 16) == 0 &&
                 ((uintptr_t)res % 16) == 0 && ((uintptr_t)bias % 16) == 0 && ((uintptr_t)gamma % 16) == 0,
             "biattn_image: operands must be 16-byte aligned");
  CUtensorMap mq, mk, mm;
  int bc1, bc2;
  int rc = make_operand_map(&mq, vn, N, 256, vn_ld, (int)B, vn_b, 1, 0, BM, &bc1, &bc2);
  if (rc) return rc;
  MQ_REQUIRE((H == 1 || (g_bh != 0 && m_bh != 0)) && (B == 1 || (g_b != 0 && m_b != 0)), "biattn_image: head / image strides must be non-zero");
  rc = make_operand_map(&mk, gT, T, 256, g_ld, (int)H, g_bh, (int)B, g_b, 256, &bc1, &bc2);  // [B][H][T][256 c]
  if (rc) return rc;
  rc = make_operand_map(&mm, mT, 256, T, m_ld, (int)H, m_bh, (int)B, m_b, 256, &bc1, &bc2);  // [B][H][256 o][T]
  if (rc) return rc;
  MQ_REQUIRE(B == 1 || o_b != 0, "biattn_image: output batch stride must be non-zero");
  BiP p;
  memset(&p, 0, sizeof(p));
  p.mask = mask;
  p.bias = bias;
  p.gamma = gamma;
  p.res = (const __half*)res;
  p.res_ld = res_ld;
  p.res_b = res_b;
  p.out = (__half*)out;
  p.o_ld = o_ld;
  p.o_b = o_b;
  p.colmax_part = workspace;
  p.gbias = gbias;
  p.gb_ld = (int)(gb_ld > 0 ? gb_ld : 1);
  p.clamp = clamp;
  p.B = (int)B; p.H = (int)H; p.T = (int)T; p.N = (int)N;
  p.tiles_per_img = (int)((N + BM - 1) / BM);
  rc = ensure_dyn_smem(reinterpret_cast<const void*>(&biattn_image_kernel), BiCfg::SMEM_BYTES);
  if (rc) return rc;
  biattn_image_kernel<<<(unsigned)(p.tiles_per_img * B), 128, BiCfg::SMEM_BYTES, (cudaStream_t)stream>>>(mq, mk, mm, p);
  rc = check_launch("biattn_image_kernel");
  if (rc) return rc;
  colmax_reduce_kernel<<<(unsigned)(B * H), 256, 0, (cudaStream_t)stream>>>(workspace, p.tiles_per_img, (int)T, colmax);
  return check_launch("colmax_reduce_kernel");
}
