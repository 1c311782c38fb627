// mqdet_b200 — the bi-directional image <-> text attention of the VL fusion tower (BiMultiHeadAttention,
// maskrcnn_benchmark/utils/fuse_helper.py:218-303) as two wgmma kernels that never materialise the score matrix:
//
//   biattn_image_kernel : image -> text side.  Per 64 image tokens and head: S = Q K^T (fp32, registers) -> +-5e4 clamp ->
//                         column-max partials (for the text side) -> masked row softmax over the T tokens in the accumulator
//                         fragments -> P (fp16, registers: the A operand of the next wgmma) -> P . mT_h, summed over the heads
//                         -> v' = residual + gamma * (acc + bias).  Neither the scores nor the per-head context reach HBM.
//   biattn_text_kernel  : text -> image side (one CTA per (image, head, 128 text tokens): a TMA producer warpgroup streams all
//                         image tokens through a ring to two consumer warpgroups of 64 text tokens each):
//                         S^T recomputed on the tensor cores, exp(S^T - column max), P . V accumulated in registers, with
//                         V = the layer-normed image tokens themselves (read MN-major from the same [n x c] tile, loaded once
//                         when q is those tokens): the value projection is applied AFTER the token reduction (sum_n p[n] = 1),
//                         and the column sums are accumulated in-kernel, so the [B, E, N] value tensor of the image side is
//                         never built.
// Each MMA warpgroup keeps a 64 x 256 fp32 accumulator in its registers (128 per thread).  Operands arrive by TMA (128B swizzle);
// accumulator fragment: row / column of element i of thread t = wg_row / wg_col.
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
// one step of a transposing max-butterfly over the lanes that differ in bit `mask`: the lane with that bit set keeps the upper
// n values, the other the lower n, and each takes the maximum with the half its partner sends; the result is in v[0 .. n)
template <int n>
__device__ __forceinline__ void butterfly_max(float (&v)[32], int lane, int mask) {
  const bool hi = lane & mask;
#pragma unroll
  for (int k = 0; k < n; ++k) {
    const float send = hi ? v[k] : v[k + n];
    const float keep = hi ? v[k + n] : v[k];
    v[k] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, mask));
  }
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// =====================================================================================================================
// Fused text -> image side of the bi-directional attention (BiMultiHeadAttention, fuse_helper.py:257-275, 289-291):
//     out[t, :] = sum_n softmax_n(clamp(k_t . q_n + rowbias_t)) * vn[n, :]   per (image, head), t = text token, n = image token
// One CTA per (z, 128 text tokens), 384 threads.  The transposed probabilities [T, N] never reach HBM.
//   warpgroup 0     : producer.  One thread loads the K tiles once, then streams the image tokens 64 at a time through a ring
//                     with a full and an empty mbarrier per stage.  When q is vn itself (same memory, the head broadcast - the
//                     fusion layers pass it so) a stage is ONE [64 n x 256 c] tile that serves as both operands: K-major as the
//                     B operand of S^T, MN-major as the B operand of P . vn (5 stages).  Otherwise a stage carries the q tile
//                     next to it (2 stages).
//   warpgroups 1, 2 : consumers; warpgroup w owns the text tokens 64 w .. 64 w + 63 of the CTA: its resident K tile, its O
//                     accumulator (64 x 256 fp32 in registers), its column sums and its epilogue.  A consumer whose tokens all
//                     lie at or beyond T exits at once, and the empty barriers count only the active consumers.
// Per step of 64 image tokens, per consumer:
//     S^T   = K_tile (64 x 256, resident) . Q_step^T           16 wgmma 64x64x16
//     P     = exp(clamp(S^T + rowbias) - colmax_t)             in the accumulator fragments -> fp16 A operand (registers)
//     O    += P . vn_step                                        4 wgmma 64x256x16, O (64 x 256) in registers
//     out   = O / colsum_t  -> fp16
// The products are issued one step apart: S^T of step i + 1 goes to the tensor cores ahead of P . vn of step i, so the exps of
// step i + 1 can run while P . vn of step i (and the other consumer's products) execute; a stage is released once the P . vn
// that read it has retired.  Every sum keeps the order of one warpgroup walking the image tokens.
// colmax comes from biattn_image_kernel (the column maxima of the same clamped fp32 scores), so no online rescaling is needed;
// colsum is accumulated here from the fp32 scores.
// =====================================================================================================================
constexpr int BT_STEP = 64;     // image tokens per step
constexpr int BT_ROWS = 2 * BM;  // text tokens per CTA: one 64-token tile per consumer warpgroup
struct BtCfg {
  static constexpr int TILE_BYTES = 4 * KB_BYTES;    // [64 x 256] as four [64 x 64] k-blocks: a K tile or an image-token tile
  static constexpr int RING_TILES = 5;               // 5 stages of one tile, or 2 stages of [vn tile | q tile]
  static constexpr int SMEM_BYTES = 2 * TILE_BYTES + RING_TILES * TILE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};
static_assert(BtCfg::SMEM_BYTES <= 232448, "biattn_text: dynamic shared memory above the 227 KB per-CTA limit");
static_assert((1 + 2 * BtCfg::RING_TILES) * 8 <= 256, "biattn_text: barrier space");
struct BtP {
  const float* stat;  // [Z][T] column max
  float clamp;
  int nb1, T, N, n_steps;
  int k_bc1, k_bc2, q_bc1, q_bc2, v_bc1, v_bc2;  // 1 -> batch coordinate pinned to 0
  int q_is_vn;                                    // q and vn are the same tokens: one tile per stage serves both operands
  const float* rowbias;                           // optional [Z][T * rb_ld] additive score bias per text token (folded q bias)
  int rb_ld;
  __half* out;                                    // [nb2][nb1][T][256]
  long o_ld, o_b1, o_b2;
};

// keeps the compiler from reusing the A-fragment registers of an asynchronous wgmma before it has retired
__device__ __forceinline__ void keep_a_live(uint32_t (&a)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(a[i][j])::"memory");
}

__global__ void __launch_bounds__(384, 1) biattn_text_kernel(const __grid_constant__ CUtensorMap tma_k,
                                                             const __grid_constant__ CUtensorMap tma_q,
                                                             const __grid_constant__ CUtensorMap tma_v, const BtP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* kt = smem;                         // [2 consumers] K tiles
  uint8_t* ring = kt + 2 * BtCfg::TILE_BYTES;  // stages of [vn tile] or [vn tile | q tile]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + BtCfg::RING_TILES * BtCfg::TILE_BYTES);
  uint64_t* kt_full = bars;
  uint64_t* full = bars + 1;                 // [stages]
  uint64_t* empty = full + BtCfg::RING_TILES;  // [stages]

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int mt = blockIdx.x, z = blockIdx.y;
  const int z1 = z % p.nb1, z2 = z / p.nb1;
  const int NS = p.n_steps;
  const int nact = p.T - mt * BT_ROWS > BM ? 2 : 1;  // consumers with at least one text token
  const int stage_bytes = (p.q_is_vn ? 1 : 2) * BtCfg::TILE_BYTES;
  const int stages = p.q_is_vn ? BtCfg::RING_TILES : BtCfg::RING_TILES / 2;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_k);
    tma_prefetch_desc(&tma_q);
    tma_prefetch_desc(&tma_v);
    mbar_init(kt_full, 1);
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 128 * nact);  // every thread of each active consumer releases every stage
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (tid == 0) {
      mbar_expect_tx(kt_full, nact * BtCfg::TILE_BYTES);
      for (int w = 0; w < nact; ++w)
        for (int kb = 0; kb < 4; ++kb)
          tma_load_4d(kt + w * BtCfg::TILE_BYTES + kb * KB_BYTES, &tma_k, kt_full, kb * BK, mt * BT_ROWS + w * BM,
                      p.k_bc1 ? 0 : z1, p.k_bc2 ? 0 : z2);
      const int qz1 = p.q_bc1 ? 0 : z1, qz2 = p.q_bc2 ? 0 : z2, vz1 = p.v_bc1 ? 0 : z1, vz2 = p.v_bc2 ? 0 : z2;
      int s = 0;
      uint32_t ph = 0;
      for (int i = 0; i < NS; ++i) {
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = ring + s * stage_bytes;
        mbar_expect_tx(&full[s], stage_bytes);
        // image tokens [64 n x 256 c] as four [64 n x 64 c] blocks
        for (int cb = 0; cb < 4; ++cb) tma_load_4d(st + cb * KB_BYTES, &tma_v, &full[s], cb * BK, i * BT_STEP, vz1, vz2);
        if (!p.q_is_vn)
          for (int kb = 0; kb < 4; ++kb)
            tma_load_4d(st + BtCfg::TILE_BYTES + kb * KB_BYTES, &tma_q, &full[s], kb * BK, i * BT_STEP, qz1, qz2);
        if (++s == stages) {
          s = 0;
          ph ^= 1;
        }
      }
    }
    return;
  }
  const int w = wg - 1;
  if (w >= nact) return;
  setmaxnreg_inc<232>();
  const int t0 = mt * BT_ROWS + w * BM;  // first text token of this consumer

  // the two text tokens (rows) of this thread
  constexpr float L2E = 1.4426950408889634f;
  float m_l2[2] = {0.f, 0.f}, inv[2] = {0.f, 0.f}, gb[2] = {0.f, 0.f}, lsum[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = t0 + wg_row(tid, 2 * h);
    if (t < p.T) {
      m_l2[h] = -p.stat[(long)z * p.T + t] * L2E;
      if (p.rowbias) gb[h] = p.rowbias[((long)z * p.T + t) * p.rb_ld];
    }
  }
  const float clampv = p.clamp > 0.f ? p.clamp : 3.0e38f;
  const uint32_t kt_addr = smem_u32(kt + w * BtCfg::TILE_BYTES), ring_addr = smem_u32(ring);
  const uint32_t q_off = p.q_is_vn ? 0 : BtCfg::TILE_BYTES;
  float o[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) o[i] = 0.f;
  float sc[32];
  // S^T of the image-token tile in stage s -> sc (committed, not waited for)
  auto scores = [&](int s) {
    const uint32_t q0 = ring_addr + s * stage_bytes + q_off;
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
  };
  // retired scores of step i -> e = exp(...), column sums, and the fp16 A fragments of P . vn
  auto probs = [&](int i, uint32_t (&pa)[4][4]) {
    wgmma_fence_acc(sc);
    const int nrem = p.N - i * BT_STEP;  // valid image tokens of this step
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int h = (j >> 1) & 1;
      const float a = fminf(fmaxf(sc[j] + gb[h], -clampv), clampv);
      float e = ex2_approx(fmaf(a, L2E, m_l2[h]));
      if (wg_col(tid, j) >= nrem) e = 0.f;  // image tokens beyond N (zero-filled q rows) must not contribute exp(-max)
      lsum[h] += e;
      sc[j] = e;
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) acc_to_a(sc, kk, pa[kk]);
  };
  // O += P . vn of the tile in stage s (committed, not waited for)
  auto pv = [&](int s, const uint32_t (&pa)[4][4]) {
    const uint32_t v0 = ring_addr + s * stage_bytes;
    wgmma_fence_acc(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      // B = vn tile read MN-major (N = channel contiguous): 16 image tokens per MMA = 2 KB further down the block,
      // next 8 tokens (SBO) 1 KB apart, next 64 channels (LBO) one [64 n x 64 c] block = 8 KB apart
      wgmma_rs_m64n256_kmn(o, pa[kk], wg_desc_mn_sw128(v0 + kk * 2048, KB_BYTES, 1024), 1);
    }
    wgmma_commit();
  };
  uint32_t pa[4][4];
  mbar_wait(kt_full, 0);
  mbar_wait(&full[0], 0);
  scores(0);
  wgmma_wait<0>();
  probs(0, pa);
  int s = 0;
  uint32_t ph = 0;
  for (int i = 0; i + 1 < NS; ++i) {
    const int sn = s + 1 == stages ? 0 : s + 1;
    const uint32_t phn = sn == 0 ? ph ^ 1 : ph;
    mbar_wait(&full[sn], phn);
    scores(sn);
    pv(s, pa);
    wgmma_wait<1>();  // S^T of step i + 1 has retired; P . vn of step i may still run
    uint32_t pn[4][4];
    probs(i + 1, pn);
    wgmma_wait<0>();
    wgmma_fence_acc(o);
    keep_a_live(pa);
    mbar_arrive(&empty[s]);  // P . vn of step i has read stage s
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[kk][r] = pn[kk][r];
    s = sn;
    ph = phn;
  }
  pv(s, pa);
  wgmma_wait<0>();
  wgmma_fence_acc(o);
  // total column sum of this text token: the four threads of a quad hold its columns
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float tot = quad_sum(lsum[h]);
    inv[h] = tot > 0.f ? 1.f / tot : 0.f;
  }
  // ---- epilogue: O / colsum -> fp16 ----
  __half* out = p.out + z1 * p.o_b1 + z2 * p.o_b2;
#pragma unroll
  for (int j = 0; j < 128; j += 2) {
    const int h = (j >> 1) & 1;
    const int t = t0 + wg_row(tid, j);
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
// One CTA per (image, 64-token tile), 384 threads; per tile the heads run back to back:
//   warpgroup 0      : producer.  One thread loads the image-token tile once, then streams per head the 4 k-blocks of gT_h and
//                      the 4 of mT_h ([256 x 64] each, 32 KB) through a STAGES-deep ring with a full and an empty mbarrier per
//                      stage, so up to STAGES - 1 k-blocks are in flight while the consumers compute.
//   warpgroups 1, 2  : consumers; warpgroup w owns the text tokens t and the output columns o in [128 w, 128 w + 128):
//     S_w (64 x 128)  = vn . gT_h[t]^T            16 wgmma 64x128x16 (rows 128 w.. of each gT stage)
//     column maxima of the clamped scores over the tile's valid rows -> colmax_part[b][h][tile][t] (reduced by
//                       colmax_reduce_kernel): the text side needs them as the softmax shift
//     P               = softmax_t(clamp(S) + mask): row max and row sum combined over the two halves in shared memory; both
//                       halves of P are written to shared memory as one 128B-swizzled [64 x 256 t] A operand
//     D_h,w (64 x 128) = P . mT_h[o]^T            16 wgmma 64x128x16 over all T (rows 128 w.. of each mT stage)
//     Dsum_w          += D_h,w                     the head sum, in registers
//   out[:, o] = res + gamma * (Dsum_w + bias).
// Every sum runs in the order of a single warpgroup walking the whole row (the row sum continues warpgroup 0's per-thread partial,
// each D_h element is one K = T chain, and the head sum adds one D_h per head), so the result is bit-identical to computing a
// tile in one warpgroup.
// =====================================================================================================================
struct BiCfg {
  static constexpr int STAGES = 4;
  static constexpr int VN_BYTES = 4 * KB_BYTES;     // image-token tile [64 x 256 c]
  static constexpr int STAGE_BYTES = 256 * BK * 2;  // one [256 x 64] k-block of gT_h or mT_h
  static constexpr int P_BYTES = 4 * KB_BYTES;      // probabilities [64 x 256 t] fp16, the A operand of P . mT_h
  static constexpr int MAX_HEADS = 8;
  static constexpr int GK_BYTES = MAX_HEADS * 256 * 4;  // additive row-softmax term per (head, token)
  static constexpr int GC_BYTES = MAX_HEADS * 256 * 4;  // folded query bias per (head, token) for the column maxima
  static constexpr int CMX_BYTES = 2 * 4 * 128 * 4;     // column-max partials [consumer warpgroup][warp][128 tokens]
  static constexpr int XCH_BYTES = (2 * BM + BM + 2 * 128) * 4;  // row max halves, row sums, warpgroup 0's row-sum partials
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = VN_BYTES + STAGES * STAGE_BYTES + P_BYTES + GK_BYTES + GC_BYTES + CMX_BYTES + XCH_BYTES +
                                    BAR_BYTES + 1024 /*align*/;
};
static_assert(BiCfg::SMEM_BYTES <= 232448, "biattn_image: dynamic shared memory above the 227 KB per-CTA limit");
static_assert((1 + 2 * BiCfg::STAGES) * 8 <= BiCfg::BAR_BYTES, "biattn_image: barrier space");
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

__global__ void __launch_bounds__(384, 1) biattn_image_kernel(const __grid_constant__ CUtensorMap tma_q,
                                                              const __grid_constant__ CUtensorMap tma_k,
                                                              const __grid_constant__ CUtensorMap tma_m, const BiP p) {
  constexpr int STAGES = BiCfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* vnt = smem;
  uint8_t* ring = vnt + BiCfg::VN_BYTES;
  uint8_t* pt = ring + STAGES * BiCfg::STAGE_BYTES;
  float* gk = reinterpret_cast<float*>(pt + BiCfg::P_BYTES);  // [H][256]: folded query bias + mask (0 / -inf)
  float* gc = gk + BiCfg::MAX_HEADS * 256;  // [H][256]: folded query bias, unmasked
  float* cmx = gc + BiCfg::MAX_HEADS * 256;
  float* xmax = cmx + 2 * 4 * 128;  // [warpgroup][64 rows]
  float* xsum = xmax + 2 * BM;      // [64 rows]
  float* xpart = xsum + BM;         // [128 threads][2 rows]
  uint64_t* bars = reinterpret_cast<uint64_t*>(xpart + 2 * 128);
  uint64_t* vn_full = bars;
  uint64_t* full = bars + 1;        // [STAGES]
  uint64_t* empty = full + STAGES;  // [STAGES]

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int H = p.H;
  const int b = blockIdx.x / p.tiles_per_img, ti = blockIdx.x - b * p.tiles_per_img, m0 = ti * BM;
  const int nq = 8 * H;  // ring sequence: per head 4 k-blocks of gT_h, then 4 of mT_h
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_q);
    tma_prefetch_desc(&tma_k);
    tma_prefetch_desc(&tma_m);
    mbar_init(vn_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 256);  // both consumer warpgroups read every stage
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (tid == 0) {
      mbar_expect_tx(vn_full, BiCfg::VN_BYTES);
      for (int kb = 0; kb < 4; ++kb) tma_load_4d(vnt + kb * KB_BYTES, &tma_q, vn_full, kb * BK, m0, b, 0);
      for (int q = 0; q < nq; ++q) {
        const int s = q % STAGES;
        mbar_wait(&empty[s], ((q / STAGES) & 1) ^ 1);
        mbar_expect_tx(&full[s], BiCfg::STAGE_BYTES);
        tma_load_4d(ring + s * BiCfg::STAGE_BYTES, (q & 4) ? &tma_m : &tma_k, &full[s], (q & 3) * BK, 0, q >> 3, b);
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int w = wg - 1, warp = tid >> 5, lane = tid & 31;
  const int t0 = 128 * w;  // first text token and first output column of this warpgroup
  constexpr float L2E = 1.4426950408889634f;
  const float NEG_INF = __int_as_float(0xff800000);
  const float clampv = p.clamp > 0.f ? p.clamp : 3.0e38f;
  {
    const int t = threadIdx.x - 128;
    const bool kept = t < p.T && (!p.mask || p.mask[(long)b * p.T + t] != 0.f);
    for (int hh = 0; hh < H; ++hh) {
      const float gb = p.gbias && t < p.T ? p.gbias[(((long)b * H + hh) * p.T + t) * p.gb_ld] : 0.f;
      gc[hh * 256 + t] = gb;
      gk[hh * 256 + t] = kept ? gb : NEG_INF;
    }
  }
  named_bar_sync(1, 256);
  bool valid[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) valid[r] = m0 + wg_row(tid, 2 * r) < p.N;
  const int row0 = wg_row(tid, 0);  // this thread's rows: row0 and row0 + 8
  const uint32_t vn_addr = smem_u32(vnt), ring_addr = smem_u32(ring), pt_addr = smem_u32(pt);
  float* cw = cmx + w * 512;
  auto stage_wait = [&](int q) { mbar_wait(&full[q % STAGES], (q / STAGES) & 1); };
  float dsum[64];
  mbar_wait(vn_full, 0);
  for (int h = 0; h < H; ++h) {
    const int qh = 8 * h;
    // ================= S_w = vn . gT_h[t0 .. t0 + 127]^T; each k-block's stage is released once its MMAs have retired =========
    float sc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) sc[j] = 0.f;
    wgmma_fence_acc(sc);
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
      stage_wait(qh + kb);
      wgmma_fence();
      // rows 128 w.. of the [256 x 64] stage: 16 KB further, a multiple of the 1 KB swizzle atom
      const uint32_t b0 = ring_addr + ((qh + kb) % STAGES) * BiCfg::STAGE_BYTES + w * (128 * 128);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss_m64n128_kk(sc, wg_desc_k_sw128(vn_addr + kb * KB_BYTES + k * 32), wg_desc_k_sw128(b0 + k * 32), 1);
      wgmma_commit();
      if (kb > 0) {
        wgmma_wait<1>();
        mbar_arrive(&empty[(qh + kb - 1) % STAGES]);
      }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(sc);
    mbar_arrive(&empty[(qh + 3) % STAGES]);
    // rows at or beyond N (in the last tile of an image only) drop out of the column maxima as -inf.  Nothing else reads their
    // scores: a row's softmax and its P . mT row use only its own scores, and its output is never written
    if (m0 + BM > p.N) {
#pragma unroll
      for (int j = 0; j < 64; ++j)
        if (!valid[(j >> 1) & 1]) sc[j] = NEG_INF;
    }
    // ---- column maxima over the tile's valid rows (for the text side): two rows per thread, then the 8 row groups of the warp,
    //      then the 4 warps of the warpgroup through shared memory.  The +-5e4 clamp (fuse_helper.py:245-252) is applied to the
    //      REDUCED values (clamp is monotonic) ----
    {
      // cm[k]: column 8 (k >> 1) + 2 (lane & 3) + (k & 1).  The row groups meet in a transposing butterfly: at the xor-(4 << st)
      // step a lane keeps one half of its columns, sends the other half to its partner and takes the maximum with what the
      // partner sends, so after three steps it holds the warp's maxima of 4 of the 32 columns (28 shuffles, where reducing each
      // column on its own takes 96)
      float cm[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) cm[k] = fmaxf(sc[4 * (k >> 1) + (k & 1)], sc[4 * (k >> 1) + 2 + (k & 1)]);
      butterfly_max<16>(cm, lane, 4);
      butterfly_max<8>(cm, lane, 8);
      butterfly_max<4>(cm, lane, 16);
      // cm[k] (k < 4) now holds column index k + 4 b2 + 8 b1 + 16 b0 of the 32, b_i = bit i of lane >> 2
      const int k0 = 16 * ((lane >> 2) & 1) + 8 * ((lane >> 3) & 1) + 4 * ((lane >> 4) & 1);
#pragma unroll
      for (int k = 0; k < 4; ++k) cw[warp * 128 + 8 * ((k0 + k) >> 1) + 2 * (lane & 3) + (k & 1)] = cm[k];
    }
    // ---- row softmax over the T tokens; `kk` carries the folded query bias and the token mask as an additive 0 / -inf.
    //      Each warpgroup holds half of a row; the halves meet in xmax / xpart / xsum ----
    const float* kl = gk + h * 256 + t0;
    float mr[2] = {NEG_INF, NEG_INF};
#pragma unroll
    for (int j = 0; j < 64; ++j) {
      sc[j] += kl[wg_col(tid, j)];  // from here on sc holds S + kk (-inf for masked tokens)
      mr[(j >> 1) & 1] = fmaxf(mr[(j >> 1) & 1], sc[j]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mr[r] = quad_max(mr[r]);
      if ((lane & 3) == 0) xmax[w * BM + row0 + 8 * r] = mr[r];
    }
    named_bar_sync(1, 256);  // cw and xmax written; the previous head's P . mT MMAs have retired in both warpgroups
    {
      const int t = t0 + tid;
      if (t < p.T) {
        float c4 = fmaxf(fmaxf(cw[tid], cw[128 + tid]), fmaxf(cw[256 + tid], cw[384 + tid]));
        if (p.gbias) c4 += gc[h * 256 + t];  // the text side sees the full score, no mask
        c4 = fminf(fmaxf(c4, -clampv), clampv);
        p.colmax_part[(((long)b * H + h) * p.tiles_per_img + ti) * p.T + t] = c4;
      }
    }
    float ml2[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m_raw = fmaxf(xmax[row0 + 8 * r], xmax[BM + row0 + 8 * r]);
      ml2[r] = fminf(fmaxf(m_raw, -clampv), clampv) * L2E;  // max over the kept tokens of the CLAMPED scores
    }
    const bool uniform = xmax[row0] == NEG_INF && xmax[BM + row0] == NEG_INF;
#pragma unroll
    for (int j = 0; j < 64; ++j) {
      const int r = (j >> 1) & 1;
      sc[j] = (sc[j] == NEG_INF) ? 0.f : ex2_approx(fmaf(fminf(fmaxf(sc[j], -clampv), clampv), L2E, -ml2[r]));
    }
    // every token of the image masked (the row maximum is -inf for every row of the tile): the reference's fp32 sum
    // A + (-9e15) swallows A and the softmax is uniform over the T tokens
    if (__any_sync(0xffffffffu, uniform)) {
#pragma unroll
      for (int j = 0; j < 64; ++j)
        if (uniform) sc[j] = (t0 + wg_col(tid, j) < p.T) ? 1.f : 0.f;
    }
    // row sum: the thread of warpgroup 1 continues the sequential sum of the same thread of warpgroup 0 (the same rows, the
    // columns 128 further), then the four threads of a row combine
    float ls[2] = {0.f, 0.f};
    if (w == 0) {
#pragma unroll
      for (int j = 0; j < 64; ++j) ls[(j >> 1) & 1] += sc[j];
      xpart[2 * tid] = ls[0];
      xpart[2 * tid + 1] = ls[1];
    }
    named_bar_sync(1, 256);  // xpart written; cw and xmax have been read
    if (w == 1) {
      ls[0] = xpart[2 * tid];
      ls[1] = xpart[2 * tid + 1];
#pragma unroll
      for (int j = 0; j < 64; ++j) ls[(j >> 1) & 1] += sc[j];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        ls[r] = quad_sum(ls[r]);
        if ((lane & 3) == 0) xsum[row0 + 8 * r] = ls[r];
      }
    }
    named_bar_sync(1, 256);  // xsum written; xpart has been read
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) inv[r] = 1.f / xsum[row0 + 8 * r];
    // P (fp16) -> this warpgroup's two [64 x 64 t] k-blocks of the swizzled A tile: row r, 16-byte chunk c at chunk c ^ (r & 7)
#pragma unroll
    for (int j = 0; j < 64; j += 2) {
      const int r = wg_row(tid, j), kc = wg_col(tid, j) & 63;
      const uint32_t a = pt_addr + (2 * w + (j >> 5)) * KB_BYTES + r * 128 + ((((kc >> 3) ^ (r & 7))) << 4) + (kc & 7) * 2;
      sts32(a, pack_half2(sc[j] * inv[(j >> 1) & 1], sc[j + 1] * inv[(j >> 1) & 1]));
    }
    fence_proxy_async();     // the A tile's generic-proxy writes are visible to wgmma
    named_bar_sync(1, 256);  // both halves of P written; xsum has been read
    // ================= D_h,w = P . mT_h[t0 .. t0 + 127 (o)]^T over the T tokens, added to the head sum =================
    float dh[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) dh[j] = 0.f;
    wgmma_fence_acc(dh);
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
      stage_wait(qh + 4 + kb);
      wgmma_fence();
      const uint32_t b0 = ring_addr + ((qh + 4 + kb) % STAGES) * BiCfg::STAGE_BYTES + w * (128 * 128);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss_m64n128_kk(dh, wg_desc_k_sw128(pt_addr + kb * KB_BYTES + k * 32), wg_desc_k_sw128(b0 + k * 32), 1);
      wgmma_commit();
      if (kb > 0) {
        wgmma_wait<1>();
        mbar_arrive(&empty[(qh + 4 + kb - 1) % STAGES]);
      }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(dh);
    mbar_arrive(&empty[(qh + 7) % STAGES]);
#pragma unroll
    for (int j = 0; j < 64; ++j) dsum[j] = (h == 0 ? 0.f : dsum[j]) + dh[j];
  }
  // ================= epilogue: out = res + gamma * (Dsum + bias) on this warpgroup's 128 columns =================
  // elements j, j + 1 (row0) and j + 2, j + 3 (row0 + 8) share the columns c, c + 1 and their gamma / bias
  const __half* res = p.res ? p.res + (long)b * p.res_b : nullptr;
  __half* out = p.out + (long)b * p.o_b;
#pragma unroll
  for (int j = 0; j < 64; j += 4) {
    const int c = t0 + wg_col(tid, j);
    const float2 g = p.gamma ? *reinterpret_cast<const float2*>(p.gamma + c) : make_float2(1.f, 1.f);
    const float2 bi = p.bias ? *reinterpret_cast<const float2*>(p.bias + c) : make_float2(0.f, 0.f);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const long row = m0 + row0 + 8 * r;
      if (row >= p.N) continue;
      // gamma * (D + bias), then + res, rounded step by step (never contracted into one fma)
      float o0 = __fmul_rn(dsum[j + 2 * r] + bi.x, g.x);
      float o1 = __fmul_rn(dsum[j + 2 * r + 1] + bi.y, g.y);
      if (res) {
        const float2 rv = __half22float2(*reinterpret_cast<const __half2*>(res + row * p.res_ld + c));
        o0 = __fadd_rn(o0, rv.x);
        o1 = __fadd_rn(o1, rv.y);
      }
      *reinterpret_cast<__half2*>(out + row * p.o_ld + c) = __floats2half2_rn(o0, o1);
    }
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

extern "C" int mqdet_biattn_text_vn(const void* k, int64_t k_ld, int64_t k_b1, int64_t k_b2, const void* q, int64_t q_ld,
                                    int64_t q_b1, int64_t q_b2, const void* vn, int64_t vn_ld, int64_t vn_b1, int64_t vn_b2,
                                    const float* colmax, const float* rowbias, int64_t rb_ld, float clamp, void* out, int64_t o_ld,
                                    int64_t o_b1, int64_t o_b2, int64_t nb1, int64_t nb2, int64_t T, int64_t N, void* stream) {
  MQ_REQUIRE(k && q && vn && colmax && out, "biattn_text_vn: null pointer");
  MQ_REQUIRE(T >= 1 && T <= 256 && N >= 1, "biattn_text_vn: need 1 <= T <= 256, N >= 1");
  MQ_REQUIRE(nb1 >= 1 && nb2 >= 1 && nb1 * nb2 <= 65535, "biattn_text_vn: bad batch");
  const int64_t lds[] = {k_ld, k_b1, k_b2, q_ld, q_b1, q_b2, vn_ld, vn_b1, vn_b2, o_ld, o_b1, o_b2};
  for (int64_t x : lds) MQ_REQUIRE((x % 8) == 0, "biattn_text_vn: strides must be multiples of 8 elements");
  MQ_REQUIRE(((uintptr_t)k % 16) == 0 && ((uintptr_t)q % 16) == 0 && ((uintptr_t)vn % 16) == 0 && ((uintptr_t)out % 16) == 0,
             "biattn_text_vn: operands must be 16-byte aligned");
  CUtensorMap mk, mq, mv;
  BtP p;
  memset(&p, 0, sizeof(p));
  int rc = make_operand_map(&mk, k, T, 256, k_ld, (int)nb1, k_b1, (int)nb2, k_b2, BM, &p.k_bc1, &p.k_bc2);
  if (rc) return rc;
  // image tokens [N][256 c]: box [64 n x 64 c]
  rc = make_operand_map(&mv, vn, N, 256, vn_ld, (int)nb1, vn_b1, (int)nb2, vn_b2, BT_STEP, &p.v_bc1, &p.v_bc2);
  if (rc) return rc;
  // q is vn itself when both address the same elements for every (image, head): then the kernel loads one tile per step
  const bool same_b1 = (q_b1 == 0 || nb1 == 1) ? (vn_b1 == 0 || nb1 == 1) : q_b1 == vn_b1;
  const bool same_b2 = (q_b2 == 0 || nb2 == 1) ? (vn_b2 == 0 || nb2 == 1) : q_b2 == vn_b2;
  p.q_is_vn = q == vn && q_ld == vn_ld && same_b1 && same_b2;
  if (p.q_is_vn) {
    mq = mv;
    p.q_bc1 = p.v_bc1;
    p.q_bc2 = p.v_bc2;
  } else {
    rc = make_operand_map(&mq, q, N, 256, q_ld, (int)nb1, q_b1, (int)nb2, q_b2, BT_STEP, &p.q_bc1, &p.q_bc2);
    if (rc) return rc;
  }
  MQ_REQUIRE((nb1 == 1 || o_b1 != 0) && (nb2 == 1 || o_b2 != 0), "biattn_text_vn: output batch strides must be non-zero");
  p.out = (__half*)out;
  p.o_ld = o_ld;
  p.o_b1 = o_b1;
  p.o_b2 = o_b2;
  p.stat = colmax;
  p.clamp = clamp;
  p.nb1 = (int)nb1;
  p.T = (int)T;
  p.N = (int)N;
  p.n_steps = (int)((N + BT_STEP - 1) / BT_STEP);
  p.rowbias = rowbias;
  p.rb_ld = (int)(rb_ld > 0 ? rb_ld : 1);
  dim3 grid((unsigned)((T + BT_ROWS - 1) / BT_ROWS), (unsigned)(nb1 * nb2));
  rc = ensure_dyn_smem(reinterpret_cast<const void*>(&biattn_text_kernel), BtCfg::SMEM_BYTES);
  if (rc) return rc;
  biattn_text_kernel<<<grid, 384, BtCfg::SMEM_BYTES, (cudaStream_t)stream>>>(mk, mq, mv, p);
  return check_launch("biattn_text_kernel");
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
  biattn_image_kernel<<<(unsigned)(p.tiles_per_img * B), 384, BiCfg::SMEM_BYTES, (cudaStream_t)stream>>>(mq, mk, mm, p);
  rc = check_launch("biattn_image_kernel");
  if (rc) return rc;
  colmax_reduce_kernel<<<(unsigned)(B * H), 256, 0, (cudaStream_t)stream>>>(workspace, p.tiles_per_img, (int)T, colmax);
  return check_launch("colmax_reduce_kernel");
}
