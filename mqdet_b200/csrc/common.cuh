// mqdet_b200 — shared device/host helpers for the sm_90a kernels.
// PTX wrappers (mbarrier, TMA, wgmma) are written out here so the kernels read as plain CUDA.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#define MQDET_OK 0
#define MQDET_ERR_ARG -1
#define MQDET_ERR_CUDA -2
#define MQDET_ERR_UNSUPPORTED -3

namespace mqdet {

// thread-local last error string (exposed through mqdet_last_error()).
void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define MQ_REQUIRE(cond, ...)                      \
  do {                                             \
    if (!(cond)) {                                 \
      mqdet::set_error(__VA_ARGS__);               \
      return MQDET_ERR_ARG;                        \
    }                                              \
  } while (0)

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// All FPN levels of an image live in one tensor x[B][N][C] (level l at row offset off_l, row-major (h, w)).
#ifndef MQDET_MAX_LEVELS
#define MQDET_MAX_LEVELS 8
#endif
struct LevelTable {
  int n;
  int H[MQDET_MAX_LEVELS], W[MQDET_MAX_LEVELS], off[MQDET_MAX_LEVELS];
};
static inline int fill_levels(LevelTable* t, const int32_t* hw, int64_t nlev) {
  if (nlev < 1 || nlev > MQDET_MAX_LEVELS) return -1;
  t->n = (int)nlev;
  int off = 0;
  for (int l = 0; l < nlev; ++l) {
    t->H[l] = hw[2 * l];
    t->W[l] = hw[2 * l + 1];
    t->off[l] = off;
    off += t->H[l] * t->W[l];
  }
  return off;
}

// host helpers of the TMA / wgmma kernels (capi.cu): cached TMA tensor maps, per-device SM count / shared-memory opt-in
int make_operand_map(CUtensorMap* map, const void* ptr, long rows, long K, long ld, int nb1, long s1, int nb2, long s2,
                     int box_rows, int* bcast1, int* bcast2);
int make_store_map(CUtensorMap* map, void* C, int c_dtype, long M, long N, long ldc, int nb1, long c_b1, int nb2, long c_b2);
int num_sms();
int ensure_dyn_smem(const void* func, int bytes);

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

// erf-GELU in ~18 issue slots (no branches): erfc(|z|) = t * P4(t) * exp(-z^2), t = 1 / (1 + 0.3275911 |z|)
// (Abramowitz-Stegun 7.1.26, |abs err| < 1.5e-7), and 1 + erf(z) = erfc(|z|) for z < 0 (no cancellation), 2 - erfc(z) else.
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = x * 0.70710678118654752440f;
  const float az = fabsf(z);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, az, 1.f)));
  float q = fmaf(1.061405429f, t, -1.453152027f);
  q = fmaf(q, t, 1.421413741f);
  q = fmaf(q, t, -0.284496736f);
  q = fmaf(q, t, 0.254829592f);
  const float e = q * t * __expf(-az * az);
  return 0.5f * x * (z < 0.f ? e : 2.f - e);
}

// ---- mbarrier ------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// explicit shared-space 128-bit accesses on 32-bit addresses (pointers derived from the aligned dynamic-smem base are
// otherwise compiled as generic LD.E/ST.E with 64-bit address arithmetic)
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ float4 lds128f(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ float ex2_approx(float x) {  // one MUFU.EX2 (flushes results below 2^-126 to zero)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float x, float y) {
  const __half2 h = __floats2half2_rn(x, y);
  return *reinterpret_cast<const uint32_t*>(&h);
}
// (d0, d1) = (a0, a1) * s + (b0, b1): two fused multiply-adds
__device__ __forceinline__ void ffma2(float& d0, float& d1, float a0, float a1, float s, float b0, float b1) {
  d0 = fmaf(a0, s, b0);
  d1 = fmaf(a1, s, b1);
}
// (d0, d1) = (a0, a1) * (s0, s1) + (b0, b1)
__device__ __forceinline__ void ffma2v(float& d0, float& d1, float a0, float a1, float s0, float s1, float b0, float b1) {
  d0 = fmaf(a0, s0, b0);
  d1 = fmaf(a1, s1, b1);
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}

// ---- TMA (cp.async.bulk.tensor) ------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 4-D tiled load, coordinates innermost-first.
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// L2 prefetch of a 4-D tile (no shared-memory destination, no completion tracking)
__device__ __forceinline__ void tma_prefetch_l2_4d(const CUtensorMap* m, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}

// 4-D tiled store shared -> global (bulk group completion); out-of-bounds parts of the box are clipped by the TMA unit.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit_and_wait_read1() {  // leave the newest group in flight
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_read_all() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void tma_store_commit_and_wait_read() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// ---- wgmma (sm_90a warpgroup MMA) -----------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major, 128-byte-swizzled shared-memory matrix descriptor (8-row groups 1024 B apart; the tile base 1024-aligned).
//   bits [0,14) start address >> 4   bits [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1)
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout: 1 = SWIZZLE_128B
// Advancing the start address by 32 B steps 16 fp16 along K inside the swizzle row.
__device__ __forceinline__ uint64_t wg_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// MN-major (the M / N index is the contiguous one), 128-byte-swizzled: the swizzle atom is 64 MN elements (128 B) x 8 K rows;
// `lbo` = byte distance between atoms along MN (next 64 elements), `sbo` = between atoms along K (next 8 rows).
__device__ __forceinline__ uint64_t wg_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// Accumulator fragment of a 64 x N wgmma: thread t of the warpgroup holds d[i] at
//   row = 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),   col = 8 * (i / 4) + 2 * (t % 4) + (i % 2)
__device__ __forceinline__ int wg_row(int t, int i) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int wg_col(int t, int i) { return 8 * (i >> 2) + 2 * (t & 3) + (i & 1); }

// erf-GELU of TWO values: the same Abramowitz-Stegun 7.1.26 form as gelu_fast,
//   gelu(x) = 0.5 (x + |x| (1 - erfc(|z|))),  z = x / sqrt(2),  erfc(|z|) = t P4(t) exp(-z^2),  t = 1 / (1 + 0.3275911 |z|),
// with z pre-scaled by sqrt(log2 e) so that exp(-z^2) is one MUFU.EX2 of -(z')^2.  ~10 issue slots per value instead of ~17:
// the GELU epilogues of the K <= 384 MLP GEMMs (Swin fc1, FFNs) are issue-bound on the eight epilogue warps.
__device__ __forceinline__ void gelu_fast2(float& x0, float& x1) {
  constexpr float SL = 1.2011224087864498f;                 // sqrt(log2(e))
  constexpr float C = 0.70710678118654752440f * SL;          // x -> z' = x / sqrt(2) * sqrt(log2 e)
  constexpr float P = 0.3275911f / SL;
  const float a0 = fabsf(x0), a1 = fabsf(x1);
  float z0, z1, d0, d1, q0, q1, w0, w1, e0, e1, u0, u1, h0, h1;
  ffma2(z0, z1, a0, a1, C, 0.f, 0.f);                         // |z'|
  ffma2(d0, d1, z0, z1, P, 1.f, 1.f);                         // 1 + 0.3275911 |z|
  float t0, t1;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(d0));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(d1));
  ffma2(q0, q1, t0, t1, 1.061405429f, -1.453152027f, -1.453152027f);
  ffma2v(q0, q1, q0, q1, t0, t1, 1.421413741f, 1.421413741f);
  ffma2v(q0, q1, q0, q1, t0, t1, -0.284496736f, -0.284496736f);
  ffma2v(q0, q1, q0, q1, t0, t1, 0.254829592f, 0.254829592f);
  ffma2v(w0, w1, z0, z1, z0, z1, 0.f, 0.f);                   // (z')^2 = z^2 log2 e
  e0 = ex2_approx(-w0);
  e1 = ex2_approx(-w1);
  ffma2v(q0, q1, q0, q1, t0, t1, 0.f, 0.f);                   // t P4(t)
  ffma2v(e0, e1, q0, q1, e0, e1, 0.f, 0.f);                   // erfc(|z|)
  ffma2v(u0, u1, -a0, -a1, e0, e1, a0, a1);                   // |x| (1 - erfc)
  ffma2(h0, h1, x0, x1, 0.5f, 0.f, 0.f);
  ffma2(x0, x1, u0, u1, 0.5f, h0, h1);                        // 0.5 x + 0.5 |x| (1 - erfc)
}

}  // namespace mqdet
