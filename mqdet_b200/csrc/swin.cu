// mqdet_b200 — Swin backbone / FPN data-movement and window-attention kernels (HBM-bound, coalesced NHWC rows).
//
// Reference: maskrcnn_benchmark/modeling/backbone/swint.py — PatchEmbed :393-431, window_partition/reverse :33-61,
//            WindowAttention.forward :111-142, SwinTransformerBlock.forward :186-242 (pad, cyclic shift, mask),
//            BasicLayer mask build :354-373, PatchMerging.forward :256-284;
//            maskrcnn_benchmark/modeling/backbone/fpn.py FPN.forward :59-129, LastLevelP6P7 :137-154;
//            generalized_vl_rcnn_new.py flatten_fpn_features :291-293 (AvgPool2d(2)).
// Token layout everywhere: [B][H*W][C], row-major (h, w).  The dense projections (qkv, proj, MLP, reductions, 1x1/3x3
// convolutions) run on the wgmma GEMM; these kernels only gather/scatter and do the 49x49 window attention.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

// image [B,3,H,W] fp32 NCHW -> patches [B*(H/4)*(W/4), 48] fp16, k = c*16 + i*4 + j (Conv2d(3,96,4,4) weight order);
// zero padding on the right/bottom when H or W is not a multiple of 4 (swint.py:413-418).
// One CTA per run of PF_TOK consecutive patches of a patch row: the 12 (channel, image row) segments of the run are read as
// float4s (consecutive threads -> consecutive 16-byte pieces of one image row), converted, transposed through shared memory
// and written as the run's contiguous [PF_TOK x 48] fp16 block with 16-byte stores.
constexpr int PF_TOK = 64;
__global__ void __launch_bounds__(256) patchify4_kernel(const float* __restrict__ img, int B, int H, int W, int Hp, int Wp,
                                                        __half* __restrict__ out) {
  __shared__ __align__(16) __half tile[PF_TOK * 48];
  const int runs = (Wp + PF_TOK - 1) / PF_TOK;
  const int run = blockIdx.x % runs;
  const int ph = (blockIdx.x / runs) % Hp, b = blockIdx.x / (runs * Hp);
  const int pw0 = run * PF_TOK, ntok = min(PF_TOK, Wp - pw0);
  const bool vec = (W & 3) == 0 && ((uintptr_t)img & 15) == 0;
  for (int i = threadIdx.x; i < 12 * PF_TOK; i += 256) {
    const int seg = i / PF_TOK, tkn = i - seg * PF_TOK;  // seg = c * 4 + ii
    if (tkn >= ntok) continue;
    const int c = seg >> 2, ii = seg & 3;
    const int y = ph * 4 + ii, x = (pw0 + tkn) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (y < H) {
      const float* src = img + (((long)b * 3 + c) * H + y) * W + x;
      if (vec && x + 3 < W) {
        v = __ldg(reinterpret_cast<const float4*>(src));
      } else {
        if (x < W) v.x = src[0];
        if (x + 1 < W) v.y = src[1];
        if (x + 2 < W) v.z = src[2];
        if (x + 3 < W) v.w = src[3];
      }
    }
    const __half2 lo = __floats2half2_rn(v.x, v.y), hi = __floats2half2_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<const uint32_t*>(&lo);
    o.y = *reinterpret_cast<const uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(tile + tkn * 48 + seg * 4) = o;
  }
  __syncthreads();
  uint4* dst = reinterpret_cast<uint4*>(out + (((long)b * Hp + ph) * Wp + pw0) * 48);  // 96 bytes per patch: 16-byte aligned
  const uint4* srcv = reinterpret_cast<const uint4*>(tile);
  for (int i = threadIdx.x; i < ntok * 6; i += 256) dst[i] = srcv[i];
}

// Window attention for one (window, head): head_dim 32, window WS x WS (N = 49 tokens for Swin-T, 144 for Swin-L).
// qkv [B*H*W, 3*C] fp16 (q | k | v, each C = heads*32 wide); bias_pad [heads][NP][NP] fp32 = log2(e) x relative position bias
// inside [N][N] and -inf outside (NP = N rounded up to 16): one FFMA per score applies scale, bias and key/query padding;
// padded tokens (beyond H/W after padding to a multiple of the window) carry qkv = qkv_bias because the reference
// pads the NORMALISED input with zeros before the qkv Linear (:200-205); cyclic shift + region mask (-100) are index math.
//
// One CTA (4 warps) per (window, head).  The window's q / k / v head slices (64 B per token each) are staged in shared
// memory with 16-byte loads (v transposed: the B fragments of P.V need two consecutive KEYS per register); warp w then
// takes the 16-query tiles w, w+4, ...: S = Q K^T and O = P V on mma.sync.m16n8k16 (fp16 in, fp32 accumulate — a
// 49x49x32 / 144x144x32 problem per head is far below a wgmma tile), softmax in the accumulator fragments (quad
// shuffles), P re-used as the A fragment of the second product (no shared-memory round trip).
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ uint32_t pack_h2(float x, float y) {
  __half2 h = __floats2half2_rn(x, y);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int WS>
struct SwinCfg {
  static constexpr int N = WS * WS;
  static constexpr int NP = (N + 15) / 16 * 16;   // tokens padded to whole 16-row query tiles / 16-key steps
  static constexpr int NT = NP / 8;               // key tiles of 8
  static constexpr int QLD = 40;                  // halfs per staged q / k row (32 + 8: conflict-free 4-byte fragment loads)
  static constexpr int VLD = NP + 8;              // halfs per staged v^T row
  static constexpr int SMEM = (2 * NP * QLD + 32 * VLD) * 2 + 2 * NP * 4;
};

template <int WS>
__global__ void __launch_bounds__(128) swin_window_attn_kernel(const __half* __restrict__ qkv, const float* __restrict__ qkv_bias,
                                                               const float* __restrict__ bias_pad, int B, int H, int W,
                                                               int heads, int shift, float scale, __half* __restrict__ out) {
  using Cfg = SwinCfg<WS>;
  constexpr int N = Cfg::N, D = 32, NP = Cfg::NP, NT = Cfg::NT, QLD = Cfg::QLD, VLD = Cfg::VLD;
  const int C = heads * D;
  const int Hp = (H + WS - 1) / WS * WS, Wp = (W + WS - 1) / WS * WS;
  const int nWw = Wp / WS, nW = (Hp / WS) * nWw;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long unit = blockIdx.x;  // (b, window, head), head fastest: the heads of a window read the same token rows
  const int head = (int)(unit % heads);
  const int win = (int)((unit / heads) % nW);
  const int b = (int)(unit / ((long)heads * nW));
  const int wi = win / nWw, wj = win % nWw;
  extern __shared__ __align__(16) uint8_t swin_smem[];
  __half* qs = reinterpret_cast<__half*>(swin_smem);   // [NP][QLD]
  __half* ks = qs + NP * QLD;                           // [NP][QLD]
  __half* vT = ks + NP * QLD;                           // [32][VLD]
  int* tok = reinterpret_cast<int*>(vT + 32 * VLD);     // [NP]
  int* reg = tok + NP;                                  // [NP]
  // region id of the window's first token (t = 0) — every thread evaluates it, the comparison below is per token
  int rg_first = 0;
  if (shift > 0) {
    const int hs = wi * WS, wsft = wj * WS;
    rg_first = ((hs < Hp - WS) ? 0 : ((hs < Hp - shift) ? 1 : 2)) * 3 + ((wsft < Wp - WS) ? 0 : ((wsft < Wp - shift) ? 1 : 2));
  }
  bool differs = false;
  for (int t = threadIdx.x; t < NP; t += 128) {
    int tk = -2, rg = 0;  // -2: beyond the window's tokens
    if (t < N) {
      const int r = t / WS, c = t % WS;
      const int hs = wi * WS + r, wsft = wj * WS + c;              // coordinate in the shifted, padded frame
      const int ho = (hs + shift) % Hp, wo = (wsft + shift) % Wp;  // un-shifted frame (roll by -shift)
      tk = (ho < H && wo < W) ? (ho * W + wo) : -1;                // -1: padding token (qkv = bias)
      if (shift > 0) {
        const int idh = (hs < Hp - WS) ? 0 : ((hs < Hp - shift) ? 1 : 2);
        const int idw = (wsft < Wp - WS) ? 0 : ((wsft < Wp - shift) ? 1 : 2);
        rg = idh * 3 + idw;
      }
    }
    tok[t] = tk;
    reg[t] = rg;
    differs |= (t < N && rg != rg_first);
  }
  // (the table is complete after this barrier) does any token of the window lie in another shift region than its first one?
  const bool masked = __syncthreads_or(differs ? 1 : 0) != 0;
  const __half* base = qkv + (long)b * H * W * 3 * C + head * D;
  // stage q | k | v of the window: 12 x 16-byte pieces per token (which = piece / 4, 8 dims each)
  for (int i = threadIdx.x; i < NP * 12; i += 128) {
    const int t = i / 12, piece = i - t * 12, which = piece >> 2, d0 = (piece & 3) * 8;
    const int tk = tok[t];
    uint4 v = make_uint4(0, 0, 0, 0);
    if (tk >= 0) {
      v = __ldg(reinterpret_cast<const uint4*>(base + (long)tk * 3 * C + which * C + d0));
    } else if (tk == -1) {
      const float* bp = qkv_bias + which * C + head * D + d0;
      v.x = pack_h2(bp[0], bp[1]); v.y = pack_h2(bp[2], bp[3]); v.z = pack_h2(bp[4], bp[5]); v.w = pack_h2(bp[6], bp[7]);
    }
    if (which == 0) {
      *reinterpret_cast<uint4*>(qs + t * QLD + d0) = v;
    } else if (which == 1) {
      *reinterpret_cast<uint4*>(ks + t * QLD + d0) = v;
    } else {
      const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
      for (int e = 0; e < 8; ++e) vT[(d0 + e) * VLD + t] = hv[e];
    }
  }
  __syncthreads();
  const int g = lane >> 2, t4 = lane & 3;
  const float* bd = bias_pad + (long)head * NP * NP;
  constexpr float L2E = 1.4426950408889634f;
  const float sc = scale * L2E;  // scores are kept in the log2 domain: exp(x) = ex2(x * log2 e)
#pragma unroll 1
  for (int mi = warp; mi * 16 < N; mi += 4) {
    const int r0 = 16 * mi + g, r1 = r0 + 8;  // the two query rows this lane holds
    uint32_t qf[2][4];
#pragma unroll
    for (int ki = 0; ki < 2; ++ki) {
      qf[ki][0] = *reinterpret_cast<const uint32_t*>(qs + r0 * QLD + 16 * ki + 2 * t4);
      qf[ki][1] = *reinterpret_cast<const uint32_t*>(qs + r1 * QLD + 16 * ki + 2 * t4);
      qf[ki][2] = *reinterpret_cast<const uint32_t*>(qs + r0 * QLD + 16 * ki + 2 * t4 + 8);
      qf[ki][3] = *reinterpret_cast<const uint32_t*>(qs + r1 * QLD + 16 * ki + 2 * t4 + 8);
    }
    float sacc[NT][4];
#pragma unroll
    for (int nj = 0; nj < NT; ++nj) {
#pragma unroll
      for (int e = 0; e < 4; ++e) sacc[nj][e] = 0.f;
      uint32_t kf0[2], kf1[2];
      kf0[0] = *reinterpret_cast<const uint32_t*>(ks + (8 * nj + g) * QLD + 2 * t4);
      kf0[1] = *reinterpret_cast<const uint32_t*>(ks + (8 * nj + g) * QLD + 2 * t4 + 8);
      kf1[0] = *reinterpret_cast<const uint32_t*>(ks + (8 * nj + g) * QLD + 16 + 2 * t4);
      kf1[1] = *reinterpret_cast<const uint32_t*>(ks + (8 * nj + g) * QLD + 16 + 2 * t4 + 8);
      mma_16816(sacc[nj], qf[0], kf0);
      mma_16816(sacc[nj], qf[1], kf1);
    }
    // scale + relative position bias + key / query padding in ONE FFMA per score (padded table entries are -inf); row max
    const float* b0p = bd + (long)r0 * NP + 2 * t4;
    const float* b1p = bd + (long)r1 * NP + 2 * t4;
    float mx0 = -1e30f, mx1 = -1e30f;  // finite floor: a fully padded query row gives exp2(-inf - (-1e30)) = 0, not NaN
#pragma unroll
    for (int nj = 0; nj < NT; ++nj) {
      const float2 ba = __ldg(reinterpret_cast<const float2*>(b0p + 8 * nj));
      const float2 bb = __ldg(reinterpret_cast<const float2*>(b1p + 8 * nj));
      sacc[nj][0] = fmaf(sacc[nj][0], sc, ba.x);
      sacc[nj][1] = fmaf(sacc[nj][1], sc, ba.y);
      sacc[nj][2] = fmaf(sacc[nj][2], sc, bb.x);
      sacc[nj][3] = fmaf(sacc[nj][3], sc, bb.y);
    }
    if (masked) {  // CTA-uniform: only windows that straddle the cyclic-shift seam carry the -100 region mask (:186-199)
      const int rg0 = reg[r0], rg1 = reg[r1];
#pragma unroll
      for (int nj = 0; nj < NT; ++nj)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = 8 * nj + 2 * t4 + (e & 1);
          if (reg[j] != ((e < 2) ? rg0 : rg1)) sacc[nj][e] += -100.0f * L2E;
        }
    }
#pragma unroll
    for (int nj = 0; nj < NT; ++nj) {
      mx0 = fmaxf(mx0, fmaxf(sacc[nj][0], sacc[nj][1]));
      mx1 = fmaxf(mx1, fmaxf(sacc[nj][2], sacc[nj][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
    for (int nj = 0; nj < NT; ++nj) {
      sacc[nj][0] = ex2_approx(sacc[nj][0] - mx0);
      sacc[nj][1] = ex2_approx(sacc[nj][1] - mx0);
      sacc[nj][2] = ex2_approx(sacc[nj][2] - mx1);
      sacc[nj][3] = ex2_approx(sacc[nj][3] - mx1);
      sum0 += sacc[nj][0] + sacc[nj][1];
      sum1 += sacc[nj][2] + sacc[nj][3];
    }
    sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1);
    sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
    sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1);
    sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
    // O = P V : P fragments come straight from the S accumulators (key tiles 2kj, 2kj+1 -> k-step kj)
    float oacc[4][4];
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) oacc[ni][e] = 0.f;
#pragma unroll
    for (int kj = 0; kj < NT / 2; ++kj) {
      uint32_t pf[4];
      pf[0] = pack_h2(sacc[2 * kj][0], sacc[2 * kj][1]);
      pf[1] = pack_h2(sacc[2 * kj][2], sacc[2 * kj][3]);
      pf[2] = pack_h2(sacc[2 * kj + 1][0], sacc[2 * kj + 1][1]);
      pf[3] = pack_h2(sacc[2 * kj + 1][2], sacc[2 * kj + 1][3]);
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        uint32_t vf[2];
        vf[0] = *reinterpret_cast<const uint32_t*>(vT + (8 * ni + g) * VLD + 16 * kj + 2 * t4);
        vf[1] = *reinterpret_cast<const uint32_t*>(vT + (8 * ni + g) * VLD + 16 * kj + 2 * t4 + 8);
        mma_16816(oacc[ni], pf, vf);
      }
    }
    const float inv0 = (sum0 > 0.f) ? 1.f / sum0 : 0.f, inv1 = (sum1 > 0.f) ? 1.f / sum1 : 0.f;
    const int tk0 = (r0 < N) ? tok[r0] : -2, tk1 = (r1 < N) ? tok[r1] : -2;
#pragma unroll
    for (int ni = 0; ni < 4; ++ni) {
      const int d = 8 * ni + 2 * t4;
      if (tk0 >= 0)  // outputs at padded positions are cropped away (:231-232)
        *reinterpret_cast<uint32_t*>(out + ((long)b * H * W + tk0) * C + head * D + d) = pack_h2(oacc[ni][0] * inv0, oacc[ni][1] * inv0);
      if (tk1 >= 0)
        *reinterpret_cast<uint32_t*>(out + ((long)b * H * W + tk1) * C + head * D + d) = pack_h2(oacc[ni][2] * inv1, oacc[ni][3] * inv1);
    }
  }
}

// PatchMerging gather + LayerNorm(4C) (:256-284): out row (b, h2, w2) = LN(cat[x(2h2,2w2), x(2h2+1,2w2), x(2h2,2w2+1),
// x(2h2+1,2w2+1)]) with zero rows outside (odd H/W padding).  x fp32 [B, H*W, C] -> fp16 [B*H2*W2, 4C]. Warp per row.
__global__ void __launch_bounds__(256) patch_merge_ln_kernel(const float* __restrict__ x, int B, int H, int W, int C,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             float eps, __half* __restrict__ out) {
  const int H2 = (H + 1) / 2, W2 = (W + 1) / 2;
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= (long)B * H2 * W2) return;
  const int w2 = (int)(row % W2), h2 = (int)((row / W2) % H2), b = (int)(row / ((long)W2 * H2));
  const int D4 = 4 * C;
  auto src = [&](int i) -> float {
    const int q = i / C, c = i % C;
    const int hh = 2 * h2 + (q & 1), ww = 2 * w2 + (q >> 1);
    return (hh < H && ww < W) ? x[((long)b * H * W + (long)hh * W + ww) * C + c] : 0.f;
  };
  float s = 0.f;
  for (int i = lane; i < D4; i += 32) s += src(i);
  const float mean = warp_sum(s) / D4;
  float v = 0.f;
  for (int i = lane; i < D4; i += 32) {
    const float d = src(i) - mean;
    v += d * d;
  }
  const float rstd = rsqrtf(warp_sum(v) / D4 + eps);
  for (int i = lane; i < D4; i += 32) out[row * D4 + i] = __float2half_rn((src(i) - mean) * rstd * gamma[i] + beta[i]);
}

// The same, register-cached and vectorised for C = 32 * K4 (Swin-T/L stages: 96, 192, 384): the 4C-float row is read ONCE as
// float4s (lane l owns float4 #(l + 32 i); a float4 never straddles two of the four source pixels because C % 4 == 0) and
// written as 8-byte fp16 groups.  Same two-pass statistics in fp32.
template <int K4>
__global__ void __launch_bounds__(256) patch_merge_ln_vec_kernel(const float* __restrict__ x, int B, int H, int W,
                                                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                 float eps, __half* __restrict__ out) {
  constexpr int C = 32 * K4, C4 = C / 4, D4 = 4 * C;
  const int H2 = (H + 1) / 2, W2 = (W + 1) / 2;
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= (long)B * H2 * W2) return;
  const int w2 = (int)(row % W2), h2 = (int)((row / W2) % H2), b = (int)(row / ((long)W2 * H2));
  float4 v[K4];
#pragma unroll
  for (int i = 0; i < K4; ++i) {
    const int f = lane + 32 * i, q = f / C4, c4 = f - q * C4;
    const int hh = 2 * h2 + (q & 1), ww = 2 * w2 + (q >> 1);
    v[i] = (hh < H && ww < W) ? __ldg(reinterpret_cast<const float4*>(x + ((long)b * H * W + (long)hh * W + ww) * C) + c4)
                              : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < K4; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / D4;
  float qv = 0.f;
#pragma unroll
  for (int i = 0; i < K4; ++i) {
    const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    qv += (a * a + bb * bb) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(qv) / D4 + eps);
#pragma unroll
  for (int i = 0; i < K4; ++i) {
    const int f = lane + 32 * i;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + f), bt = __ldg(reinterpret_cast<const float4*>(beta) + f);
    const __half2 lo = __floats2half2_rn((v[i].x - mean) * rstd * g.x + bt.x, (v[i].y - mean) * rstd * g.y + bt.y);
    const __half2 hi = __floats2half2_rn((v[i].z - mean) * rstd * g.z + bt.z, (v[i].w - mean) * rstd * g.w + bt.w);
    uint2 o;
    o.x = *reinterpret_cast<const uint32_t*>(&lo);
    o.y = *reinterpret_cast<const uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(out + row * D4 + 4 * f) = o;
  }
}

// FPN top-down merge (fpn.py:88-95): out = lateral + nearest_upsample(top).  fp16 rows of C=256, warp per pixel.
__global__ void __launch_bounds__(256) upsample_add_kernel(const __half* __restrict__ lateral, const __half* __restrict__ top,
                                                           int B, int H, int W, int Hs, int Ws, int C,
                                                           __half* __restrict__ out) {
  const long gw = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= (long)B * H * W) return;
  const int w = (int)(gw % W), h = (int)((gw / W) % H), b = (int)(gw / ((long)W * H));
  // F.interpolate(mode="nearest"): src = floor(dst * in / out) computed in fp32 like ATen
  const int hs = min((int)floorf(h * ((float)Hs / (float)H)), Hs - 1);
  const int ws = min((int)floorf(w * ((float)Ws / (float)W)), Ws - 1);
  const __half* lp = lateral + gw * C;
  const __half* tp = top + ((long)b * Hs * Ws + (long)hs * Ws + ws) * C;
  for (int c = lane * 8; c < C; c += 256) {
    const uint4 a = *reinterpret_cast<const uint4*>(lp + c);
    const uint4 t4 = *reinterpret_cast<const uint4*>(tp + c);
    const __half2* ah = reinterpret_cast<const __half2*>(&a);
    const __half2* th = reinterpret_cast<const __half2*>(&t4);
    __half2 o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = __half22float2(ah[i]), y = __half22float2(th[i]);
      o[i] = __floats2half2_rn(x.x + y.x, x.y + y.y);
    }
    *reinterpret_cast<uint4*>(out + gw * C + c) = *reinterpret_cast<uint4*>(o);
  }
}

// Plain 3x3 / pad 1 / stride s im2col of an fp16 NHWC map [B][H*W][C] (arbitrary batch stride) -> cols [B*Ho*Wo][9*C],
// k = tap*C + c; optional ReLU on the input (LastLevelP6P7: p7 = conv(relu(p6)), fpn.py:152).  Warp per (pixel, tap).
__global__ void __launch_bounds__(256) im2col3x3_kernel(const __half* __restrict__ x, long x_batch_stride, int B, int H, int W,
                                                        int C, int stride, int relu_in, __half* __restrict__ cols) {
  const int Ho = (H + 2 - 3) / stride + 1, Wo = (W + 2 - 3) / stride + 1;
  const long gw = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= (long)B * Ho * Wo * 9) return;
  const int tap = (int)(gw % 9);
  const long r = gw / 9;
  const int wo = (int)(r % Wo), ho = (int)((r / Wo) % Ho), b = (int)(r / ((long)Wo * Ho));
  const int hi = ho * stride - 1 + tap / 3, wi = wo * stride - 1 + tap % 3;
  const bool ok = hi >= 0 && hi < H && wi >= 0 && wi < W;
  const __half* src = x + (long)b * x_batch_stride + ((long)hi * W + wi) * C;
  __half* dst = cols + (r * 9 + tap) * C;
  for (int c = lane * 8; c < C; c += 256) {
    uint4 v = make_uint4(0, 0, 0, 0);
    if (ok) {
      v = *reinterpret_cast<const uint4*>(src + c);
      if (relu_in) {
        __half2* h = reinterpret_cast<__half2*>(&v);
        const __half2 z = __float2half2_rn(0.f);
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = __hmax2(h[i], z);
      }
    }
    *reinterpret_cast<uint4*>(dst + c) = v;
  }
}

// AvgPool2d(2) (floor) of every level of the concatenated pyramid -> concatenated pooled tokens, fp16 -> fp32.
struct PoolLevels {
  int n;
  int H[MQDET_MAX_LEVELS], W[MQDET_MAX_LEVELS], off[MQDET_MAX_LEVELS], ooff[MQDET_MAX_LEVELS + 1];
};
__global__ void __launch_bounds__(256) avgpool2_levels_kernel(const __half* __restrict__ x, PoolLevels lv, int B, int N, int C,
                                                              float* __restrict__ out) {
  const long gw = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int I = lv.ooff[lv.n];
  if (gw >= (long)B * I) return;
  const int b = (int)(gw / I), q = (int)(gw % I);
  int l = 0;
  while (l + 1 < lv.n && q >= lv.ooff[l + 1]) ++l;
  const int W2 = lv.W[l] / 2;
  const int p = q - lv.ooff[l];
  const int h2 = p / W2, w2 = p % W2;
  const __half* base = x + ((long)b * N + lv.off[l]) * C;
  for (int c = lane; c < C; c += 32) {
    float s = 0.f;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) s += __half2float(base[((long)(2 * h2 + dy) * lv.W[l] + 2 * w2 + dx) * C + c]);
    out[gw * C + c] = s * 0.25f;
  }
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_patchify4(const float* img, int64_t B, int64_t H, int64_t W, void* out, void* stream) {
  MQ_REQUIRE(img && out && B > 0 && H > 0 && W > 0, "patchify4: bad args");
  const int Hp = (int)((H + 3) / 4), Wp = (int)((W + 3) / 4);
  const long blocks = B * Hp * ((Wp + PF_TOK - 1) / PF_TOK);
  MQ_REQUIRE(blocks < 2147483647L && ((uintptr_t)out & 15) == 0, "patchify4: output must be 16-byte aligned");
  patchify4_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(img, (int)B, (int)H, (int)W, Hp, Wp, (__half*)out);
  return check_launch("patchify4_kernel");
}

extern "C" int mqdet_swin_window_attn(const void* qkv, const float* qkv_bias, const float* bias_pad, int64_t B, int64_t H,
                                      int64_t W, int64_t heads, int64_t window, int64_t shift, float scale, void* out,
                                      void* stream) {
  MQ_REQUIRE(qkv && qkv_bias && bias_pad && out, "swin_window_attn: null pointer");
  MQ_REQUIRE(((uintptr_t)bias_pad & 7) == 0, "swin_window_attn: bias_pad must be 8-byte aligned");
  MQ_REQUIRE(window == 7 || window == 12, "swin_window_attn: window 7 (Swin-T) or 12 (Swin-L), got %ld", (long)window);
  MQ_REQUIRE(shift >= 0 && shift < window, "swin_window_attn: bad shift");
  MQ_REQUIRE(((uintptr_t)qkv % 16) == 0 && (heads * 32 * 3) % 8 == 0, "swin_window_attn: qkv must be 16-byte aligned");
  const int Hp = (int)((H + window - 1) / window * window), Wp = (int)((W + window - 1) / window * window);
  const int nW = (Hp / (int)window) * (Wp / (int)window);
  const long units = B * (long)nW * heads;
  MQ_REQUIRE(units < 2147483647L, "swin_window_attn: too many (window, head) units");
  dim3 grid((unsigned)units);
  if (window == 7) {
    swin_window_attn_kernel<7><<<grid, 128, SwinCfg<7>::SMEM, (cudaStream_t)stream>>>(
        (const __half*)qkv, qkv_bias, bias_pad, (int)B, (int)H, (int)W, (int)heads, (int)shift, scale, (__half*)out);
  } else {
    swin_window_attn_kernel<12><<<grid, 128, SwinCfg<12>::SMEM, (cudaStream_t)stream>>>(
        (const __half*)qkv, qkv_bias, bias_pad, (int)B, (int)H, (int)W, (int)heads, (int)shift, scale, (__half*)out);
  }
  return check_launch("swin_window_attn_kernel");
}

extern "C" int mqdet_patch_merge_ln(const float* x, int64_t B, int64_t H, int64_t W, int64_t C, const float* gamma,
                                    const float* beta, float eps, void* out, void* stream) {
  MQ_REQUIRE(x && gamma && beta && out, "patch_merge_ln: null pointer");
  const long rows = B * ((H + 1) / 2) * ((W + 1) / 2);
  const bool al = (((uintptr_t)x | (uintptr_t)gamma | (uintptr_t)beta) & 15) == 0 && ((uintptr_t)out & 7) == 0;
  cudaStream_t st = (cudaStream_t)stream;
#define MQ_PM(K4)                                                                                                             \
  patch_merge_ln_vec_kernel<K4><<<cdiv(rows, 8), 256, 0, st>>>(x, (int)B, (int)H, (int)W, gamma, beta, eps, (__half*)out)
  if (al && C == 96) MQ_PM(3);
  else if (al && C == 192) MQ_PM(6);
  else if (al && C == 384) MQ_PM(12);
  else
    patch_merge_ln_kernel<<<cdiv(rows, 8), 256, 0, st>>>(x, (int)B, (int)H, (int)W, (int)C, gamma, beta, eps, (__half*)out);
#undef MQ_PM
  return check_launch("patch_merge_ln_kernel");
}

extern "C" int mqdet_upsample_add(const void* lateral, const void* top, int64_t B, int64_t H, int64_t W, int64_t Hs,
                                  int64_t Ws, int64_t C, void* out, void* stream) {
  MQ_REQUIRE(lateral && top && out && (C % 8) == 0, "upsample_add: bad args");
  const long warps = B * H * W;
  upsample_add_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)lateral, (const __half*)top, (int)B, (int)H, (int)W, (int)Hs, (int)Ws, (int)C, (__half*)out);
  return check_launch("upsample_add_kernel");
}

extern "C" int mqdet_im2col3x3(const void* x, int64_t x_batch_stride, int64_t B, int64_t H, int64_t W, int64_t C,
                               int64_t stride, int relu_in, void* cols, void* stream) {
  MQ_REQUIRE(x && cols && (C % 8) == 0 && (stride == 1 || stride == 2), "im2col3x3: bad args");
  const int Ho = (int)((H + 2 - 3) / stride + 1), Wo = (int)((W + 2 - 3) / stride + 1);
  const long warps = B * Ho * Wo * 9;
  im2col3x3_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)x, x_batch_stride, (int)B, (int)H, (int)W, (int)C, (int)stride, relu_in, (__half*)cols);
  return check_launch("im2col3x3_kernel");
}

extern "C" int mqdet_avgpool2_levels(const void* x, const int32_t* level_hw, int64_t nlev, int64_t B, int64_t C, float* out,
                                     void* stream) {
  MQ_REQUIRE(x && level_hw && out && nlev >= 1 && nlev <= MQDET_MAX_LEVELS, "avgpool2_levels: bad args");
  PoolLevels lv;
  lv.n = (int)nlev;
  int off = 0, ooff = 0;
  for (int l = 0; l < nlev; ++l) {
    lv.H[l] = level_hw[2 * l];
    lv.W[l] = level_hw[2 * l + 1];
    lv.off[l] = off;
    lv.ooff[l] = ooff;
    off += lv.H[l] * lv.W[l];
    ooff += (lv.H[l] / 2) * (lv.W[l] / 2);
  }
  lv.ooff[nlev] = ooff;
  const long warps = B * ooff;
  avgpool2_levels_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x, lv, (int)B,
                                                                                                off, (int)C, out);
  return check_launch("avgpool2_levels_kernel");
}
