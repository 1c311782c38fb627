// mqdet_b200 — DyHead vision-path kernels (DyConv = DCNv2 x3 + GroupNorm + scale-attention + DyReLU), NHWC.
//
// Reference: maskrcnn_benchmark/modeling/rpn/vldyhead.py DyConv.forward :205-247, Conv3x3Norm :111-152;
//            maskrcnn_benchmark/csrc/cuda/deform_conv_kernel_cuda.cu :473-505 (bilinear), :578-641 (im2col);
//            maskrcnn_benchmark/layers/dyrelu.py :80-120.
//
// Layout: all FPN levels of an image live in one fp16 tensor x[B][N][C] (N = sum_l H_l*W_l, level l at row offset
// off_l, row-major (h, w)); every kernel below walks ALL levels in one launch through a LevelTable.
// The DCNv2 sampling stage writes an fp16 column matrix [rows][9*C] (k = tap*C + c) that feeds the wgmma GEMM.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

__device__ __forceinline__ void ld8h(const __half* p, float (&f)[8]) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&a);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 x = __half22float2(h[i]);
    f[2 * i] = x.x;
    f[2 * i + 1] = x.y;
  }
}
__device__ __forceinline__ void ld8f(const float* p, float (&f)[8]) {  // 32-byte aligned
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void st8h(__half* p, const float (&f)[8]) {
  __half2 h[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = *reinterpret_cast<uint4*>(h);
}

// ---------------------------------------------------------------------------------------------------------------
// DCNv2 / plain 3x3 sampling -> column matrix.   One warp per output pixel (9 taps); lanes across C (8 ch / lane).
// branch 1: input level l -> output level l, stride 1   (rows: all levels, N per image)
// branch 2: input level l-1 -> output level l, stride 2 (rows: levels 1..L-1)
// branch 0: input level l+1, output at level l+1's size, offsets/mask of level l re-read through the OUTPUT strides
//           (deform_conv_kernel_cuda.cu:605-618; rows: "virtual" levels 1..L-1 sized like the inputs)
// om: [B][N][OM_LD] fp32 pixel-major offset/mask logits (27 used: 18 offsets (dh,dw per tap), 9 mask logits);
//     om == nullptr -> plain 3x3 convolution sampling (zero offsets, mask 1).
// The reference indexes a per-(image, level) NCHW-flat buffer [27][H_l*W_l]; flat index f of the offset part maps to
// (channel f / HW_l, pixel f % HW_l), and of the (separately materialised, sigmoid-ed) mask part to channel 18 + f / HW_l.
// ---------------------------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256) dcn_cols_kernel(const __half* __restrict__ x, const float* __restrict__ om,
                                                       int om_ld, LevelTable lt, int branch, int B, long rows_per_img,
                                                       __half* __restrict__ cols) {
  // one warp per OUTPUT PIXEL, looping over the 9 taps: the level lookup / coordinate arithmetic is done once, the 27
  // offset/mask values of the pixel are fetched by 27 lanes in one request and broadcast with shuffles.
  const long r = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= (long)B * rows_per_img) return;
  const int b = (int)(r / rows_per_img);
  int q = (int)(r % rows_per_img);
  const int N = lt.off[lt.n - 1] + lt.H[lt.n - 1] * lt.W[lt.n - 1];
  int lo, li, Ho, Wo, stride;
  if (branch == 1) {
    int l = 0;
    while (l + 1 < lt.n && q >= lt.off[l + 1]) ++l;
    q -= lt.off[l];
    lo = l; li = l; Ho = lt.H[l]; Wo = lt.W[l]; stride = 1;
  } else {
    int l = 1;
    const int base = lt.off[1];
    while (l + 1 < lt.n && q + base >= lt.off[l + 1]) ++l;
    q -= lt.off[l] - base;
    Ho = lt.H[l]; Wo = lt.W[l];
    if (branch == 2) { lo = l; li = l - 1; stride = 2; }
    else { lo = l - 1; li = l; stride = 1; }
  }
  const int ho = q / Wo, wo = q % Wo;
  const int Hi = lt.H[li], Wi = lt.W[li];
  // lane c < 27 fetches channel c of this pixel's offset/mask record (flat NCHW index c*HWo + pix re-read through the
  // strides of the level the buffer was produced at)
  float omv = 0.f;
  if (om && lane < 27) {
    const int HWl = lt.H[lo] * lt.W[lo];
    const int HWo = Ho * Wo, pix = ho * Wo + wo;
    const float* omb = om + ((long)b * N + lt.off[lo]) * om_ld;
    if (lane < 18) {
      const int f = lane * HWo + pix;
      omv = omb[(long)(f % HWl) * om_ld + f / HWl];
    } else {
      const int f = (lane - 18) * HWo + pix;
      const float ml = omb[(long)(f % HWl) * om_ld + 18 + f / HWl];
      omv = 1.f / (1.f + expf(-ml));
    }
  }
  const __half* xb = x + ((long)b * N + lt.off[li]) * C + lane * 8;
  __half* dst = cols + r * 9 * C + lane * 8;
  // All four corner rows of a tap are fetched unconditionally (indices clamped into the map, invalid corners get weight 0)
  // and three taps are in flight at a time: 12 independent 16-byte loads per lane instead of one load -> use -> next load.
#pragma unroll 3
  for (int tap = 0; tap < 9; ++tap) {
    float off_h = 0.f, off_w = 0.f, m = 1.f;
    if (om) {
      off_h = __shfl_sync(0xffffffffu, omv, 2 * tap);
      off_w = __shfl_sync(0xffffffffu, omv, 2 * tap + 1);
      m = __shfl_sync(0xffffffffu, omv, 18 + tap);
    }
    const float h_im = (float)(ho * stride - 1 + tap / 3) + off_h;
    const float w_im = (float)(wo * stride - 1 + tap % 3) + off_w;
    const bool inside = h_im > -1.f && w_im > -1.f && h_im < (float)Hi && w_im < (float)Wi;
    const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
    const int h_high = h_low + 1, w_high = w_low + 1;
    const float lh = h_im - h_low, lw = w_im - w_low, hh = 1.f - lh, hw = 1.f - lw;
    const bool hl_ok = inside && h_low >= 0, hh_ok = inside && h_high <= Hi - 1;
    const bool wl_ok = w_low >= 0, wh_ok = w_high <= Wi - 1;
    const float w1 = (hl_ok && wl_ok) ? hh * hw : 0.f, w2 = (hl_ok && wh_ok) ? hh * lw : 0.f;
    const float w3 = (hh_ok && wl_ok) ? lh * hw : 0.f, w4 = (hh_ok && wh_ok) ? lh * lw : 0.f;
    const int hl = min(max(h_low, 0), Hi - 1), hh_i = min(max(h_high, 0), Hi - 1);
    const int wl = min(max(w_low, 0), Wi - 1), wh_i = min(max(w_high, 0), Wi - 1);
    float v1[8], v2[8], v3[8], v4[8];
    ld8h(xb + (long)(hl * Wi + wl) * C, v1);
    ld8h(xb + (long)(hl * Wi + wh_i) * C, v2);
    ld8h(xb + (long)(hh_i * Wi + wl) * C, v3);
    ld8h(xb + (long)(hh_i * Wi + wh_i) * C, v4);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      // same accumulation order as before (corner 1..4, then the mask): identical results; a zero weight contributes 0
      float a = w1 * v1[i];
      a += w2 * v2[i];
      a += w3 * v3[i];
      a += w4 * v4[i];
      acc[i] = a * m;
    }
    st8h(dst + tap * C, acc);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Per-(image, segment) per-channel statistics of an fp16 [rows, C] matrix: sum, sum of squares, weighted sum.
// Segments are contiguous row ranges (one per level); deterministic two-stage reduction (no atomics):
//   stage 1: grid (chunks, segments*B) -> partial[b][seg][chunk][3][C]      stage 2: folded into the consumers.
// rw: optional per-row weights (bilinear-upsample GAP weights for the DyConv[0] branch), else weighted sum == sum.
// ---------------------------------------------------------------------------------------------------------------
constexpr int STAT_CHUNKS = 32;

template <int C>
__global__ void __launch_bounds__(256) chan_stats_kernel(const __half* __restrict__ y, const int* __restrict__ seg_off,
                                                         int nseg, long rows_per_img, const float* __restrict__ rw,
                                                         float* __restrict__ partial) {
  // block = 256 threads = 8 row-lanes x 32 channel-lanes (8 channels each)
  const int chunk = blockIdx.x, sb = blockIdx.y;
  const int b = sb / nseg, seg = sb % nseg;
  const int r0 = seg_off[seg], r1 = seg_off[seg + 1];
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  float s[8], q[8], w[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = q[i] = w[i] = 0.f;
  // four independent 16-byte loads in flight per thread (level 0 gives each thread ~65 rows: one load at a time left the
  // kernel latency-bound at ~2.5 TB/s); the order of the additions per accumulator is unchanged
  constexpr int STEP = STAT_CHUNKS * 8;
  const __half* yb = y + (long)b * rows_per_img * C + cl * 8;
  int r = r0 + chunk * 8 + rl;
  for (; r + 3 * STEP < r1; r += 4 * STEP) {
    uint4 u[4];
    float wt[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      u[k] = *reinterpret_cast<const uint4*>(yb + (long)(r + k * STEP) * C);
      wt[k] = rw ? rw[r + k * STEP] : 1.f;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const __half2* h = reinterpret_cast<const __half2*>(&u[k]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(h[i]);
        s[2 * i] += f.x;
        s[2 * i + 1] += f.y;
        q[2 * i] += f.x * f.x;
        q[2 * i + 1] += f.y * f.y;
        w[2 * i] += wt[k] * f.x;
        w[2 * i + 1] += wt[k] * f.y;
      }
    }
  }
  for (; r < r1; r += STEP) {
    float v[8];
    ld8h(yb + (long)r * C, v);
    const float wt = rw ? rw[r] : 1.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i] += v[i];
      q[i] += v[i] * v[i];
      w[i] += wt * v[i];
    }
  }
  __shared__ float sh[8][3][C];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sh[rl][0][cl * 8 + i] = s[i];
    sh[rl][1][cl * 8 + i] = q[i];
    sh[rl][2][cl * 8 + i] = w[i];
  }
  __syncthreads();
  float* out = partial + (((long)b * nseg + seg) * STAT_CHUNKS + chunk) * 3 * C;
  for (int i = threadIdx.x; i < 3 * C; i += 256) {
    const int k = i / C, c = i % C;
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += sh[j][k][c];
    out[i] = t;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm parameters + scale-attention scalar per (image, segment)   [vldyhead.py:226-238]
//   partial stats -> per-group mu/rstd -> per-channel affine (ga, gb) with GN(y)[c] = ga[c]*y + gb[c]
//   GAP(fea)[c] = ga[c]*mean_w(y)[c] + gb[c]  (mean_w = plain mean, or the bilinear-upsample-weighted mean for the
//   DyConv[0] branch whose feature is upsampled AFTER the norm);  attn = h_sigmoid(relu(w_attn . GAP + b_attn))
// One block (C threads = channels) per (b, seg).  out: affine[b][seg][2][C], attn[b][seg].
// ---------------------------------------------------------------------------------------------------------------
template <int C, int G>
__global__ void __launch_bounds__(C) gn_attn_kernel(const float* __restrict__ partial, const int* __restrict__ seg_off,
                                                    int nseg, int weighted, const float* __restrict__ gn_w,
                                                    const float* __restrict__ gn_b, float eps,
                                                    const float* __restrict__ attn_w, const float* __restrict__ attn_b,
                                                    float* __restrict__ affine, float* __restrict__ attn) {
  const int sb = blockIdx.x, seg = sb % nseg;
  const int c = threadIdx.x;
  const float* p = partial + (long)sb * STAT_CHUNKS * 3 * C;
  float s = 0.f, q = 0.f, w = 0.f;
#pragma unroll 8
  for (int k = 0; k < STAT_CHUNKS; ++k) {  // unrolled: 24 independent loads in flight (same addition order)
    s += __ldg(p + (k * 3 + 0) * C + c);
    q += __ldg(p + (k * 3 + 1) * C + c);
    w += __ldg(p + (k * 3 + 2) * C + c);
  }
  const float rows = (float)(seg_off[seg + 1] - seg_off[seg]);
  __shared__ float sh_s[C], sh_q[C], sh_d[C];
  sh_s[c] = s;
  sh_q[c] = q;
  __syncthreads();
  constexpr int CPG = C / G;
  const int g = c / CPG;
  float gs = 0.f, gq = 0.f;
#pragma unroll
  for (int i = 0; i < CPG; ++i) {
    gs += sh_s[g * CPG + i];
    gq += sh_q[g * CPG + i];
  }
  const float cnt = rows * CPG;
  const float mu = gs / cnt;
  const float var = fmaxf(gq / cnt - mu * mu, 0.f);
  const float rstd = rsqrtf(var + eps);
  const float ga = rstd * gn_w[c], gb = gn_b[c] - mu * rstd * gn_w[c];
  affine[((long)sb * 2 + 0) * C + c] = ga;
  affine[((long)sb * 2 + 1) * C + c] = gb;
  const float ymean = weighted ? w : s / rows;
  sh_d[c] = (ga * ymean + gb) * attn_w[c];
  __syncthreads();
  for (int o = C / 2; o > 0; o >>= 1) {
    if (c < o) sh_d[c] += sh_d[c + o];
    __syncthreads();
  }
  if (c == 0) {
    const float a = fmaxf(sh_d[0] + attn_b[0], 0.f);   // Conv2d(256,1,1) + ReLU
    attn[sb] = fminf(fmaxf(a + 3.f, 0.f), 6.f) / 6.f;  // h_sigmoid
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Scale-aware fusion (vldyhead.py:219-238): mid[p] = mean_k attn_k * GN_k(y_k)[p]; branch 0 is bilinearly upsampled
// (align_corners=True, F.upsample_bilinear :224) from the next-coarser grid.  One warp per pixel, 8 channels per lane.
// ---------------------------------------------------------------------------------------------------------------
constexpr int MID_CHUNKS = 128;  // pixel ranges per (image, level) of dyconv_combine == partial-sum rows DyReLU reads
// grid (MID_CHUNKS, B * L): a block = one contiguous pixel range of ONE (image, level), a warp = a contiguous sub-range
// (8 channels per lane).  The (attention x GroupNorm affine) rows of the block's (image, level) are folded into one
// scale/offset pair per branch once per block; row / column advance by increment.  The per-channel sums of the (rounded)
// output — the global average pool DyReLU needs (layers/dyrelu.py:84-86) — are reduced per block into
// mid_sums[b][l][chunk][C], so `mid` is not read a second time for them.
template <int C>
__global__ void __launch_bounds__(256, 3) dyconv_combine_kernel(const __half* __restrict__ y1, const __half* __restrict__ y2,
                                                             const __half* __restrict__ y0, const float* __restrict__ aff1,
                                                             const float* __restrict__ aff2, const float* __restrict__ aff0,
                                                             const float* __restrict__ at1, const float* __restrict__ at2,
                                                             const float* __restrict__ at0, LevelTable lt, int B,
                                                             __half* __restrict__ mid, float* __restrict__ mid_sums) {
  const int chunk = blockIdx.x, sb = blockIdx.y;
  const int L = lt.n;
  const int b = sb / L, l = sb - b * L;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int N = lt.off[L - 1] + lt.H[L - 1] * lt.W[L - 1];
  const int N1 = N - lt.H[0] * lt.W[0];
  const int H = lt.H[l], W = lt.W[l], HW = H * W;
  const int len = (HW + MID_CHUNKS - 1) / MID_CHUNKS, sub = (len + 7) / 8;
  const int p0 = chunk * len + warp * sub;
  const int p1 = min(min(p0 + sub, (chunk + 1) * len), HW);
  const int c0 = lane * 8;
  const bool has2 = l > 0, has0 = l < L - 1;
  float sums[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) sums[i] = 0.f;
  if (p0 < p1) {
    float s1[8], s2[8], s0[8], off[8];  // acc = s1*y1 + s2*y2 + s0*up(y0) + off, already divided by the branch count
    {
      const float inv = 1.f / (float)(1 + (has2 ? 1 : 0) + (has0 ? 1 : 0));
      float g[8], o[8];
      {
        const float a = at1[b * L + l] * inv;
        const float* ga = aff1 + ((long)(b * L + l) * 2) * C + c0;
        ld8f(ga, g);
        ld8f(ga + C, o);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          s1[i] = a * g[i];
          off[i] = a * o[i];
          s2[i] = s0[i] = 0.f;
        }
      }
      if (has2) {  // branch 2: stride-2 conv of the finer level, already at this resolution; segment index l-1
        const float a = at2[b * (L - 1) + l - 1] * inv;
        const float* ga = aff2 + ((long)(b * (L - 1) + l - 1) * 2) * C + c0;
        ld8f(ga, g);
        ld8f(ga + C, o);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          s2[i] = a * g[i];
          off[i] += a * o[i];
        }
      }
      if (has0) {  // branch 0: conv on the coarser level (segment index l), upsampled to (H, W)
        const float a = at0[b * (L - 1) + l] * inv;
        const float* ga = aff0 + ((long)(b * (L - 1) + l) * 2) * C + c0;
        ld8f(ga, g);
        ld8f(ga + C, o);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          s0[i] = a * g[i];
          off[i] += a * o[i];  // bilinear weights sum to 1: the affine offset passes through the upsampling
        }
      }
    }
    const int Hs = has0 ? lt.H[l + 1] : 1, Ws = has0 ? lt.W[l + 1] : 1;
    // area_pixel_compute_source_index, align_corners=True (fp32 scale like ATen)
    const float sh = (H > 1) ? (float)(Hs - 1) / (float)(H - 1) : 0.f;
    const float sw = (W > 1) ? (float)(Ws - 1) / (float)(W - 1) : 0.f;
    const __half* y1b = y1 + ((long)b * N + lt.off[l]) * C + c0;
    const __half* y2b = has2 ? y2 + ((long)b * N1 + (lt.off[l] - lt.off[1])) * C + c0 : nullptr;
    const __half* y0b = has0 ? y0 + ((long)b * N1 + (lt.off[l + 1] - lt.off[1])) * C + c0 : nullptr;
    __half* mb = mid + ((long)b * N + lt.off[l]) * C + c0;
    int h = p0 / W, w = p0 - h * W;
#pragma unroll 1
    for (int p = p0; p < p1; ++p) {
      float acc[8], v[8];
      ld8h(y1b + (long)p * C, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(s1[i], v[i], off[i]);
      if (has2) {
        ld8h(y2b + (long)p * C, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(s2[i], v[i], acc[i]);
      }
      if (has0) {
        const float fh = sh * h, fw = sw * w;
        const int h0 = (int)fh, w0 = (int)fw;
        const int h1 = h0 + ((h0 < Hs - 1) ? 1 : 0), w1 = w0 + ((w0 < Ws - 1) ? 1 : 0);
        const float lh = fh - h0, lw = fw - w0;
        float t00[8], t01[8], t10[8], t11[8];
        ld8h(y0b + (long)(h0 * Ws + w0) * C, t00);
        ld8h(y0b + (long)(h0 * Ws + w1) * C, t01);
        ld8h(y0b + (long)(h1 * Ws + w0) * C, t10);
        ld8h(y0b + (long)(h1 * Ws + w1) * C, t11);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float u = (1.f - lh) * (1.f - lw) * t00[i];
          u += (1.f - lh) * lw * t01[i];
          u += lh * (1.f - lw) * t10[i];
          u += lh * lw * t11[i];
          acc[i] = fmaf(s0[i], u, acc[i]);
        }
      }
      __half2 hv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        hv[i] = __floats2half2_rn(acc[2 * i], acc[2 * i + 1]);
        const float2 r = __half22float2(hv[i]);  // the pooled mean is taken over the STORED (rounded) values
        sums[2 * i] += r.x;
        sums[2 * i + 1] += r.y;
      }
      *reinterpret_cast<uint4*>(mb + (long)p * C) = *reinterpret_cast<uint4*>(hv);
      if (++w == W) {
        w = 0;
        ++h;
      }
    }
  }
  if (mid_sums) {  // block-uniform
    __shared__ float shs[8][C];
#pragma unroll
    for (int i = 0; i < 8; ++i) shs[warp][c0 + i] = sums[i];
    __syncthreads();
    const int c = threadIdx.x;  // C == blockDim.x
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += shs[j][c];
    mid_sums[((long)sb * MID_CHUNKS + chunk) * C + c] = t;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// DyReLU coefficients (layers/dyrelu.py:80-104; K2, use_bias, reduction 4): per (image, level)
//   y = h_sigmoid(W2 relu(W1 GAP(x) + b1) + b2)  [4C] -> a1=(y0-.5)*2+1, b1=y1-.5, a2=(y2-.5)*2, b2=y3-.5
// One block of C threads per (b, level).  coef[b][l][4][C].
// ---------------------------------------------------------------------------------------------------------------
template <int C, int SQ>
__global__ void __launch_bounds__(C) dyrelu_coef_kernel(const float* __restrict__ partial, int chunks, int stats,
                                                        const int* __restrict__ seg_off, int nseg,
                                                        const float* __restrict__ w1,
                                                        const float* __restrict__ b1, const float* __restrict__ w2,
                                                        const float* __restrict__ b2, float* __restrict__ coef) {
  const int sb = blockIdx.x, seg = sb % nseg;
  const int c = threadIdx.x;
  // partial[sb][chunk][stats][C], statistic 0 = the plain sum (chan_stats: 32 x 3, dyconv_combine: MID_CHUNKS x 1)
  const float* p = partial + (long)sb * chunks * stats * C + c;
  float s = 0.f;
  for (int k0 = 0; k0 < chunks; k0 += 32) {
    float v[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) v[k] = (k0 + k < chunks) ? __ldg(p + (long)(k0 + k) * stats * C) : 0.f;  // 32 loads in flight
#pragma unroll
    for (int k = 0; k < 32; ++k) s += v[k];
  }
  __shared__ float gap[C], hid[SQ];
  gap[c] = s / (float)(seg_off[seg + 1] - seg_off[seg]);
  __syncthreads();
  // both mat-vecs read their weight rows coalesced (a thread per output row walked 1 KB / 256 B strides: 50 us of latency)
  const int warp = c >> 5, lane = c & 31;
  // hid = relu(W1 gap + b1): W1 [SQ][C]; a warp per output row, 8 floats of the row per lane.  ALL loads of a warp's rows are
  // issued before the first reduction (a load -> shuffle -> next load chain costs one memory latency per row)
  {
    constexpr int RPW = SQ / (C / 32);  // rows per warp (8)
    float4 wa[RPW], wb[RPW];
#pragma unroll
    for (int k = 0; k < RPW; ++k) {
      const float4* row = reinterpret_cast<const float4*>(w1 + (long)(warp + k * (C / 32)) * C);
      wa[k] = __ldg(row + 2 * lane);
      wb[k] = __ldg(row + 2 * lane + 1);
    }
    const float* g = gap + 8 * lane;
#pragma unroll
    for (int k = 0; k < RPW; ++k) {
      float t = wa[k].x * g[0];
      t = fmaf(wa[k].y, g[1], t); t = fmaf(wa[k].z, g[2], t); t = fmaf(wa[k].w, g[3], t);
      t = fmaf(wb[k].x, g[4], t); t = fmaf(wb[k].y, g[5], t); t = fmaf(wb[k].z, g[6], t); t = fmaf(wb[k].w, g[7], t);
      t = warp_sum(t);
      const int o = warp + k * (C / 32);
      if (lane == 0) hid[o] = fmaxf(t + b1[o], 0.f);
    }
  }
  __syncthreads();
  // y = h_sigmoid(W2 hid + b2): W2 [4C][SQ = 64]; half a warp per output row (one float4 per lane), two rows per warp step,
  // eight steps' loads in flight at a time
  {
    const int hl = lane & 15, hw = lane >> 4;
    const float h0 = hid[4 * hl], h1 = hid[4 * hl + 1], h2 = hid[4 * hl + 2], h3 = hid[4 * hl + 3];
    constexpr int STRIDE = (C / 32) * 2, STEPS = 4 * C / STRIDE, UN = 8;
    static_assert(STEPS % UN == 0, "dyrelu_coef: step count must be a multiple of the unroll");
#pragma unroll 1
    for (int s0 = 0; s0 < STEPS; s0 += UN) {
      float4 wv[UN];
#pragma unroll
      for (int u = 0; u < UN; ++u)
        wv[u] = __ldg(reinterpret_cast<const float4*>(w2 + (long)(warp * 2 + hw + (s0 + u) * STRIDE) * SQ) + hl);
#pragma unroll
      for (int u = 0; u < UN; ++u) {
        const int o = warp * 2 + hw + (s0 + u) * STRIDE;
        float t = wv[u].x * h0;
        t = fmaf(wv[u].y, h1, t); t = fmaf(wv[u].z, h2, t); t = fmaf(wv[u].w, h3, t);
        t += __shfl_xor_sync(0xffffffffu, t, 8);
        t += __shfl_xor_sync(0xffffffffu, t, 4);
        t += __shfl_xor_sync(0xffffffffu, t, 2);
        t += __shfl_xor_sync(0xffffffffu, t, 1);
        if (hl == 0) {
          t = fminf(fmaxf(t + b2[o] + 3.f, 0.f), 6.f) / 6.f;  // h_sigmoid
          const int k = o / C;
          float r;
          if (k == 0) r = (t - 0.5f) * 2.f + 1.f;
          else if (k == 1) r = t - 0.5f;
          else if (k == 2) r = (t - 0.5f) * 2.f;
          else r = t - 0.5f;
          coef[(long)sb * 4 * C + o] = r;
        }
      }
    }
  }
}

// One warp per run of DR_PPW consecutive pixels (8 channels per lane): the four coefficient rows of the run's (image,
// level) stay in registers and are reloaded only when the run crosses a level boundary; all pixel vectors of the run are
// loaded before the first one is used.
constexpr int DR_PPW = 8;
template <int C>
__global__ void __launch_bounds__(256) dyrelu_apply_kernel(const __half* __restrict__ mid, const float* __restrict__ coef,
                                                           LevelTable lt, int B, __half* __restrict__ out) {
  const long gw0 = (((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * DR_PPW;
  const int lane = threadIdx.x & 31;
  const int L = lt.n;
  const int N = lt.off[L - 1] + lt.H[L - 1] * lt.W[L - 1];
  const long total = (long)B * N;
  if (gw0 >= total) return;
  uint4 u[DR_PPW];
#pragma unroll
  for (int j = 0; j < DR_PPW; ++j)
    u[j] = (gw0 + j < total) ? *reinterpret_cast<const uint4*>(mid + (gw0 + j) * C + lane * 8) : make_uint4(0, 0, 0, 0);
  int cur = -1;
  float a1[8], b1[8], a2[8], b2[8];
#pragma unroll
  for (int j = 0; j < DR_PPW; ++j) {
    const long gw = gw0 + j;
    if (gw >= total) break;
    const int b = (int)(gw / N), pn = (int)(gw % N);
    int l = 0;
    while (l + 1 < L && pn >= lt.off[l + 1]) ++l;
    if (b * L + l != cur) {
      cur = b * L + l;
      const float* cf = coef + ((long)cur * 4) * C + lane * 8;
      ld8f(cf, a1);
      ld8f(cf + C, b1);
      ld8f(cf + 2 * C, a2);
      ld8f(cf + 3 * C, b2);
    }
    const __half2* h = reinterpret_cast<const __half2*>(&u[j]);
    float v[8], o[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      v[2 * i] = f.x;
      v[2 * i + 1] = f.y;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = fmaxf(v[i] * a1[i] + b1[i], v[i] * a2[i] + b2[i]);
    st8h(out + gw * C + lane * 8, o);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Plain 3x3 / pad 1 / stride 1 convolution with <= 32 output channels over every pyramid level at once, WITHOUT a column
// matrix: the 27-channel offset/mask conv of DyConv (vldyhead.py:150-153, 207-210).  An implicit GEMM on mma.sync
// (M = 16 pixels per warp, N = 32, K = 9 x 256): the A fragments are 16-byte loads straight from the NHWC-rows
// pyramid (neighbouring pixels hit L1), the weights [32][2304] live in shared memory (ldmatrix, rows padded by 16 B).
// Channel permutation: within each 32-channel group thread t4 of a quad owns channels 8*t4 .. 8*t4+7 (one 16-byte
// load) and feeds them to TWO k-steps as logical k = {2t4, 2t4+1, 2t4+8, 2t4+9} <- channels 8t4 + 4s + {0,1,2,3}; the
// weights are stored in that logical order, so sum over k is unchanged.
// ---------------------------------------------------------------------------------------------------------------
constexpr int CS_O = 32, CS_K = 9 * 256, CS_LD = CS_K + 8;  // smem row stride in halfs (+16 B: conflict-free ldmatrix)
constexpr int CS_WARPS = 12, CS_PIX = 16 * CS_WARPS;

__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

__global__ void __launch_bounds__(CS_WARPS * 32, 1) conv3x3_small_kernel(const __half* __restrict__ x,
                                                                         const __half* __restrict__ w, int O,
                                                                         const float* __restrict__ bias, LevelTable lt, int B,
                                                                         float* __restrict__ out, int ld) {
  extern __shared__ __align__(16) uint8_t cs_smem[];
  __half* ws = reinterpret_cast<__half*>(cs_smem);
  constexpr int C = 256;
  // weights -> shared, logical k order: ws[n][tap*256 + kp*32 + s*16 + lk] = w[n][tap*256 + kp*32 + phys(s, lk)]
  for (int i = threadIdx.x; i < CS_O * CS_K; i += blockDim.x) {
    const int n = i / CS_K, k = i % CS_K;
    const int lk = k & 15, s = (k >> 4) & 1, base = k & ~31;
    const int t = (lk & 7) >> 1, e = lk & 1, hi = lk >> 3;
    const int phys = base + 8 * t + 4 * s + 2 * hi + e;
    ws[n * CS_LD + k] = (n < O) ? w[(long)n * CS_K + phys] : __float2half_rn(0.f);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int L = lt.n;
  const int N = lt.off[L - 1] + lt.H[L - 1] * lt.W[L - 1];
  const long total = (long)B * N;
  // ldmatrix row address of this lane: matrix m = lane / 8 -> (n tile m / 2 [+2 for the second instruction], k half m % 2)
  const uint32_t ws_addr = smem_u32(ws) + (uint32_t)((((lane >> 4) * 8 + (lane & 7)) * CS_LD + ((lane >> 3) & 1) * 8) * 2);
  float bv[4][2];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = nt * 8 + 2 * t4 + e;
      bv[nt][e] = (n < O) ? bias[n] : 0.f;
    }
  for (long tile = blockIdx.x; tile * CS_PIX < total; tile += gridDim.x) {
    const long p0 = tile * CS_PIX + warp * 16;
    if (p0 >= total) continue;
    // the two pixels (fragment rows g and g + 8) of this lane
    int ph[2], pw[2], pH[2], pW[2];
    const __half* pbase[2];
    bool pok[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const long gp = p0 + g + 8 * r;
      pok[r] = gp < total;
      const long gq = pok[r] ? gp : 0;
      const int b = (int)(gq / N), pn = (int)(gq % N);
      int l = 0;
      while (l + 1 < L && pn >= lt.off[l + 1]) ++l;
      const int q = pn - lt.off[l];
      pH[r] = lt.H[l];
      pW[r] = lt.W[l];
      ph[r] = q / pW[r];
      pw[r] = q % pW[r];
      pbase[r] = x + ((long)b * N + lt.off[l]) * C + 8 * t4;
    }
    float acc[4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
    // chunk = half a tap = 4 channel groups of 32 = 8 k-steps; two register sets ping-pong (loads of chunk c+1 in flight
    // while chunk c feeds the tensor cores)
    auto load_chunk = [&](int ch, uint4 (&buf)[8]) {
      const int tap = ch >> 1, half = ch & 1;
      const int dy = tap / 3 - 1, dx = tap % 3 - 1;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int hs = ph[r] + dy, wsrc = pw[r] + dx;
        const bool ok = pok[r] && hs >= 0 && hs < pH[r] && wsrc >= 0 && wsrc < pW[r];
        const __half* src = pbase[r] + ((long)hs * pW[r] + wsrc) * C + half * 128;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          buf[r * 4 + j] = ok ? __ldg(reinterpret_cast<const uint4*>(src + j * 32)) : make_uint4(0, 0, 0, 0);
      }
    };
    auto compute_chunk = [&](int ch, const uint4 (&buf)[8]) {
      const int kbase = (ch >> 1) * 256 + (ch & 1) * 128;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 ug = buf[j], uh = buf[4 + j];
#pragma unroll
        for (int s2 = 0; s2 < 2; ++s2) {
          const uint32_t kaddr = ws_addr + (uint32_t)((kbase + j * 32 + s2 * 16) * 2);
          uint32_t b01[4], b23[4];
          ldmatrix_x4(b01, kaddr);                                 // n tiles 0, 1
          ldmatrix_x4(b23, kaddr + (uint32_t)(16 * CS_LD * 2));    // n tiles 2, 3
          const uint32_t a0 = s2 ? ug.z : ug.x, a1 = s2 ? uh.z : uh.x, a2 = s2 ? ug.w : ug.y, a3 = s2 ? uh.w : uh.y;
          mma16816(acc[0], a0, a1, a2, a3, b01[0], b01[1]);
          mma16816(acc[1], a0, a1, a2, a3, b01[2], b01[3]);
          mma16816(acc[2], a0, a1, a2, a3, b23[0], b23[1]);
          mma16816(acc[3], a0, a1, a2, a3, b23[2], b23[3]);
        }
      }
    };
    uint4 bufA[8], bufB[8];
    load_chunk(0, bufA);
#pragma unroll 1
    for (int ch = 0; ch < 18; ch += 2) {
      load_chunk(ch + 1, bufB);
      compute_chunk(ch, bufA);
      if (ch + 2 < 18) load_chunk(ch + 2, bufA);
      compute_chunk(ch + 1, bufB);
    }
    // C fragment: (row g, cols 2t4, 2t4+1), (row g+8, same cols) per n tile
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const long gp = p0 + g + 8 * r;
      if (gp >= total) continue;
      float* o = out + gp * ld;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = nt * 8 + 2 * t4 + e;
          if (n < O) o[n] = acc[nt][2 * r + e] + bv[nt][e];
        }
    }
  }
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_dcn_cols(const void* x, const float* om, int64_t om_ld, const int32_t* level_hw, int64_t nlev,
                              int64_t B, int64_t C, int branch, void* cols, void* stream) {
  MQ_REQUIRE(x && cols && level_hw, "dcn_cols: null pointer");
  MQ_REQUIRE(C == 256, "dcn_cols: C must be 256 (got %ld)", (long)C);
  MQ_REQUIRE(branch >= 0 && branch <= 2, "dcn_cols: branch must be 0, 1 or 2");
  LevelTable lt;
  const int N = fill_levels(&lt, level_hw, nlev);
  MQ_REQUIRE(N > 0, "dcn_cols: bad level table");
  MQ_REQUIRE(branch == 1 || nlev >= 2, "dcn_cols: branches 0/2 need at least two levels");
  const long rows_per_img = branch == 1 ? N : N - lt.H[0] * lt.W[0];
  const long warps = B * rows_per_img;
  const long blocks = (warps * 32 + 255) / 256;
  dcn_cols_kernel<256><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __half*)x, om, (int)om_ld, lt, branch,
                                                                          (int)B, rows_per_img, (__half*)cols);
  return check_launch("dcn_cols_kernel");
}

extern "C" int64_t mqdet_chan_stats_floats(int64_t B, int64_t nseg, int64_t C) { return B * nseg * STAT_CHUNKS * 3 * C; }

extern "C" int mqdet_chan_stats(const void* y, const int32_t* seg_off_dev, int64_t nseg, int64_t B, int64_t rows_per_img,
                                int64_t C, const float* row_weights, float* partial, void* stream) {
  MQ_REQUIRE(y && seg_off_dev && partial, "chan_stats: null pointer");
  MQ_REQUIRE(C == 256, "chan_stats: C must be 256");
  chan_stats_kernel<256><<<dim3(STAT_CHUNKS, (unsigned)(B * nseg)), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)y, seg_off_dev, (int)nseg, rows_per_img, row_weights, partial);
  return check_launch("chan_stats_kernel");
}

extern "C" int mqdet_gn_attn(const float* partial, const int32_t* seg_off_dev, int64_t nseg, int64_t B, int64_t C,
                             int64_t groups, int weighted, const float* gn_w, const float* gn_b, float eps,
                             const float* attn_w, const float* attn_b, float* affine, float* attn, void* stream) {
  MQ_REQUIRE(partial && seg_off_dev && gn_w && gn_b && attn_w && attn_b && affine && attn, "gn_attn: null pointer");
  MQ_REQUIRE(C == 256 && groups == 16, "gn_attn: C=256, groups=16 only (MODEL.GROUP_NORM.NUM_GROUPS)");
  gn_attn_kernel<256, 16><<<(unsigned)(B * nseg), 256, 0, (cudaStream_t)stream>>>(partial, seg_off_dev, (int)nseg, weighted,
                                                                                  gn_w, gn_b, eps, attn_w, attn_b, affine,
                                                                                  attn);
  return check_launch("gn_attn_kernel");
}

extern "C" int64_t mqdet_dyconv_combine_chunks(void) { return MID_CHUNKS; }

extern "C" int mqdet_dyconv_combine(const void* y1, const void* y2, const void* y0, const float* aff1, const float* aff2,
                                    const float* aff0, const float* at1, const float* at2, const float* at0,
                                    const int32_t* level_hw, int64_t nlev, int64_t B, int64_t C, void* mid, float* mid_sums,
                                    void* stream) {
  MQ_REQUIRE(y1 && aff1 && at1 && mid && level_hw, "dyconv_combine: null pointer");
  MQ_REQUIRE(C == 256, "dyconv_combine: C must be 256");
  LevelTable lt;
  const int N = fill_levels(&lt, level_hw, nlev);
  MQ_REQUIRE(N > 0, "dyconv_combine: bad level table");
  MQ_REQUIRE(nlev == 1 || (y2 && y0 && aff2 && aff0 && at2 && at0), "dyconv_combine: missing cross-level inputs");
  MQ_REQUIRE(B >= 1 && B * nlev <= 65535, "dyconv_combine: B * levels must be in 1..65535");
  dyconv_combine_kernel<256><<<dim3(MID_CHUNKS, (unsigned)(B * nlev)), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)y1, (const __half*)y2, (const __half*)y0, aff1, aff2, aff0, at1, at2, at0, lt, (int)B, (__half*)mid, mid_sums);
  return check_launch("dyconv_combine_kernel");
}

extern "C" int mqdet_dyrelu_coef(const float* partial, int64_t chunks, int64_t stats, const int32_t* seg_off_dev, int64_t nseg,
                                 int64_t B, int64_t C, int64_t squeeze, const float* w1, const float* b1, const float* w2,
                                 const float* b2, float* coef, void* stream) {
  MQ_REQUIRE(partial && seg_off_dev && w1 && b1 && w2 && b2 && coef, "dyrelu_coef: null pointer");
  MQ_REQUIRE(chunks >= 1 && stats >= 1, "dyrelu_coef: chunks / stats must be positive");
  MQ_REQUIRE((((uintptr_t)w1 | (uintptr_t)w2) & 15) == 0, "dyrelu_coef: weights must be 16-byte aligned");
  MQ_REQUIRE(C == 256 && squeeze == 64, "dyrelu_coef: C=256, squeeze=64 only");
  dyrelu_coef_kernel<256, 64><<<(unsigned)(B * nseg), 256, 0, (cudaStream_t)stream>>>(partial, (int)chunks, (int)stats, seg_off_dev,
                                                                                      (int)nseg, w1, b1, w2, b2, coef);
  return check_launch("dyrelu_coef_kernel");
}

extern "C" int mqdet_dyrelu_apply(const void* mid, const float* coef, const int32_t* level_hw, int64_t nlev, int64_t B,
                                  int64_t C, void* out, void* stream) {
  MQ_REQUIRE(mid && coef && out && level_hw, "dyrelu_apply: null pointer");
  MQ_REQUIRE(C == 256, "dyrelu_apply: C must be 256");
  LevelTable lt;
  const int N = fill_levels(&lt, level_hw, nlev);
  MQ_REQUIRE(N > 0, "dyrelu_apply: bad level table");
  const long blocks = (((long)B * N + DR_PPW - 1) / DR_PPW * 32 + 255) / 256;
  dyrelu_apply_kernel<256><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __half*)mid, coef, lt, (int)B,
                                                                              (__half*)out);
  return check_launch("dyrelu_apply_kernel");
}

extern "C" int mqdet_conv3x3_small(const void* x, const void* w, const float* bias, const int32_t* level_hw, int64_t nlev,
                                   int64_t B, int64_t C, int64_t O, float* out, int64_t ld, void* stream) {
  MQ_REQUIRE(x && w && bias && out && level_hw, "conv3x3_small: null pointer");
  MQ_REQUIRE(C == 256 && O >= 1 && O <= CS_O && ld >= O, "conv3x3_small: C must be 256, O <= 32, ld >= O");
  MQ_REQUIRE(((uintptr_t)x % 16) == 0, "conv3x3_small: x must be 16-byte aligned");
  LevelTable lt;
  const int N = fill_levels(&lt, level_hw, nlev);
  MQ_REQUIRE(N > 0, "conv3x3_small: bad level table");
  constexpr int SMEM = CS_O * CS_LD * 2;
  if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(&conv3x3_small_kernel), SMEM)) return rc;
  const int sms = num_sms();
  const long tiles = ((long)B * N + CS_PIX - 1) / CS_PIX;
  const int grid = (int)(tiles < sms ? tiles : sms);
  conv3x3_small_kernel<<<grid, CS_WARPS * 32, SMEM, (cudaStream_t)stream>>>((const __half*)x, (const __half*)w, (int)O, bias, lt,
                                                                           (int)B, out, (int)ld);
  return check_launch("conv3x3_small_kernel");
}
