// mqdet_b200 — the test-time image transform on the device: PIL-exact bilinear resize, ToTensor, Normalize, to_image_list.
//
// Reference: maskrcnn_benchmark/data/transforms/transforms.py (Resize -> torchvision F.resize on a PIL image, i.e.
// PIL.Image.resize((ow, oh), BILINEAR); ToTensor; Normalize with format 'rgb' / 'bgr255'), structures/image_list.py
// (to_image_list: zero padding to SIZE_DIVISIBILITY).
//
//   resize_coeffs_kernel  : one (in, out) length pair -> per output index: first input index, tap count and the 22-bit
//                           fixed-point weights of Pillow's bilinear resampler (fp64, every operation rounded)
//   test_transform_kernel : B uint8 HWC RGB images (any source sizes) -> one fp32 [B, 3, Hp, Wp] batch, image i resized to its
//                           own (oh_i, ow_i) and zero beyond it (to_image_list of a batch of differently sized images).
//                           One CTA per (128 output columns, 16 output rows, image): it walks the intermediate rows its 16
//                           output rows read, computes each one's horizontal pass for its columns (uint8, clipped, held in
//                           registers only) and adds it into the vertical accumulators of the rows whose window holds it.
//                           A CTA whose tile lies wholly outside its image's (oh_i, ow_i) only writes zeros.
//
// Pillow's resampler is integer arithmetic behind fp64 coefficients, so it is reproduced bit for bit: the coefficient kernel
// uses __d*_rn intrinsics (no contraction; Pillow's x86-64 build has no FMA), the passes are the same int32 sums.  A pass whose
// length does not change is the identity through its coefficients (weights {2^22, 0}), so it is not special-cased.
// ToTensor / Normalize are fp32 operations one at a time (__f*_rn), as torch computes them on the CPU.
#include <vector>

#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

constexpr int TT_PREC = 22;               // Pillow's PRECISION_BITS (32 - 8 - 2)
constexpr int TT_TX = 128;                // output columns per CTA (one per thread)
constexpr int TT_TY = 16;                 // output rows per CTA (accumulators per thread: 16 x 3)
constexpr int TT_MAX_B = 64;              // images per launch (kernel-parameter table); larger batches take several launches

struct TTImage {
  const uint8_t* src;                     // [h][w][3]
  const int32_t* xtab;                    // [ow][2 + kx]: first column, taps, weights
  const int32_t* ytab;                    // [oh][2 + ky]
  uint8_t* resized;                       // [oh][ow][3] or null
  int h, w, kx, ky;
  int oh, ow;                             // the resized size; the rest of the padded [Hp, Wp] plane is zero
};

struct TTBatch {
  TTImage im[TT_MAX_B];
};

__host__ __device__ inline int tt_ksize(long n_in, long n_out) {
  const double scale = (double)n_in / (double)n_out;
  const double fs = scale < 1.0 ? 1.0 : scale;
  return (int)ceil(fs) * 2 + 1;
}

__device__ __forceinline__ double tt_triangle(double x) {
  if (x < 0.0) x = -x;
  return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
}

__global__ void __launch_bounds__(256) resize_coeffs_kernel(int n_in, int n_out, int K, int32_t* __restrict__ table) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  const double scale = __ddiv_rn((double)n_in, (double)n_out);
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = fs;               // bilinear support 1.0 x filterscale
  const double ss = __ddiv_rn(1.0, fs);
  const double center = __dmul_rn(__dadd_rn((double)i, 0.5), scale);
  int lo = __double2int_rz(__dadd_rn(__dsub_rn(center, support), 0.5));
  int hi = __double2int_rz(__dadd_rn(__dadd_rn(center, support), 0.5));
  lo = lo < 0 ? 0 : lo;
  hi = hi > n_in ? n_in : hi;
  const int n = hi - lo;
  double total = 0.0;                      // sequential sum, as Pillow's loop
  for (int x = 0; x < n; ++x) total = __dadd_rn(total, tt_triangle(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + lo), center), 0.5), ss)));
  int32_t* row = table + (long)i * (2 + K);
  row[0] = lo;
  row[1] = n;
  for (int x = 0; x < K; ++x) {
    int32_t k = 0;
    if (x < n) {
      double w = tt_triangle(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + lo), center), 0.5), ss));
      if (total != 0.0) w = __ddiv_rn(w, total);
      const double f = __dmul_rn(w, (double)(1 << TT_PREC));
      k = w < 0.0 ? __double2int_rz(__dadd_rn(-0.5, f)) : __double2int_rz(__dadd_rn(0.5, f));
    }
    row[2 + x] = k;
  }
}

__device__ __forceinline__ int tt_clip8(int acc) {
  const int v = acc >> TT_PREC;            // arithmetic shift, as Pillow's clip8
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

__global__ void __launch_bounds__(TT_TX, 4) test_transform_kernel(const __grid_constant__ TTBatch batch, int Hp, int Wp, int bgr,
                                                               int times255, float m0, float m1, float m2, float s0, float s1,
                                                               float s2, float* __restrict__ out) {
  const TTImage& im = batch.im[blockIdx.z];
  const int oh = im.oh, ow = im.ow;
  const int x = blockIdx.x * TT_TX + threadIdx.x;
  const int y0 = blockIdx.y * TT_TY;
  const long plane = (long)Hp * Wp;
  float* o = out + (long)blockIdx.z * 3 * plane;
  if (x >= Wp) return;
  if (blockIdx.x * TT_TX >= ow || y0 >= oh) {   // the tile is padding only
    for (int r = 0; r < TT_TY && y0 + r < Hp; ++r)
      for (int c = 0; c < 3; ++c) o[c * plane + (long)(y0 + r) * Wp + x] = 0.f;
    return;
  }

  int acc[TT_TY][3];
  int ylo[TT_TY], yn[TT_TY];
  int jlo = 0x7fffffff, jhi = 0;
#pragma unroll
  for (int r = 0; r < TT_TY; ++r) {
    acc[r][0] = acc[r][1] = acc[r][2] = 1 << (TT_PREC - 1);
    ylo[r] = 0;
    yn[r] = 0;
    if (y0 + r < oh) {
      const int32_t* row = im.ytab + (long)(y0 + r) * (2 + im.ky);
      ylo[r] = row[0];
      yn[r] = row[1];
      jlo = min(jlo, ylo[r]);
      jhi = max(jhi, ylo[r] + yn[r]);
    }
  }

  if (x < ow) {
    const int32_t* xrow = im.xtab + (long)x * (2 + im.kx);
    const int xlo = xrow[0], xn = xrow[1];
    const int32_t* xk = xrow + 2;
    for (int j = jlo; j < jhi; ++j) {
      const uint8_t* p = im.src + ((long)j * im.w + xlo) * 3;
      int h0 = 1 << (TT_PREC - 1), h1 = h0, h2 = h0;
      for (int t = 0; t < xn; ++t) {
        const int k = __ldg(xk + t);
        h0 += (int)__ldg(p + 3 * t) * k;
        h1 += (int)__ldg(p + 3 * t + 1) * k;
        h2 += (int)__ldg(p + 3 * t + 2) * k;
      }
      h0 = tt_clip8(h0);
      h1 = tt_clip8(h1);
      h2 = tt_clip8(h2);
#pragma unroll
      for (int r = 0; r < TT_TY; ++r) {
        const int t = j - ylo[r];
        if (t >= 0 && t < yn[r]) {
          const int k = __ldg(im.ytab + (long)(y0 + r) * (2 + im.ky) + 2 + t);
          acc[r][0] += h0 * k;
          acc[r][1] += h1 * k;
          acc[r][2] += h2 * k;
        }
      }
    }
  }

  const float mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
#pragma unroll
  for (int r = 0; r < TT_TY; ++r) {
    const int y = y0 + r;
    if (y >= Hp) break;
    const bool in = x < ow && y < oh;
    int u[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) u[c] = tt_clip8(acc[r][c]);
    if (in && im.resized) {
      uint8_t* d = im.resized + ((long)y * ow + x) * 3;
      d[0] = (uint8_t)u[0];
      d[1] = (uint8_t)u[1];
      d[2] = (uint8_t)u[2];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = 0.f;
      if (in) {
        v = __fdiv_rn((float)u[bgr ? 2 - c : c], 255.f);       // ToTensor
        if (times255) v = __fmul_rn(v, 255.f);
        v = __fdiv_rn(__fsub_rn(v, mean[c]), stdv[c]);         // F.normalize: sub_(mean).div_(std)
      }
      o[c * plane + (long)y * Wp + x] = v;
    }
  }
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int64_t mqdet_resize_coeffs_ksize(int64_t n_in, int64_t n_out) {
  if (n_in <= 0 || n_out <= 0) return 0;
  return tt_ksize(n_in, n_out);
}

extern "C" int mqdet_resize_coeffs(int64_t n_in, int64_t n_out, int32_t* table, void* stream) {
  MQ_REQUIRE(table, "resize_coeffs: null pointer");
  MQ_REQUIRE(n_in > 0 && n_out > 0 && n_in < (1 << 24) && n_out < (1 << 24), "resize_coeffs: bad lengths %ld -> %ld", (long)n_in,
             (long)n_out);
  resize_coeffs_kernel<<<cdiv(n_out, 256), 256, 0, (cudaStream_t)stream>>>((int)n_in, (int)n_out, tt_ksize(n_in, n_out), table);
  return check_launch("resize_coeffs_kernel");
}

extern "C" int mqdet_test_transform_sizes(const void* const* src, const int64_t* hw, const int64_t* out_hw, const int32_t* const* xtab,
                                          const int32_t* const* ytab, int64_t B, int64_t Hp, int64_t Wp, int bgr, int times255,
                                          const float* mean, const float* stdv, float* out, uint8_t* resized, void* stream) {
  MQ_REQUIRE(src && hw && out_hw && xtab && ytab && mean && stdv && out, "test_transform: null pointer");
  MQ_REQUIRE(B > 0 && Hp > 0 && Wp > 0 && Hp < (1 << 16) && Wp < (1 << 16), "test_transform: bad sizes B=%ld padded to %ldx%ld",
             (long)B, (long)Hp, (long)Wp);
  for (int64_t b = 0; b < B; ++b) {
    MQ_REQUIRE(src[b] && xtab[b] && ytab[b], "test_transform: null pointer for image %ld", (long)b);
    MQ_REQUIRE(hw[2 * b] > 0 && hw[2 * b + 1] > 0 && hw[2 * b] < (1 << 16) && hw[2 * b + 1] < (1 << 16),
               "test_transform: image %ld has bad size %ldx%ld", (long)b, (long)hw[2 * b], (long)hw[2 * b + 1]);
    MQ_REQUIRE(out_hw[2 * b] > 0 && out_hw[2 * b + 1] > 0 && out_hw[2 * b] <= Hp && out_hw[2 * b + 1] <= Wp,
               "test_transform: image %ld has bad size %ldx%ld padded to %ldx%ld", (long)b, (long)out_hw[2 * b], (long)out_hw[2 * b + 1],
               (long)Hp, (long)Wp);
  }
  for (int c = 0; c < 3; ++c) MQ_REQUIRE(stdv[c] != 0.f, "test_transform: std[%d] is zero", c);
  long roff = 0;   // resized images back to back
  for (int64_t b0 = 0; b0 < B; b0 += TT_MAX_B) {
    const int nb = (int)(B - b0 < TT_MAX_B ? B - b0 : TT_MAX_B);
    TTBatch batch;
    memset(&batch, 0, sizeof(batch));
    for (int i = 0; i < nb; ++i) {
      const int64_t b = b0 + i, oh = out_hw[2 * b], ow = out_hw[2 * b + 1];
      batch.im[i] = TTImage{(const uint8_t*)src[b], xtab[b], ytab[b], resized ? resized + roff : nullptr, (int)hw[2 * b],
                            (int)hw[2 * b + 1], tt_ksize(hw[2 * b + 1], ow), tt_ksize(hw[2 * b], oh), (int)oh, (int)ow};
      roff += oh * ow * 3;
    }
    const dim3 grid(cdiv(Wp, TT_TX), cdiv(Hp, TT_TY), nb);
    test_transform_kernel<<<grid, TT_TX, 0, (cudaStream_t)stream>>>(batch, (int)Hp, (int)Wp, bgr, times255, mean[0], mean[1], mean[2],
                                                                    stdv[0], stdv[1], stdv[2], out + b0 * 3 * Hp * Wp);
    const int rc = check_launch("test_transform_kernel");
    if (rc != MQDET_OK) return rc;
  }
  return MQDET_OK;
}

extern "C" int mqdet_test_transform(const void* const* src, const int64_t* hw, const int32_t* const* xtab,
                                    const int32_t* const* ytab, int64_t B, int64_t oh, int64_t ow, int64_t Hp, int64_t Wp, int bgr,
                                    int times255, const float* mean, const float* stdv, float* out, uint8_t* resized,
                                    void* stream) {
  MQ_REQUIRE(src && hw && xtab && ytab && mean && stdv && out, "test_transform: null pointer");
  MQ_REQUIRE(B > 0 && oh > 0 && ow > 0 && Hp >= oh && Wp >= ow && Hp < (1 << 16) && Wp < (1 << 16),
             "test_transform: bad sizes B=%ld %ldx%ld padded to %ldx%ld", (long)B, (long)oh, (long)ow, (long)Hp, (long)Wp);
  std::vector<int64_t> out_hw(2 * B);
  for (int64_t b = 0; b < B; ++b) {
    out_hw[2 * b] = oh;
    out_hw[2 * b + 1] = ow;
  }
  return mqdet_test_transform_sizes(src, hw, out_hw.data(), xtab, ytab, B, Hp, Wp, bgr, times255, mean, stdv, out, resized, stream);
}
