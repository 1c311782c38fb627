// mqdet_b200 — vision-query extraction: FPN level mapping + aligned ROIAlign (+ the 7x7 mean) over the NHWC pyramid.
//
// Reference: GeneralizedVLRCNN_New.extract_query (maskrcnn_benchmark/modeling/detector/generalized_vl_rcnn_new.py:232-288):
//   Pooler (modeling/poolers.py:46-129) = LevelMapper (:11-43, FPN paper eq. 1) + one ROIAlignV2 per level
//   (layers/roi_align.py:71-81 -> torchvision.ops.roi_align(aligned=True), sampling_ratio 0 = adaptive), then
//   query_feats.mean(dim=[-2,-1]) (:263).  The arithmetic follows torchvision's roi_align kernel (aligned: half-pixel offset,
//   no minimum ROI size; adaptive grid = ceil(roi / pooled); bilinear samples outside [-1, size] contribute 0).
// HBM-bound gather: one CTA per box, one thread per channel (the pyramid rows are channel-contiguous: every sample is one
// coalesced 512-byte read), all bins of the box accumulated in registers.
#include "common.cuh"
#include "../../include/mqdet_b200.h"

namespace mqdet {

struct RoiLevels {
  int n;
  int H[MQDET_MAX_LEVELS], W[MQDET_MAX_LEVELS], off[MQDET_MAX_LEVELS];
  float scale[MQDET_MAX_LEVELS];
  float k_min, k_max;
};

__device__ __forceinline__ float bilinear_nhwc(const __half* __restrict__ f, int H, int W, int C, int c, float y, float x) {
  if (y < -1.0f || y > (float)H || x < -1.0f || x > (float)W) return 0.f;
  if (y <= 0.f) y = 0.f;
  if (x <= 0.f) x = 0.f;
  int y_low = (int)y, x_low = (int)x, y_high, x_high;
  if (y_low >= H - 1) {
    y_high = y_low = H - 1;
    y = (float)y_low;
  } else {
    y_high = y_low + 1;
  }
  if (x_low >= W - 1) {
    x_high = x_low = W - 1;
    x = (float)x_low;
  } else {
    x_high = x_low + 1;
  }
  const float ly = y - y_low, lx = x - x_low, hy = 1.f - ly, hx = 1.f - lx;
  const float v1 = __half2float(f[((long)y_low * W + x_low) * C + c]);
  const float v2 = __half2float(f[((long)y_low * W + x_high) * C + c]);
  const float v3 = __half2float(f[((long)y_high * W + x_low) * C + c]);
  const float v4 = __half2float(f[((long)y_high * W + x_high) * C + c]);
  return hy * hx * v1 + hy * lx * v2 + ly * hx * v3 + ly * lx * v4;
}

// rois [R][5] = (image index, x1, y1, x2, y2) in image pixels.  mean_only: out [R][C] = mean over the P x P bins;
// else out [R][C][P][P] (the Pooler.forward layout).  level_out (optional) receives the mapped level of every box.
__global__ void roi_align_levels_kernel(const __half* __restrict__ x, RoiLevels lv, int N, int C, const float* __restrict__ rois,
                                        int R, int P, int sampling_ratio, int mean_only, float* __restrict__ out,
                                        int* __restrict__ level_out, const int* __restrict__ n_dev) {
  const int r = blockIdx.x;
  if (r >= R || (n_dev && r >= *n_dev)) return;
  const float* roi = rois + (long)r * 5;
  const int b = (int)roi[0];
  const float x1 = roi[1], y1 = roi[2], x2 = roi[3], y2 = roi[4];
  // LevelMapper (poolers.py:32-43): s = sqrt(area) with BoxList.area()'s TO_REMOVE = 1
  const float s = sqrtf((x2 - x1 + 1.f) * (y2 - y1 + 1.f));
  float tl = floorf(4.f + log2f(s / 224.f + 1e-6f));
  tl = fminf(fmaxf(tl, lv.k_min), lv.k_max);
  const int l = (int)tl - (int)lv.k_min;
  if (level_out && threadIdx.x == 0) level_out[r] = l;
  const int H = lv.H[l], W = lv.W[l];
  const __half* f = x + ((long)b * N + lv.off[l]) * C;
  const float sc = lv.scale[l];
  const float rsw = x1 * sc - 0.5f, rsh = y1 * sc - 0.5f;  // aligned = True
  const float rw = x2 * sc - 0.5f - rsw, rh = y2 * sc - 0.5f - rsh;
  const float bin_h = rh / (float)P, bin_w = rw / (float)P;
  const int gh = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(rh / (float)P);
  const int gw = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(rw / (float)P);
  const float count = fmaxf((float)(gh * gw), 1.f);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float total = 0.f;
    for (int ph = 0; ph < P; ++ph)
      for (int pw = 0; pw < P; ++pw) {
        float acc = 0.f;
        for (int iy = 0; iy < gh; ++iy) {
          const float yy = rsh + ph * bin_h + ((float)iy + 0.5f) * bin_h / (float)gh;
          for (int ix = 0; ix < gw; ++ix) {
            const float xx = rsw + pw * bin_w + ((float)ix + 0.5f) * bin_w / (float)gw;
            acc += bilinear_nhwc(f, H, W, C, c, yy, xx);
          }
        }
        acc /= count;
        if (mean_only) total += acc;
        else out[(((long)r * C + c) * P + ph) * P + pw] = acc;
      }
    if (mean_only) out[(long)r * C + c] = total / (float)(P * P);
  }
}

}  // namespace mqdet

using namespace mqdet;

static int roi_align_launch(const void* x, const int32_t* level_hw, int64_t nlev, const float* scales, int64_t B, int64_t C,
                            const float* rois, int64_t R, const int32_t* n_dev, int64_t pooled, int64_t sampling_ratio, int mean_only,
                            float* out, int32_t* level_out, void* stream) {
  MQ_REQUIRE(x && level_hw && scales && ((rois && out) || R == 0), "roi_align_levels: null pointer");
  MQ_REQUIRE(nlev >= 1 && nlev <= MQDET_MAX_LEVELS && B >= 1 && C >= 1 && pooled >= 1 && pooled <= 32 && sampling_ratio >= 0,
             "roi_align_levels: bad arguments");
  if (R == 0) return MQDET_OK;
  RoiLevels lv;
  lv.n = (int)nlev;
  int off = 0;
  for (int l = 0; l < nlev; ++l) {
    lv.H[l] = level_hw[2 * l];
    lv.W[l] = level_hw[2 * l + 1];
    lv.off[l] = off;
    lv.scale[l] = scales[l];
    off += lv.H[l] * lv.W[l];
    MQ_REQUIRE(lv.H[l] > 0 && lv.W[l] > 0 && scales[l] > 0.f, "roi_align_levels: bad level table");
  }
  // poolers.py:76-78: levels from the first / last scale (the network halves the resolution per level)
  lv.k_min = -log2f(scales[0]);
  lv.k_max = -log2f(scales[nlev - 1]);
  roi_align_levels_kernel<<<(unsigned)R, 256, 0, (cudaStream_t)stream>>>((const __half*)x, lv, off, (int)C, rois, (int)R, (int)pooled,
                                                                      (int)sampling_ratio, mean_only, out, level_out, n_dev);
  return check_launch("roi_align_levels_kernel");
}

extern "C" int mqdet_roi_align_levels(const void* x, const int32_t* level_hw, int64_t nlev, const float* scales, int64_t B,
                                      int64_t C, const float* rois, int64_t R, int64_t pooled, int64_t sampling_ratio,
                                      int mean_only, float* out, int32_t* level_out, void* stream) {
  return roi_align_launch(x, level_hw, nlev, scales, B, C, rois, R, nullptr, pooled, sampling_ratio, mean_only, out, level_out, stream);
}

// The same over the first *count (device) of cap rows: blocks past the count return at once, so no host read is needed.
extern "C" int mqdet_roi_align_levels_counted(const void* x, const int32_t* level_hw, int64_t nlev, const float* scales, int64_t B,
                                              int64_t C, const float* rois, const int32_t* count, int64_t cap, int64_t pooled,
                                              int64_t sampling_ratio, int mean_only, float* out, int32_t* level_out, void* stream) {
  MQ_REQUIRE(count, "roi_align_levels_counted: null count");
  return roi_align_launch(x, level_hw, nlev, scales, B, C, rois, cap, count, pooled, sampling_ratio, mean_only, out, level_out, stream);
}
