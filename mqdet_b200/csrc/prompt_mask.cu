// mqdet_b200 — vision-only evaluation: the prompt tokens of categories that have vision queries replaced by [MASK]
// (maskrcnn_benchmark/modeling/detector/generalized_vl_rcnn_new.py:397-407 with VISION_QUERY.MASK_DURING_INFERENCE).
//
//   mask_prompt_tokens_kernel : out[e][t] = mask_id if tok_cat[e][t] >= 0 and flags[e][tok_cat[e][t]] != 0, else ids[e][t]
//
// The ids are written out of place so that the unmasked ids of a cached prompt stay as they are; the per-category flags
// (draw < TEXT_DROPOUT and the category has queries) come from the host, the per-token category table is built once per prompt.
#include "common.cuh"

namespace mqdet {

__global__ void __launch_bounds__(256) mask_prompt_tokens_kernel(const int64_t* __restrict__ ids, const int32_t* __restrict__ tok_cat,
                                                                 const uint8_t* __restrict__ flags, int64_t T, int64_t C,
                                                                 int64_t n, int64_t mask_id, int64_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t c = tok_cat[i];
  const bool masked = c >= 0 && c < C && flags[(i / T) * C + c] != 0;
  out[i] = masked ? mask_id : ids[i];
}

}  // namespace mqdet

using namespace mqdet;

extern "C" int mqdet_mask_prompt_tokens(const int64_t* ids, const int32_t* tok_cat, const uint8_t* flags, int64_t E, int64_t T,
                                        int64_t C, int64_t mask_id, int64_t* out, void* stream) {
  MQ_REQUIRE(ids && tok_cat && out && (flags || C == 0), "mask_prompt_tokens: null pointer");
  MQ_REQUIRE(E > 0 && T > 0 && C >= 0 && E * T < ((int64_t)1 << 40), "mask_prompt_tokens: bad sizes E=%ld T=%ld C=%ld", (long)E,
             (long)T, (long)C);
  MQ_REQUIRE((const void*)ids != (const void*)out, "mask_prompt_tokens: out must not alias ids");
  mask_prompt_tokens_kernel<<<cdiv(E * T, 256), 256, 0, (cudaStream_t)stream>>>(ids, tok_cat, flags, T, C, E * T, mask_id, out);
  return check_launch("mask_prompt_tokens_kernel");
}
