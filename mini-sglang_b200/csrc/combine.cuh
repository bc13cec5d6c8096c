// Split-KV combine shared by the decode kernels: merges the per-chunk partial (o, m, l) written by
// the attention kernel into the final output (flash-decoding reduction).
#pragma once
#include "attn.cuh"

namespace b200 {

// ------------------------------------------------------------------------------- combine
// grid (bs, hq), 128 threads (one per output dim). Requests with a single chunk were already
// written by the attention kernel.
template <typename T>
__global__ void __launch_bounds__(kHeadDim) attn_combine_kernel(const float* __restrict__ part_o,
                                                          const float* __restrict__ part_ml,
                                                          const int32_t* __restrict__ plan, int hq,
                                                          T* __restrict__ out) {
  const int r = blockIdx.x, hh = blockIdx.y, d = threadIdx.x;
  pdl_wait();                // the decode kernel's partials
  pdl_launch_dependents();   // the next kernel may start its prologue
  const int32_t* chunk_start = plan + kPlanHeader;
  const int n = chunk_start[r + 1] - chunk_start[r];
  if (n <= 1) return;
  // Every load of the merge is issued before anything is consumed (their addresses do not depend on one
  // another): one global round trip instead of three -- the kernel is pure latency at decode sizes.
  const int64_t idx0 = ((int64_t)r * kMaxSplits) * hq + hh;
  float mc[kMaxSplits], lc[kMaxSplits], oc[kMaxSplits];
#pragma unroll
  for (int c = 0; c < kMaxSplits; ++c) {
    const bool on = c < n;
    const int64_t idx = idx0 + (int64_t)c * hq;
    const float2 ml = on ? __ldcg(reinterpret_cast<const float2*>(part_ml + idx * 2)) : make_float2(-INFINITY, 0.f);
    mc[c] = ml.x;
    lc[c] = ml.y;
    oc[c] = on ? __ldcg(part_o + idx * kHeadDim + d) : 0.f;
  }
  float m = -INFINITY;
#pragma unroll
  for (int c = 0; c < kMaxSplits; ++c) m = fmaxf(m, mc[c]);
  float acc = 0.f, l = 0.f;
#pragma unroll
  for (int c = 0; c < kMaxSplits; ++c) {
    if (c < n) {  // same accumulation order as before: chunk 0, 1, ...
      const float w = fast_exp2(mc[c] - m);
      l += w * lc[c];
      acc += w * oc[c];
    }
  }
  out[((int64_t)r * hq + hh) * kHeadDim + d] = DTypeTraits<T>::from_float(acc / l);
}


}  // namespace b200
