// Memory-bound elementwise kernels of the attention path, sm_90a:
//   K1 store_kv        (reference: python/minisgl/kernel/csrc/jit/store.cu:28-53)
//   K7 rmsnorm / fused_add_rmsnorm (reference call sites python/minisgl/layers/norm.py:8-38)
//   K6 rope_neox       (reference call site python/minisgl/layers/rotary.py:45-51)
//   fused qk-norm + rope (the three launches of python/minisgl/layers/attention.py:50-54 in one)
// All are HBM-bound: 128-bit coalesced accesses, loads batched before stores, no smem staging
// (no reuse), grids sized from the row count.
#include "b200attn.h"
#include "common.cuh"
#include "qknorm_rope.cuh"

namespace b200 {

// =============================================================================== K1 store
// One warp per token: copies the K row and the V row (row_bytes each) with 16-byte lanes.
// All loads of a lane are issued before its stores so 2*ceil(row/512) requests are in flight.
template <typename IdxT, int kMaxIter>
__global__ void __launch_bounds__(256) store_kv_kernel(
    uint8_t* __restrict__ k_cache, uint8_t* __restrict__ v_cache, int64_t cache_stride,
    const uint8_t* __restrict__ k, const uint8_t* __restrict__ v, int64_t in_stride,
    const IdxT* __restrict__ indices, int64_t n, int chunks /* row_bytes / 16 */) {
  const int64_t token = (int64_t)blockIdx.x * (blockDim.x / kWarp) + threadIdx.x / kWarp;
  const int lane = threadIdx.x % kWarp;
  if (token >= n) return;
  const int64_t slot = (int64_t)indices[token];
  const uint8_t* ks = k + token * in_stride;
  const uint8_t* vs = v + token * in_stride;
  uint8_t* kd = k_cache + slot * cache_stride;
  uint8_t* vd = v_cache + slot * cache_stride;
  if constexpr (kMaxIter > 0) {
    Vec8 a[kMaxIter], b[kMaxIter];
#pragma unroll
    for (int i = 0; i < kMaxIter; ++i) {
      int c = lane + i * kWarp;
      if (c < chunks) {
        a[i] = ldg_stream(ks + c * 16);
        b[i] = ldg_stream(vs + c * 16);
      }
    }
#pragma unroll
    for (int i = 0; i < kMaxIter; ++i) {
      int c = lane + i * kWarp;
      if (c < chunks) {
        stg_stream(kd + c * 16, a[i]);
        stg_stream(vd + c * 16, b[i]);
      }
    }
  } else {
    for (int c = lane; c < chunks; c += kWarp) {
      Vec8 a = ldg_stream(ks + c * 16), b = ldg_stream(vs + c * 16);
      stg_stream(kd + c * 16, a);
      stg_stream(vd + c * 16, b);
    }
  }
}

template <typename IdxT>
static int launch_store(uint8_t* kc, uint8_t* vc, int64_t cs, const uint8_t* k, const uint8_t* v,
                        int64_t is, const void* idx, int64_t n, int chunks, cudaStream_t st) {
  const int warps = 8;
  dim3 grid((unsigned)ceil_div<int64_t>(n, warps)), block(warps * kWarp);
  if (chunks <= 32 * 4) {  // rows up to 2 KiB (Hkv_local*D*2 for every BASELINE config)
    store_kv_kernel<IdxT, 4><<<grid, block, 0, st>>>(kc, vc, cs, k, v, is, (const IdxT*)idx, n,
                                                     chunks);
  } else {
    store_kv_kernel<IdxT, 0><<<grid, block, 0, st>>>(kc, vc, cs, k, v, is, (const IdxT*)idx, n,
                                                     chunks);
  }
  B200_POST_LAUNCH();
  return 0;
}

// ============================================================================ K7 rmsnorm
// Small rows (dim = 8*G, G in {8,16,32} lanes): one lane-group per (row, head).
template <typename T, int G>
__global__ void __launch_bounds__(256) rmsnorm_group_kernel(
    T* out, const T* x /* may alias out */, const T* __restrict__ w, int64_t rows, int heads,
    int64_t xrs, int64_t xhs, int64_t ors, int64_t ohs, float eps) {
  constexpr int kDim = G * 8;
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const int j = threadIdx.x % G;
  const bool active = gid < rows * heads;
  const int64_t r = active ? gid / heads : 0;
  const int h = active ? (int)(gid % heads) : 0;
  float f[8], wf[8];
  Vec8 xv = {}, wv = {};
  if (active) {
    xv = *reinterpret_cast<const Vec8*>(x + r * xrs + h * xhs + j * 8);
    wv = *reinterpret_cast<const Vec8*>(w + j * 8);
  }
  unpack8<T>(xv, f);
  unpack8<T>(wv, wf);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rcp = rsqrtf(ss / (float)kDim + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = f[i] * rcp * wf[i];
  if (active) *reinterpret_cast<Vec8*>(out + r * ors + h * ohs + j * 8) = pack8<T>(f);
}

// block-wide sum, result broadcast to all threads
__device__ __forceinline__ float block_sum(float v, float* red /* [33] */) {
  const int lane = threadIdx.x % kWarp, wid = threadIdx.x / kWarp;
  const int nw = (blockDim.x + kWarp - 1) / kWarp;
  v = warp_sum(v);
  if (lane == 0) red[wid] = v;
  __syncthreads();
  if (wid == 0) {
    float t = lane < nw ? red[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}

// General rows: one CTA per row, <= kIter 16-byte chunks per thread kept in registers.
template <typename T, int kIter, bool kFusedAdd>
__global__ void __launch_bounds__(1024) rmsnorm_row_kernel(T* out_or_x,
                                                           const T* x_in /* may alias out */,
                                                           T* residual,
                                                           const T* __restrict__ w, int dim,
                                                           int64_t xrs, int64_t ors_or_rrs,
                                                           float eps) {
  __shared__ float red[33];
  const int64_t r = blockIdx.x;
  const int chunks = dim / 8;
  float f[kIter][8];
  float ss = 0.f;
#pragma unroll
  for (int it = 0; it < kIter; ++it) {
    const int c = threadIdx.x + it * blockDim.x;
    if (c < chunks) {
      Vec8 xv = *reinterpret_cast<const Vec8*>(x_in + r * xrs + c * 8);
      unpack8<T>(xv, f[it]);
      if constexpr (kFusedAdd) {
        Vec8 rv = *reinterpret_cast<const Vec8*>(residual + r * ors_or_rrs + c * 8);
        float g[8];
        unpack8<T>(rv, g);
#pragma unroll
        for (int i = 0; i < 8; ++i) f[it][i] += g[i];
        // residual <- round(x + residual); the norm below uses the unrounded fp32 sum
        *reinterpret_cast<Vec8*>(residual + r * ors_or_rrs + c * 8) = pack8<T>(f[it]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) ss += f[it][i] * f[it][i];
    }
  }
  const float tot = block_sum(ss, red);
  const float rcp = rsqrtf(tot / (float)dim + eps);
#pragma unroll
  for (int it = 0; it < kIter; ++it) {
    const int c = threadIdx.x + it * blockDim.x;
    if (c < chunks) {
      Vec8 wv = *reinterpret_cast<const Vec8*>(w + c * 8);
      float wf[8];
      unpack8<T>(wv, wf);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[it][i] = f[it][i] * rcp * wf[i];
      T* dst = kFusedAdd ? (out_or_x + r * xrs) : (out_or_x + r * ors_or_rrs);
      *reinterpret_cast<Vec8*>(dst + c * 8) = pack8<T>(f[it]);
    }
  }
}

template <typename T>
static int launch_rmsnorm(void* out, const void* x, const void* w, int64_t rows, int heads, int dim,
                          int64_t xrs, int64_t xhs, int64_t ors, int64_t ohs, float eps,
                          cudaStream_t st) {
  if (rows == 0) return 0;
  const int g = dim / 8;
  if (dim % 8 == 0 && (g == 8 || g == 16 || g == 32)) {
    const int64_t threads = rows * heads * g;
    dim3 grid((unsigned)ceil_div<int64_t>(threads, 256)), block(256);
#define L(G_)                                                                                  \
  rmsnorm_group_kernel<T, G_><<<grid, block, 0, st>>>((T*)out, (const T*)x, (const T*)w, rows, \
                                                      heads, xrs, xhs, ors, ohs, eps)
    if (g == 8) L(8);
    else if (g == 16) L(16);
    else L(32);
#undef L
    B200_POST_LAUNCH();
    return 0;
  }
  B200_CHECK_ARG(heads == 1, "rmsnorm: multi-head rows need dim in {64,128,256}, got %d", dim);
  const int chunks = dim / 8;
  int threads = (int)ceil_div(chunks, 32) * 32;
  if (threads > 1024) threads = 1024;
  if (chunks > 512) threads = (int)ceil_div(ceil_div(chunks, 2), 32) * 32;
  const int iters = ceil_div(chunks, threads);
  B200_CHECK_ARG(iters <= 2, "rmsnorm: dim %d too large (max 16384)", dim);
  dim3 grid((unsigned)rows), block(threads);
  if (iters == 1)
    rmsnorm_row_kernel<T, 1, false><<<grid, block, 0, st>>>((T*)out, (const T*)x, nullptr,
                                                            (const T*)w, dim, xrs, ors, eps);
  else
    rmsnorm_row_kernel<T, 2, false><<<grid, block, 0, st>>>((T*)out, (const T*)x, nullptr,
                                                            (const T*)w, dim, xrs, ors, eps);
  B200_POST_LAUNCH();
  return 0;
}

template <typename T>
static int launch_fused_add_rmsnorm(void* x, void* res, const void* w, int64_t rows, int dim,
                                    int64_t xrs, int64_t rrs, float eps, cudaStream_t st) {
  if (rows == 0) return 0;
  const int chunks = dim / 8;
  int threads = (int)ceil_div(chunks, 32) * 32;
  if (threads > 1024) threads = 1024;
  if (chunks > 512) threads = (int)ceil_div(ceil_div(chunks, 2), 32) * 32;
  const int iters = ceil_div(chunks, threads);
  B200_CHECK_ARG(iters <= 2, "fused_add_rmsnorm: dim %d too large (max 16384)", dim);
  dim3 grid((unsigned)rows), block(threads);
  if (iters == 1)
    rmsnorm_row_kernel<T, 1, true><<<grid, block, 0, st>>>((T*)x, (const T*)x, (T*)res,
                                                           (const T*)w, dim, xrs, rrs, eps);
  else
    rmsnorm_row_kernel<T, 2, true><<<grid, block, 0, st>>>((T*)x, (const T*)x, (T*)res,
                                                           (const T*)w, dim, xrs, rrs, eps);
  B200_POST_LAUNCH();
  return 0;
}

// ====================================================== K6 rope / fused qk-norm + rope
// One lane-group of G = D/8 lanes per (token, head); lane j holds elements [8j, 8j+8).
// Lanes j < G/2 hold the first half, their rotation partner is lane j ^ (G/2).
template <typename T, typename PosT, int G, bool kNorm>
__global__ void __launch_bounds__(256) qknorm_rope_kernel(
    T* __restrict__ q, T* __restrict__ k, const T* __restrict__ qw, const T* __restrict__ kw,
    float eps, const PosT* __restrict__ positions, const float* __restrict__ cos_sin, int64_t nnz,
    int hq, int hkv, int64_t qrs, int64_t krs) {
  constexpr int kDim = G * 8;
  pdl_wait();
  pdl_launch_dependents();
  const int heads = hq + hkv;
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const int j = threadIdx.x % G;
  const bool active = gid < nnz * heads;
  const int64_t t = active ? gid / heads : 0;
  const int h = active ? (int)(gid % heads) : 0;
  const bool is_q = h < hq;
  T* ptr = is_q ? (q + t * qrs + (int64_t)h * kDim) : (k + t * krs + (int64_t)(h - hq) * kDim);
  Vec8 xv = {};
  if (active) xv = *reinterpret_cast<const Vec8*>(ptr + j * 8);
  const T* w = kNorm ? (is_q ? qw : kw) : nullptr;
  const float* cs_row = cos_sin + (active ? (int64_t)positions[t] : 0) * kDim;
  // (two rows per lane group were tried for more bytes in flight: 67 us vs 59 us on 16 384 tokens -- slower)
  const Vec8 out = qknorm_rope_lanes<T, G, kNorm>(xv, j, w, eps, cs_row, active);
  if (active) *reinterpret_cast<Vec8*>(ptr + j * 8) = out;
}

template <typename T, typename PosT, bool kNorm>
static int launch_qknorm_rope_g(void* q, void* k, const void* qw, const void* kw, float eps,
                                const void* pos, const float* cs, int64_t nnz, int hq, int hkv,
                                int d, int64_t qrs, int64_t krs, cudaStream_t st) {
  if (nnz == 0) return 0;
  const int g = d / 8;
  const int64_t threads = nnz * (hq + hkv) * g;
  dim3 grid((unsigned)ceil_div<int64_t>(threads, 256)), block(256);
#define L(G_)                                                                                        \
  B200_CHECK_CUDA(launch_pdl(qknorm_rope_kernel<T, PosT, G_, kNorm>, grid, block, 0, st, (T*)q, (T*)k, \
                             (const T*)qw, (const T*)kw, eps, (const PosT*)pos, cs, nnz, hq, hkv, qrs, krs))
  if (g == 8) L(8);
  else if (g == 16) L(16);
  else if (g == 32) L(32);
  else {
    set_error("rope: head_dim must be 64, 128 or 256 (got %d)", d);
    return 1;
  }
#undef L
  B200_POST_LAUNCH();
  return 0;
}

template <bool kNorm>
static int launch_qknorm_rope(void* q, void* k, const void* qw, const void* kw, float eps,
                              const void* pos, int pos64, const float* cs, int64_t nnz, int hq,
                              int hkv, int d, int64_t qrs, int64_t krs, int dtype,
                              cudaStream_t st) {
  B200_CHECK_ARG(dtype == B200_DTYPE_BF16 || dtype == B200_DTYPE_FP16, "bad dtype %d", dtype);
  B200_CHECK_ARG(qrs % 8 == 0 && krs % 8 == 0, "rope: row strides must be multiples of 8");
  B200_CHECK_ARG(((uintptr_t)q % 16) == 0 && ((uintptr_t)k % 16) == 0, "rope: q/k not 16B aligned");
  if (dtype == B200_DTYPE_BF16) {
    return pos64 ? launch_qknorm_rope_g<__nv_bfloat16, int64_t, kNorm>(q, k, qw, kw, eps, pos, cs,
                                                                      nnz, hq, hkv, d, qrs, krs, st)
                 : launch_qknorm_rope_g<__nv_bfloat16, int32_t, kNorm>(q, k, qw, kw, eps, pos, cs,
                                                                      nnz, hq, hkv, d, qrs, krs, st);
  }
  return pos64 ? launch_qknorm_rope_g<__half, int64_t, kNorm>(q, k, qw, kw, eps, pos, cs, nnz, hq,
                                                             hkv, d, qrs, krs, st)
               : launch_qknorm_rope_g<__half, int32_t, kNorm>(q, k, qw, kw, eps, pos, cs, nnz, hq,
                                                             hkv, d, qrs, krs, st);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_store_kv(void* k_cache, void* v_cache, int64_t cache_row_stride_bytes,
                             const void* k, const void* v, int64_t input_row_stride_bytes,
                             const void* indices, int idx64, int64_t num_tokens, int64_t row_bytes,
                             void* stream) {
  B200_CHECK_ARG(row_bytes > 0 && row_bytes % 16 == 0, "store_kv: row_bytes %lld not a multiple of 16",
                 (long long)row_bytes);
  B200_CHECK_ARG(cache_row_stride_bytes % 16 == 0 && input_row_stride_bytes % 16 == 0,
                 "store_kv: strides must be multiples of 16 bytes");
  B200_CHECK_ARG(((uintptr_t)k_cache % 16) == 0 && ((uintptr_t)v_cache % 16) == 0 &&
                     ((uintptr_t)k % 16) == 0 && ((uintptr_t)v % 16) == 0,
                 "store_kv: pointers must be 16-byte aligned");
  B200_CHECK_ARG(num_tokens >= 0, "store_kv: negative length");
  if (num_tokens == 0) return 0;
  auto st = (cudaStream_t)stream;
  const int chunks = (int)(row_bytes / 16);
  if (idx64)
    return launch_store<int64_t>((uint8_t*)k_cache, (uint8_t*)v_cache, cache_row_stride_bytes,
                                 (const uint8_t*)k, (const uint8_t*)v, input_row_stride_bytes,
                                 indices, num_tokens, chunks, st);
  return launch_store<int32_t>((uint8_t*)k_cache, (uint8_t*)v_cache, cache_row_stride_bytes,
                               (const uint8_t*)k, (const uint8_t*)v, input_row_stride_bytes, indices,
                               num_tokens, chunks, st);
}

extern "C" int b200_rmsnorm(void* out, const void* x, const void* weight, int64_t rows, int heads,
                            int dim, int64_t x_row_stride, int64_t x_head_stride,
                            int64_t out_row_stride, int64_t out_head_stride, float eps, int dtype,
                            void* stream) {
  B200_CHECK_ARG(dim > 0 && dim % 8 == 0, "rmsnorm: dim %d must be a positive multiple of 8", dim);
  B200_CHECK_ARG(heads >= 1, "rmsnorm: heads must be >= 1");
  B200_CHECK_ARG(x_row_stride % 8 == 0 && out_row_stride % 8 == 0 && x_head_stride % 8 == 0 &&
                     out_head_stride % 8 == 0,
                 "rmsnorm: strides must be multiples of 8 elements");
  B200_CHECK_ARG(((uintptr_t)out % 16) == 0 && ((uintptr_t)x % 16) == 0 &&
                     ((uintptr_t)weight % 16) == 0,
                 "rmsnorm: pointers must be 16-byte aligned");
  auto st = (cudaStream_t)stream;
  if (dtype == B200_DTYPE_BF16)
    return launch_rmsnorm<__nv_bfloat16>(out, x, weight, rows, heads, dim, x_row_stride,
                                         x_head_stride, out_row_stride, out_head_stride, eps, st);
  if (dtype == B200_DTYPE_FP16)
    return launch_rmsnorm<__half>(out, x, weight, rows, heads, dim, x_row_stride, x_head_stride,
                                  out_row_stride, out_head_stride, eps, st);
  set_error("rmsnorm: bad dtype %d", dtype);
  return 1;
}

extern "C" int b200_fused_add_rmsnorm(void* x, void* residual, const void* weight, int64_t rows,
                                      int dim, int64_t x_row_stride, int64_t res_row_stride,
                                      float eps, int dtype, void* stream) {
  B200_CHECK_ARG(dim > 0 && dim % 8 == 0, "fused_add_rmsnorm: dim %d must be a multiple of 8", dim);
  B200_CHECK_ARG(x_row_stride % 8 == 0 && res_row_stride % 8 == 0,
                 "fused_add_rmsnorm: strides must be multiples of 8 elements");
  B200_CHECK_ARG(((uintptr_t)x % 16) == 0 && ((uintptr_t)residual % 16) == 0 &&
                     ((uintptr_t)weight % 16) == 0,
                 "fused_add_rmsnorm: pointers must be 16-byte aligned");
  auto st = (cudaStream_t)stream;
  if (dtype == B200_DTYPE_BF16)
    return launch_fused_add_rmsnorm<__nv_bfloat16>(x, residual, weight, rows, dim, x_row_stride,
                                                   res_row_stride, eps, st);
  if (dtype == B200_DTYPE_FP16)
    return launch_fused_add_rmsnorm<__half>(x, residual, weight, rows, dim, x_row_stride,
                                            res_row_stride, eps, st);
  set_error("fused_add_rmsnorm: bad dtype %d", dtype);
  return 1;
}

extern "C" int b200_rope_neox_inplace(void* q, void* k, const void* positions, int pos64,
                                      const float* cos_sin_cache, int64_t nnz, int hq, int hkv,
                                      int head_dim, int64_t q_row_stride, int64_t k_row_stride,
                                      int dtype, void* stream) {
  return launch_qknorm_rope<false>(q, k, nullptr, nullptr, 0.f, positions, pos64, cos_sin_cache,
                                   nnz, hq, hkv, head_dim, q_row_stride, k_row_stride, dtype,
                                   (cudaStream_t)stream);
}

extern "C" int b200_qknorm_rope_inplace(void* q, void* k, const void* q_weight,
                                        const void* k_weight, float eps, const void* positions,
                                        int pos64, const float* cos_sin_cache, int64_t nnz, int hq,
                                        int hkv, int head_dim, int64_t q_row_stride,
                                        int64_t k_row_stride, int dtype, void* stream) {
  return launch_qknorm_rope<true>(q, k, q_weight, k_weight, eps, positions, pos64, cos_sin_cache,
                                  nnz, hq, hkv, head_dim, q_row_stride, k_row_stride, dtype,
                                  (cudaStream_t)stream);
}
