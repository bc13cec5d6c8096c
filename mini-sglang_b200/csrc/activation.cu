// Gated-MLP activation: out[t, i] = silu(x[t, i]) * x[t, d + i] for x of shape [rows, 2d].
//
// Replaces flashinfer.silu_and_mul, which GatedMLP.forward calls through python/minisgl/layers/activation.py:9-13
// for every dense model the reference serves (models/utils.py:33).  HBM-bound: 4 * d bytes read and 2 * d
// written per row, no reuse.
//
// Bit identity with FlashInfer: its JIT modules are compiled with -use_fast_math, so its
// `v / (1.0f + __expf(-v)) * y` becomes the five fp32 instructions of silu_mul() below (ftz multiply by
// -log2(e), ex2.approx.ftz, ftz add of 1, div.approx.ftz, ftz multiply by the up value), then one
// round-to-nearest conversion.  This library is not built with fast math, so the sequence is spelled out in
// PTX: the same SASS (FMUL.FTZ, MUFU.EX2, FADD.FTZ, MUFU.RCP + FMUL.FTZ, FMUL.FTZ, F2FP) comes out whatever
// the compiler flags.
#include "b200attn.h"
#include "common.cuh"

namespace b200 {

__device__ __forceinline__ float silu_mul(float g, float u) {
  float t, e, den, s, r;
  asm("mul.ftz.f32 %0, %1, 0fBFB8AA3B;" : "=f"(t) : "f"(g));  // -log2(e) * g
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
  asm("add.ftz.f32 %0, %1, 0f3F800000;" : "=f"(den) : "f"(e));
  asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(s) : "f"(g), "f"(den));
  asm("mul.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(s), "f"(u));
  return r;
}

// 16-byte path: rows are 16-byte aligned and d % 8 == 0.  blockIdx.x picks 8-wide column vectors, blockIdx.y
// (strided by gridDim.y) the rows: no 64-bit index division, one gate and one up load per thread per row.
template <typename T>
__global__ void __launch_bounds__(128) silu_and_mul_vec_kernel(T* __restrict__ out, int64_t out_stride,
                                                               const T* __restrict__ x, int64_t x_stride,
                                                               int64_t rows, int d) {
  pdl_wait();
  pdl_launch_dependents();
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (c >= d) return;
  for (int64_t r = blockIdx.y; r < rows; r += gridDim.y) {
    const T* xr = x + r * x_stride + c;
    const Vec8 gv = ldg_stream(xr), uv = ldg_stream(xr + d);
    float g[8], u[8];
    unpack8<T>(gv, g);
    unpack8<T>(uv, u);
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = silu_mul(g[i], u[i]);
    stg_stream(out + r * out_stride + c, pack8<T>(g));
  }
}

// Any d, any element-aligned rows: one element per thread.
template <typename T>
__global__ void __launch_bounds__(256) silu_and_mul_scalar_kernel(T* __restrict__ out, int64_t out_stride,
                                                                  const T* __restrict__ x, int64_t x_stride,
                                                                  int64_t rows, int d) {
  using Tr = DTypeTraits<T>;
  pdl_wait();
  pdl_launch_dependents();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d) return;
  for (int64_t r = blockIdx.y; r < rows; r += gridDim.y) {
    const T* xr = x + r * x_stride;
    out[r * out_stride + i] = Tr::from_float(silu_mul(Tr::to_float(xr[i]), Tr::to_float(xr[d + i])));
  }
}

template <typename T>
static int launch_silu_and_mul(void* out, int64_t ors, const void* x, int64_t xrs, int64_t rows, int d,
                               cudaStream_t st) {
  const bool vec = d % 8 == 0 && ors % 8 == 0 && xrs % 8 == 0 && (uintptr_t)out % 16 == 0 &&
                   (uintptr_t)x % 16 == 0;
  const unsigned grid_rows = (unsigned)(rows < 65535 ? rows : 65535);
  if (vec) {
    const dim3 grid((unsigned)ceil_div(d / 8, 128), grid_rows);
    B200_CHECK_CUDA(launch_pdl(silu_and_mul_vec_kernel<T>, grid, dim3(128), 0, st, (T*)out, ors, (const T*)x,
                               xrs, rows, d));
  } else {
    const dim3 grid((unsigned)ceil_div(d, 256), grid_rows);
    B200_CHECK_CUDA(launch_pdl(silu_and_mul_scalar_kernel<T>, grid, dim3(256), 0, st, (T*)out, ors,
                               (const T*)x, xrs, rows, d));
  }
  B200_POST_LAUNCH();
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_silu_and_mul(void* out, int64_t out_row_stride, const void* x, int64_t x_row_stride,
                                 int64_t rows, int d, int dtype, void* stream) {
  B200_CHECK_ARG(dtype == B200_DTYPE_BF16 || dtype == B200_DTYPE_FP16, "silu_and_mul: bad dtype %d", dtype);
  B200_CHECK_ARG(d >= 1 && d <= (1 << 30), "silu_and_mul: d %d must lie in [1, 2^30]", d);
  B200_CHECK_ARG(rows >= 0, "silu_and_mul: negative row count");
  B200_CHECK_ARG(x_row_stride >= 2 * (int64_t)d && out_row_stride >= d,
                 "silu_and_mul: row strides must cover a row (x >= 2d, out >= d elements)");
  B200_CHECK_ARG(((uintptr_t)out % 2) == 0 && ((uintptr_t)x % 2) == 0,
                 "silu_and_mul: pointers must be aligned to the 2-byte element");
  if (rows == 0) return 0;
  auto st = (cudaStream_t)stream;
  if (dtype == B200_DTYPE_BF16)
    return launch_silu_and_mul<__nv_bfloat16>(out, out_row_stride, x, x_row_stride, rows, d, st);
  return launch_silu_and_mul<__half>(out, out_row_stride, x, x_row_stride, rows, d, st);
}
