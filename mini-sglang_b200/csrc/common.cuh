// Shared device/host helpers for the sm_90a kernels of libb200attn.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <utility>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

namespace b200 {

// ----------------------------------------------------------------------------- host side
void set_error(const char* fmt, ...);  // defined in capi.cu (thread-local buffer)
extern std::atomic<uint64_t> g_launch_count;

#define B200_CHECK_ARG(cond, ...)    \
  do {                               \
    if (!(cond)) {                   \
      ::b200::set_error(__VA_ARGS__); \
      return 1;                      \
    }                                \
  } while (0)

// A failed runtime call also records its error as the thread's last error; it is cleared here, so that it
// is reported by this call only and not again by the next launch check (sticky errors stay sticky).
#define B200_CHECK_CUDA(expr)                                                       \
  do {                                                                              \
    cudaError_t err__ = (expr);                                                     \
    if (err__ != cudaSuccess) {                                                     \
      (void)cudaGetLastError();                                                     \
      ::b200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(err__),  \
                        __FILE__, __LINE__);                                        \
      return 2;                                                                     \
    }                                                                               \
  } while (0)

// call after every <<< >>> launch: reports (and clears) a launch error once
#define B200_POST_LAUNCH()                        \
  do {                                            \
    ::b200::g_launch_count.fetch_add(1);          \
    B200_CHECK_CUDA(cudaGetLastError());          \
  } while (0)

inline int num_sms() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
    if (cached <= 0) cached = 132;
  }
  return cached;
}

// b200_set_option knobs (defined, with their defaults, in capi.cu; include/b200attn.h documents them)
extern std::atomic<int> g_use_pdl;
extern std::atomic<int> g_decode_impl;
extern std::atomic<int> g_prefill_impl;
extern std::atomic<int> g_prefill_order;
extern std::atomic<int> g_prefill_skip_append;
extern std::atomic<int> g_decode_plan_target;
extern std::atomic<int> g_decode_plan_nosplit;
extern std::atomic<int> g_decode_fused_combine;
extern std::atomic<int> g_decode_early_kv;
extern std::atomic<int> g_decode_exact_tail;

// kernel<<<grid, block, smem, stream>>>(args...) with the programmatic-stream-serialization attribute
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = g_use_pdl.load() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

template <typename T>
constexpr T ceil_div(T a, T b) {
  return (a + b - 1) / b;
}

// --------------------------------------------------------------------------- device side
constexpr int kWarp = 32;
constexpr float kLog2e = 1.4426950408889634f;

template <typename T>
struct DTypeTraits;
template <>
struct DTypeTraits<__nv_bfloat16> {
  using T2 = __nv_bfloat162;
  static __device__ __forceinline__ float to_float(__nv_bfloat16 x) { return __bfloat162float(x); }
  static __device__ __forceinline__ __nv_bfloat16 from_float(float x) {
    return __float2bfloat16_rn(x);
  }
  static __device__ __forceinline__ float2 to_float2(__nv_bfloat162 x) {
    return __bfloat1622float2(x);
  }
  static __device__ __forceinline__ __nv_bfloat162 from_float2(float a, float b) {
    return __floats2bfloat162_rn(a, b);
  }
};
template <>
struct DTypeTraits<__half> {
  using T2 = __half2;
  static __device__ __forceinline__ float to_float(__half x) { return __half2float(x); }
  static __device__ __forceinline__ __half from_float(float x) { return __float2half_rn(x); }
  static __device__ __forceinline__ float2 to_float2(__half2 x) { return __half22float2(x); }
  static __device__ __forceinline__ __half2 from_float2(float a, float b) {
    return __floats2half2_rn(a, b);
  }
};

// 16-byte vector of 8 16-bit values
struct alignas(16) Vec8 {
  uint32_t w[4];
};

template <typename T>
__device__ __forceinline__ void unpack8(const Vec8& v, float (&f)[8]) {
  using Tr = DTypeTraits<T>;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    typename Tr::T2 p = *reinterpret_cast<const typename Tr::T2*>(&v.w[i]);
    float2 x = Tr::to_float2(p);
    f[2 * i] = x.x;
    f[2 * i + 1] = x.y;
  }
}

template <typename T>
__device__ __forceinline__ Vec8 pack8(const float (&f)[8]) {
  using Tr = DTypeTraits<T>;
  Vec8 v;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    typename Tr::T2 p = Tr::from_float2(f[2 * i], f[2 * i + 1]);
    v.w[i] = *reinterpret_cast<uint32_t*>(&p);
  }
  return v;
}

__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}
__device__ __forceinline__ float warp_max(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// streaming 16-byte global load / store (bypass L1 allocation)
__device__ __forceinline__ Vec8 ldg_stream(const void* p) {
  Vec8 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.w[0]), "=r"(r.w[1]), "=r"(r.w[2]), "=r"(r.w[3])
               : "l"(p));
  return r;
}
__device__ __forceinline__ void stg_stream(void* p, const Vec8& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]),
               "r"(v.w[1]), "r"(v.w[2]), "r"(v.w[3])
               : "memory");
}

// cp.async 16 B global -> shared (LDGSTS), L2-only caching
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gptr)
               : "memory");
}
// as cp_async16, but !valid writes 16 zero bytes and reads nothing
__device__ __forceinline__ void cp_async16_zfill(uint32_t smem_addr, const void* gptr, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr), "l"(gptr), "r"(sz)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Programmatic dependent launch (PDL): a kernel launched with launch_pdl() may start while its
// predecessor in the stream is still running; it must execute pdl_wait() before it reads anything
// the predecessor writes or writes anything the predecessor (or ITS predecessors) may still read.
// Every PDL kernel of this library waits before its first global write, so completion stays
// transitive along the stream.  pdl_launch_dependents() lets the successor begin its prologue.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

}  // namespace b200
