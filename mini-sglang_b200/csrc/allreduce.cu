// One-shot tensor-parallel all-reduce over NVLink peer memory, fused with the residual add + RMSNorm
// that follows it (SURVEY 8(f) rank 4).
//
// Replaces, for decode-sized messages, the reference's capturable NCCL wrapper
//   PyNCCLCommunicator.all_reduce  (python/minisgl/kernel/csrc/src/pynccl.cu:93-134: D2D copy into
//   the symmetric window, ncclAllReduce, D2D copy back), called once per layer after o_proj
//   (python/minisgl/layers/linear.py:102-106) and after the MLP down projection (linear.py:122-126),
// and optionally the flashinfer.fused_add_rmsnorm that consumes its result
//   (python/minisgl/layers/norm.py:32-38 via models/qwen3.py:38-41).
//
// Design (one-shot "push", flag-in-data / Lamport style: one kernel, no fence, no separate flag):
//   every rank owns a region  data[2 parities][world senders][slot] | (reserved) | epoch, done
//   that all peers have mapped (CUDA IPC).  At rest every 16-bit lane of the data region holds the SENTINEL
//   0x8000 (negative zero).  A thread of CTA b of rank s
//     1. loads its 16-byte chunk of x (any device memory, no staging copy), replaces -0.0 lanes by +0.0 (so a
//        payload never contains the sentinel) and STORES it into slot[parity][s] of EVERY rank -- 16-byte
//        peer stores over NVLink, posted writes, no round trip;
//     2. polls the same chunk of slot[parity][0..world) in its OWN region (volatile 16-byte loads from L2)
//        until no lane is the sentinel: the data is its own arrival flag (a 16-byte store lands atomically), so
//        there is no system-scope fence, no flag store and no flag propagation on the critical path, and no
//        CTA-level synchronisation at all -- the thread that pushed chunk c is the thread that reduces it;
//     3. sums the world chunks in rank order in fp32 (every rank gets bit-identical results; == NCCL at world 2
//        except for the sign of an all-negative-zero sum), rounds once to the 16-bit type (= the tensor the
//        reference's all-reduce returns), writes the sentinel back into the chunks it consumed, and either
//        stores the sum or applies  residual <- round(y + residual); out <- rmsnorm(y + residual) * w  with
//        the arithmetic of rmsnorm_row_kernel<.., kFusedAdd> (elementwise.cu), bit for bit.
//   The parity alternates per launch and comes from a device-resident epoch (advanced by the last CTA of each
//   launch), so the kernel is CUDA-graph capturable and replays correctly.  Two parities suffice: a rank can
//   only push launch e+2 (same parity as e) after it finished launch e+1, i.e. after it received every peer's
//   e+1 chunks, which those peers sent after completing (reading AND re-arming) launch e.
//   Polls are bounded (globaltimer): a dead peer traps the kernel instead of hanging the GPU.
//
// Bytes per launch and rank: world x rows x dim x 2 pushed over NVLink (incl. the local copy), the same amount
// read back and re-armed locally; latency-bound for the <= 512 KB messages of decode (one NVLink write flight).
#include "b200attn.h"
#include "common.cuh"

#include <cstring>
#include <type_traits>

namespace b200 {
namespace ar {

constexpr int kMaxWorld = 8;
constexpr int kMaxCtas = 512;  // one CTA per row up to 512 rows: the reduce phase is one row deep

struct Comm {
  int rank, world;
  size_t slot_bytes;   // capacity of one sender slot (max message bytes, 256-aligned)
  size_t flags_off, ctr_off, region_bytes;
  uint8_t* base[kMaxWorld];  // base[rank] = local region, others = IPC mappings
  void* opened[kMaxWorld];   // mappings this process opened (closed in destroy)
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

template <typename T>
struct Params {
  const T* x;
  int64_t x_rs;
  T* out;
  int64_t out_rs;
  T* residual;
  int64_t res_rs;
  const T* w;
  int rows, dim;
  float eps;
  int rank, world;
  size_t slot_bytes, flags_off, ctr_off;
  uint8_t* base[kMaxWorld];
};

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ Vec8 ld_volatile16(const void* p) {
  Vec8 r;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.w[0]), "=r"(r.w[1]), "=r"(r.w[2]), "=r"(r.w[3])
               : "l"(p)
               : "memory");
  return r;
}
constexpr uint32_t kSentinel2 = 0x80008000u;  // two 16-bit negative zeros
__device__ __forceinline__ bool has_sentinel(const Vec8& v) {
  bool hit = false;
#pragma unroll
  for (int i = 0; i < 4; ++i) hit |= ((v.w[i] & 0xffffu) == 0x8000u) | ((v.w[i] >> 16) == 0x8000u);
  return hit;
}
__device__ __forceinline__ Vec8 without_negative_zero(Vec8 v) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if ((v.w[i] & 0xffffu) == 0x8000u) v.w[i] &= 0xffff0000u;
    if ((v.w[i] >> 16) == 0x8000u) v.w[i] &= 0x0000ffffu;
  }
  return v;
}

// block-wide sum with the reduction order of elementwise.cu::block_sum (bit-identical norms)
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

template <typename T, int kIter, bool kNorm>
__global__ void __launch_bounds__(512) allreduce_push_kernel(const Params<T> p) {
  __shared__ float red[33];
  __shared__ uint32_t s_epoch;
  const int b = blockIdx.x, grid = gridDim.x, tid = threadIdx.x;
  const int chunks = p.dim / 8;
  uint8_t* mine = p.base[p.rank];
  uint32_t* ctr = reinterpret_cast<uint32_t*>(mine + p.ctr_off);
  // programmatic dependent launch: x is the predecessor's output (and the epoch counter was advanced by the
  // previous all-reduce, complete by transitivity); the successor may begin its own prologue right away
  pdl_wait();
  pdl_launch_dependents();
  // the first row's chunks of x are requested before the epoch is read: the two global round trips overlap
  Vec8 x0[kIter];
#pragma unroll
  for (int it = 0; it < kIter; ++it) {
    const int c = tid + it * blockDim.x;
    if (b < p.rows && c < chunks) x0[it] = *reinterpret_cast<const Vec8*>(p.x + (int64_t)b * p.x_rs + c * 8);
  }
  if (tid == 0) {
    // epoch of this launch = stored epoch + 1 (acquire: the count-in below cannot overtake this read)
    uint32_t e;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(e) : "l"(ctr) : "memory");
    s_epoch = e + 1u;
  }
  __syncthreads();
  const uint32_t epoch = s_epoch;
  const size_t parity_off = (size_t)(epoch & 1u) * p.world * p.slot_bytes;

  // ---- 1. push my chunks into slot[parity][rank] of every rank (peers first, own copy last)
  for (int r = b; r < p.rows; r += grid) {
#pragma unroll
    for (int it = 0; it < kIter; ++it) {
      const int c = tid + it * blockDim.x;
      if (c < chunks) {
        const Vec8 v = without_negative_zero(r == b ? x0[it] : *reinterpret_cast<const Vec8*>(p.x + (int64_t)r * p.x_rs + c * 8));
        const size_t off = parity_off + (size_t)p.rank * p.slot_bytes + ((size_t)r * p.dim + c * 8) * sizeof(T);
        for (int i = 1; i <= p.world; ++i) {
          const int t = (p.rank + i) % p.world;
          *reinterpret_cast<Vec8*>(p.base[t] + off) = v;
        }
      }
    }
  }

  // Every CTA counts in after reading the epoch; the CTA that counts in last knows that every CTA of the launch
  // has read the old value and advances it for the next launch.  Done here, between the push and the poll, the
  // atomic's round trip hides behind the NVLink flight of the data instead of extending the kernel's tail.
  if (tid == 0 && atomicAdd(ctr + 1, 1u) == (uint32_t)grid - 1u) {
    ctr[1] = 0u;
    __threadfence();
    *reinterpret_cast<volatile uint32_t*>(ctr) = epoch;
  }

  // ---- 2. + 3. poll my own region for every sender's chunk (the data is its own flag), reduce in rank order,
  // re-arm the consumed chunks with the sentinel, epilogue
  const uint64_t t0 = globaltimer_ns();
  for (int r = b; r < p.rows; r += grid) {
    float f[kIter][8];
    float ss = 0.f;
#pragma unroll
    for (int it = 0; it < kIter; ++it) {
      const int c = tid + it * blockDim.x;
      if (c < chunks) {
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        const size_t off = parity_off + ((size_t)r * p.dim + c * 8) * sizeof(T);
        // all senders' chunks are requested at once (one L2 round trip instead of `world` dependent ones);
        // only the ones that have not landed yet are polled again
        Vec8 v[kMaxWorld];
#pragma unroll
        for (int s = 0; s < kMaxWorld; ++s)
          if (s < p.world) v[s] = ld_volatile16(mine + off + (size_t)s * p.slot_bytes);
        uint32_t spins = 0;
        for (;;) {
          bool missing = false;
#pragma unroll
          for (int s = 0; s < kMaxWorld; ++s)
            if (s < p.world && has_sentinel(v[s])) {
              v[s] = ld_volatile16(mine + off + (size_t)s * p.slot_bytes);
              missing = true;
            }
          if (!missing) break;
          if ((++spins & 0x3ffu) == 0 && globaltimer_ns() - t0 > 8000000000ull) __trap();  // 8 s: a peer died
        }
        Vec8 arm;
        arm.w[0] = arm.w[1] = arm.w[2] = arm.w[3] = kSentinel2;
#pragma unroll
        for (int s = 0; s < kMaxWorld; ++s) {  // rank order: identical bits on every rank
          if (s < p.world) {
            *reinterpret_cast<Vec8*>(mine + off + (size_t)s * p.slot_bytes) = arm;  // ready for the launch after next
            float g[8];
            unpack8<T>(v[s], g);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] += g[i];
          }
        }
        // y = the all-reduced tensor, rounded once to the 16-bit type like the reference's result
        const Vec8 y = pack8<T>(acc);
        if constexpr (!kNorm) {
          *reinterpret_cast<Vec8*>(p.out + (int64_t)r * p.out_rs + c * 8) = y;
        } else {
          unpack8<T>(y, f[it]);
          const Vec8 rv = *reinterpret_cast<const Vec8*>(p.residual + (int64_t)r * p.res_rs + c * 8);
          float g[8];
          unpack8<T>(rv, g);
#pragma unroll
          for (int i = 0; i < 8; ++i) f[it][i] += g[i];
          *reinterpret_cast<Vec8*>(p.residual + (int64_t)r * p.res_rs + c * 8) = pack8<T>(f[it]);
#pragma unroll
          for (int i = 0; i < 8; ++i) ss += f[it][i] * f[it][i];
        }
      }
    }
    if constexpr (kNorm) {
      const float tot = block_sum(ss, red);
      const float rcp = rsqrtf(tot / (float)p.dim + p.eps);
#pragma unroll
      for (int it = 0; it < kIter; ++it) {
        const int c = tid + it * blockDim.x;
        if (c < chunks) {
          const Vec8 wv = *reinterpret_cast<const Vec8*>(p.w + c * 8);
          float wf[8];
          unpack8<T>(wv, wf);
#pragma unroll
          for (int i = 0; i < 8; ++i) f[it][i] = f[it][i] * rcp * wf[i];
          *reinterpret_cast<Vec8*>(p.out + (int64_t)r * p.out_rs + c * 8) = pack8<T>(f[it]);
        }
      }
      __syncthreads();  // red[] is reused by the next row
    }
  }

}

template <typename T>
static int launch(const Comm* c, const void* x, int64_t x_rs, void* out, int64_t out_rs, void* residual,
                  int64_t res_rs, const void* w, int64_t rows, int dim, float eps, cudaStream_t st) {
  Params<T> p;
  p.x = (const T*)x;
  p.x_rs = x_rs;
  p.out = (T*)out;
  p.out_rs = out_rs;
  p.residual = (T*)residual;
  p.res_rs = res_rs;
  p.w = (const T*)w;
  p.rows = (int)rows;
  p.dim = dim;
  p.eps = eps;
  p.rank = c->rank;
  p.world = c->world;
  p.slot_bytes = c->slot_bytes;
  p.flags_off = c->flags_off;
  p.ctr_off = c->ctr_off;
  for (int i = 0; i < kMaxWorld; ++i) p.base[i] = c->base[i];
  // thread <-> chunk mapping of launch_fused_add_rmsnorm (elementwise.cu): identical reductions
  const int chunks = dim / 8;
  int threads = (int)ceil_div(chunks, 32) * 32;
  if (threads > 1024) threads = 1024;
  if (chunks > 512) threads = (int)ceil_div(ceil_div(chunks, 2), 32) * 32;
  const int iters = ceil_div(chunks, threads);
  B200_CHECK_ARG(iters <= 2 && threads <= 512, "allreduce: dim %d too large (max 8192)", dim);
  const int grid = rows < kMaxCtas ? (int)rows : kMaxCtas;
  const bool norm = residual != nullptr;
#define L(IT_, N_) B200_CHECK_CUDA(launch_pdl(allreduce_push_kernel<T, IT_, N_>, dim3(grid), dim3(threads), 0, st, p))
  if (iters == 1) {
    if (norm) L(1, true);
    else L(1, false);
  } else {
    if (norm) L(2, true);
    else L(2, false);
  }
#undef L
  B200_POST_LAUNCH();
  return 0;
}

}  // namespace ar
}  // namespace b200

using namespace b200;

extern "C" size_t b200_ar_region_bytes(int world, size_t max_bytes) {
  const size_t slot = ar::align_up(max_bytes, 256);
  return 2 * (size_t)world * slot + ar::align_up((size_t)world * ar::kMaxCtas * 4, 256) + 256;
}

namespace b200 {
namespace ar {
__global__ void fill_u32_kernel(uint32_t* p, size_t n, uint32_t v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
}  // namespace ar
}  // namespace b200

extern "C" int b200_ar_alloc(size_t bytes, void** ptr) {
  B200_CHECK_ARG(ptr != nullptr && bytes >= 512 && bytes % 256 == 0, "ar_alloc: bad arguments");
  B200_CHECK_CUDA(cudaMalloc(ptr, bytes));
  // data region: every 16-bit lane = the sentinel (negative zero); trailing 256 bytes (epoch, done counter) = 0
  ar::fill_u32_kernel<<<256, 256>>>(static_cast<uint32_t*>(*ptr), (bytes - 256) / 4, ar::kSentinel2);
  B200_CHECK_CUDA(cudaGetLastError());
  B200_CHECK_CUDA(cudaMemset(static_cast<char*>(*ptr) + bytes - 256, 0, 256));
  B200_CHECK_CUDA(cudaDeviceSynchronize());
  return 0;
}

extern "C" int b200_ar_ipc_handle(void* ptr, void* handle64) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  B200_CHECK_CUDA(cudaIpcGetMemHandle(&h, ptr));
  std::memcpy(handle64, &h, 64);
  return 0;
}

extern "C" int b200_ar_ipc_open(const void* handle64, void** ptr) {
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle64, 64);
  B200_CHECK_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}

extern "C" int b200_ar_create(int rank, int world, void* const* bases, const int* opened_mask,
                              size_t max_bytes, void** comm) {
  B200_CHECK_ARG(world >= 1 && world <= ar::kMaxWorld && rank >= 0 && rank < world,
                 "ar_create: bad rank/world %d/%d (world <= %d)", rank, world, ar::kMaxWorld);
  B200_CHECK_ARG(bases != nullptr && comm != nullptr && max_bytes > 0, "ar_create: bad arguments");
  auto* c = new ar::Comm();
  c->rank = rank;
  c->world = world;
  c->slot_bytes = ar::align_up(max_bytes, 256);
  c->flags_off = 2 * (size_t)world * c->slot_bytes;
  c->ctr_off = c->flags_off + ar::align_up((size_t)world * ar::kMaxCtas * 4, 256);
  c->region_bytes = b200_ar_region_bytes(world, max_bytes);
  for (int i = 0; i < ar::kMaxWorld; ++i) {
    c->base[i] = i < world ? static_cast<uint8_t*>(bases[i]) : nullptr;
    c->opened[i] = (i < world && opened_mask != nullptr && opened_mask[i]) ? bases[i] : nullptr;
  }
  *comm = c;
  return 0;
}

extern "C" int b200_ar_destroy(void* comm, int free_local) {
  if (comm == nullptr) return 0;
  auto* c = static_cast<ar::Comm*>(comm);
  for (int i = 0; i < c->world; ++i)
    if (c->opened[i] != nullptr) cudaIpcCloseMemHandle(c->opened[i]);
  if (free_local && c->base[c->rank] != nullptr) cudaFree(c->base[c->rank]);
  delete c;
  return 0;
}

extern "C" size_t b200_ar_max_bytes(const void* comm) {
  return comm == nullptr ? 0 : static_cast<const ar::Comm*>(comm)->slot_bytes;
}

extern "C" int b200_ar_allreduce(void* comm, const void* x, int64_t x_row_stride, void* out,
                                 int64_t out_row_stride, void* residual, int64_t res_row_stride,
                                 const void* weight, int64_t rows, int dim, float eps, int dtype,
                                 void* stream) {
  B200_CHECK_ARG(comm != nullptr, "allreduce: communicator is NULL");
  auto* c = static_cast<ar::Comm*>(comm);
  if (rows == 0) return 0;
  B200_CHECK_ARG(rows > 0 && dim > 0 && dim % 8 == 0, "allreduce: bad rows/dim %lld/%d", (long long)rows, dim);
  B200_CHECK_ARG((size_t)rows * dim * 2 <= c->slot_bytes, "allreduce: message of %lld x %d exceeds the %zu-byte slot",
                 (long long)rows, dim, c->slot_bytes);
  B200_CHECK_ARG((residual == nullptr) == (weight == nullptr), "allreduce: residual and weight go together");
  B200_CHECK_ARG(x_row_stride % 8 == 0 && out_row_stride % 8 == 0 && res_row_stride % 8 == 0 &&
                     ((uintptr_t)x % 16) == 0 && ((uintptr_t)out % 16) == 0 && ((uintptr_t)residual % 16) == 0 &&
                     ((uintptr_t)weight % 16) == 0,
                 "allreduce: pointers / row strides must be 16-byte aligned");
  auto st = (cudaStream_t)stream;
  if (dtype == B200_DTYPE_BF16)
    return ar::launch<__nv_bfloat16>(c, x, x_row_stride, out, out_row_stride, residual, res_row_stride, weight, rows, dim, eps, st);
  if (dtype == B200_DTYPE_FP16)
    return ar::launch<__half>(c, x, x_row_stride, out, out_row_stride, residual, res_row_stride, weight, rows, dim, eps, st);
  set_error("allreduce: bad dtype %d", dtype);
  return 1;
}
