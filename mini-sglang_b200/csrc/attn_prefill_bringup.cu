// mma.sync prefill kernel: the cross-check of the wgmma product kernel (attn_prefill_tc.cu), compiled into
// B200_BUILD_BRINGUP=1 builds only and selected with b200_set_option("prefill_impl", 0) or a NULL prefill_plan.
//
// Ragged chunked-prefill / extend attention over per-request slot tables
// (replaces store_kv + BatchPrefillWithPagedKVCacheWrapper.run of the reference,
// python/minisgl/attention/fi.py:185-188, causal=True fi.py:164).
//
// Flash-attention tiling with legacy mma.sync tensor-core instructions (m16n8k16, bf16/fp16 in, fp32
// accumulate).  One CTA = (request, q head, 64-row q tile), 4 warps x 16 rows; K/V tiles of 64 tokens
// gathered from the paged pool with 16-byte cp.async into XOR-swizzled, double-buffered shared memory;
// ldmatrix fragment loads; online softmax in registers (row reductions with warp shuffles).
// Compute-bound: exact causal flops per launch = 4*Hq*D*sum_r[q*cached + q(q+1)/2].
// The KV append of the new rows runs as the store kernel in front (same C-ABI call).
#ifdef B200_BRINGUP_KERNELS
#include "attn.cuh"

namespace b200 {

constexpr int kD = kHeadDim;
constexpr int kBM = 64;   // q rows per CTA
constexpr int kBN = 64;   // kv tokens per tile
constexpr int kRowBytes = kD * 2;
constexpr int kThreads = 128;
constexpr int kSlotRing = 4;  // slot-id prefetch ring (tiles)

template <typename T>
struct PrefillParams {
  const T* q;
  int64_t q_rs;
  const T* k_cache;
  const T* v_cache;
  const int32_t* slot_table;
  int64_t st_stride;
  const int32_t* seq_lens;
  const int32_t* cu_q;
  int bs, hq, hkv;
  float scale_log2;
  T* out;
};

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                            uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1,
                                                  uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}

template <typename T>
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                         uint32_t b1);
template <>
__device__ __forceinline__ void mma16816<__nv_bfloat16>(float (&c)[4], const uint32_t (&a)[4],
                                                        uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma16816<__half>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                                 uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  typename DTypeTraits<T>::T2 v = DTypeTraits<T>::from_float2(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <typename T>
__global__ void __launch_bounds__(kThreads, 2) attn_prefill_kernel(const PrefillParams<T> p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sQ = smem;                         // 64 x 256 B (reused as the output staging tile)
  uint8_t* sK = sQ + kBM * kRowBytes;         // 2 stages
  uint8_t* sV = sK + 2 * kBN * kRowBytes;     // 2 stages
  int32_t* sSlot = reinterpret_cast<int32_t*>(sV + 2 * kBN * kRowBytes);  // [kSlotRing][kBN]

  const int r = blockIdx.z;
  const int head = blockIdx.y;
  const int q_begin = p.cu_q[r];
  const int q_len = p.cu_q[r + 1] - q_begin;
  const int q_start = blockIdx.x * kBM;
  if (q_start >= q_len) return;
  const int kv_len = p.seq_lens[r];
  const int cached = kv_len - q_len;  // bottom-right aligned causal mask offset
  const int hk = head / (p.hq / p.hkv);
  const int tid = threadIdx.x, lane = tid % kWarp, warp = tid / kWarp;
  const int32_t* slots = p.slot_table + (int64_t)r * p.st_stride;
  const int64_t slot_stride = (int64_t)p.hkv * kD;
  const uint32_t sQ_u = smem_u32(sQ), sK_u = smem_u32(sK), sV_u = smem_u32(sV);
  const uint32_t sSlot_u = smem_u32(sSlot);

  // keys visible to the last row of this q tile
  const int kv_hi = min(kv_len, cached + min(q_len, q_start + kBM));
  const int n_tiles = (kv_hi + kBN - 1) / kBN;

  // ---- Q tile
#pragma unroll
  for (int i = 0; i < (kBM * 16) / kThreads; ++i) {
    const int idx = tid + i * kThreads;
    const int row = idx >> 4, cc = idx & 15;
    const bool valid = q_start + row < q_len;
    const T* src = valid ? p.q + (int64_t)(q_begin + q_start + row) * p.q_rs + (int64_t)head * kD + cc * 8
                         : p.q;
    cp_async16_zfill(sQ_u + swz(row, cc), src, valid);
  }
  // slot ids of tile t -> ring entry t % kSlotRing (asynchronous; joins the next commit group)
  auto fetch_slots = [&](int t) {
    if (t < n_tiles && tid < kBN) {
      const int pos = t * kBN + tid;
      if (pos < kv_hi)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(
                         sSlot_u + (uint32_t)(((t % kSlotRing) * kBN + tid) * 4)),
                     "l"(slots + pos)
                     : "memory");
    }
  };
  // K/V rows of tile t (its slot ids are already visible in the ring) + slot ids of tile t+2
  auto issue_tile = [&](int t) {
    if (t < n_tiles) {
      const int stage = t & 1;
      const int tile_begin = t * kBN;
      const int32_t* ring = sSlot + (t % kSlotRing) * kBN;
#pragma unroll
      for (int i = 0; i < (kBN * 16) / kThreads; ++i) {
        const int idx = tid + i * kThreads;
        const int row = idx >> 4, cc = idx & 15;
        const int pos = tile_begin + row;
        const bool valid = pos < kv_hi;
        int64_t off = 0;
        if (valid) off = (int64_t)ring[row] * slot_stride + (int64_t)hk * kD + cc * 8;
        const uint32_t o = stage * (kBN * kRowBytes) + swz(row, cc);
        cp_async16_zfill(sK_u + o, p.k_cache + off, valid);
        cp_async16_zfill(sV_u + o, p.v_cache + off, valid);
      }
    }
    fetch_slots(t + 2);
    cp_async_commit();
  };
  fetch_slots(0);
  fetch_slots(1);
  cp_async_commit();  // also carries the Q tile issued above
  cp_async_wait<0>();
  __syncthreads();
  issue_tile(0);

  // ---- Q fragments (persistent): 8 k16-blocks x 4 regs
  uint32_t qf[8][4];
  float o_acc[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o_acc[i][j] = 0.f;
  float m_row[2] = {-INFINITY, -INFINITY};
  float l_row[2] = {0.f, 0.f};
  const int g = lane >> 2, tq = lane & 3;
  const int row0 = q_start + warp * 16 + g;  // q row (within request) of c0/c1; +8 for c2/c3

  for (int t = 0; t < n_tiles; ++t) {
    issue_tile(t + 1);
    cp_async_wait<1>();
    __syncthreads();
    if (t == 0) {
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const int row = warp * 16 + (lane & 15);
        const int cc = 2 * kk + (lane >> 4);
        ldmatrix_x4(sQ_u + swz(row, cc), qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
      }
    }
    const uint32_t kt = sK_u + (t & 1) * (kBN * kRowBytes);
    const uint32_t vt = sV_u + (t & 1) * (kBN * kRowBytes);
    const int tile_begin = t * kBN;

    // ---- S = Q K^T  (16 x 64 per warp)
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int x = 0; x < 4; ++x) s[j][x] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {  // pairs of n-tiles (16 keys)
        const int key = jp * 16 + (lane & 7) + 8 * (lane >> 4);
        const int cc = 2 * kk + ((lane >> 3) & 1);
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4(kt + swz(key, cc), b0, b1, b2, b3);
        mma16816<T>(s[2 * jp], qf[kk], b0, b1);
        mma16816<T>(s[2 * jp + 1], qf[kk], b2, b3);
      }
    }

    // ---- scale, mask, online softmax (rows g and g+8 of this warp's 16)
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        const int key = tile_begin + j * 8 + 2 * tq + (x & 1);
        const int qrow = row0 + (x >> 1) * 8;
        const bool ok = (key <= cached + qrow) && (key < kv_len);
        const float v = ok ? s[j][x] * p.scale_log2 : -INFINITY;
        s[j][x] = v;
        mx[x >> 1] = fmaxf(mx[x >> 1], v);
      }
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      mx[h2] = fmaxf(mx[h2], __shfl_xor_sync(0xffffffffu, mx[h2], 1));
      mx[h2] = fmaxf(mx[h2], __shfl_xor_sync(0xffffffffu, mx[h2], 2));
      const float m_new = fmaxf(m_row[h2], mx[h2]);
      m_use[h2] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[h2] = fast_exp2(m_row[h2] - m_use[h2]);
      m_row[h2] = m_new;
    }
    float ps[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        const float e = fast_exp2(s[j][x] - m_use[x >> 1]);
        s[j][x] = e;
        ps[x >> 1] += e;
      }
    }
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      ps[h2] += __shfl_xor_sync(0xffffffffu, ps[h2], 1);
      ps[h2] += __shfl_xor_sync(0xffffffffu, ps[h2], 2);
      l_row[h2] = l_row[h2] * alpha[h2] + ps[h2];
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      o_acc[i][0] *= alpha[0];
      o_acc[i][1] *= alpha[0];
      o_acc[i][2] *= alpha[1];
      o_acc[i][3] *= alpha[1];
    }

    // ---- O += P V   (k = keys: 4 k16-blocks; n = d: 16 n-tiles)
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
      uint32_t a[4];
      a[0] = pack2<T>(s[2 * kb][0], s[2 * kb][1]);
      a[1] = pack2<T>(s[2 * kb][2], s[2 * kb][3]);
      a[2] = pack2<T>(s[2 * kb + 1][0], s[2 * kb + 1][1]);
      a[3] = pack2<T>(s[2 * kb + 1][2], s[2 * kb + 1][3]);
#pragma unroll
      for (int np = 0; np < 8; ++np) {  // pairs of d n-tiles
        const int key = kb * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
        const int cc = 2 * np + (lane >> 4);
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4_trans(vt + swz(key, cc), b0, b1, b2, b3);
        mma16816<T>(o_acc[2 * np], a, b0, b1);
        mma16816<T>(o_acc[2 * np + 1], a, b2, b3);
      }
    }
    __syncthreads();  // all warps done with stage (t&1) before tile t+2 overwrites it
  }

  // ---- epilogue: normalise, stage through sQ (each warp owns its 16 rows), coalesced stores
  const float inv0 = 1.f / l_row[0], inv1 = 1.f / l_row[1];
#pragma unroll
  for (int nt = 0; nt < 16; ++nt) {
    const int rl0 = warp * 16 + g, rl1 = rl0 + 8;
    const uint32_t v0 = pack2<T>(o_acc[nt][0] * inv0, o_acc[nt][1] * inv0);
    const uint32_t v1 = pack2<T>(o_acc[nt][2] * inv1, o_acc[nt][3] * inv1);
    *reinterpret_cast<uint32_t*>(sQ + swz(rl0, nt) + tq * 4) = v0;
    *reinterpret_cast<uint32_t*>(sQ + swz(rl1, nt) + tq * 4) = v1;
  }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = lane + i * kWarp;  // 16 rows x 16 chunks
    const int rl = warp * 16 + (idx >> 4), cc = idx & 15;
    if (q_start + rl < q_len) {
      const Vec8 v = *reinterpret_cast<const Vec8*>(sQ + swz(rl, cc));
      *reinterpret_cast<Vec8*>(p.out + ((int64_t)(q_begin + q_start + rl) * p.hq + head) * kD +
                               cc * 8) = v;
    }
  }
}

template <typename T>
static int launch_prefill(const PrefillArgs& a) {
  const PrefillParams<T> p{(const T*)a.q, a.q_rs, (const T*)a.k_cache, (const T*)a.v_cache, a.slot_table,
                           a.st_stride, a.seq_lens, a.cu_q, a.bs, a.hq, a.hkv, a.scale * kLog2e, (T*)a.out};
  const size_t smem = (kBM + 4 * kBN) * kRowBytes + kSlotRing * kBN * sizeof(int32_t);  // 81 KB
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(attn_prefill_kernel<T>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  dim3 grid(ceil_div(a.max_q, kBM), p.hq, p.bs);
  attn_prefill_kernel<T><<<grid, kThreads, smem, a.stream>>>(p);
  B200_POST_LAUNCH();
  return 0;
}

int launch_prefill_bringup(const PrefillArgs& a) {
  // append the new rows first (same stream => ordered before the attention kernel reads them)
  const int64_t row_bytes = (int64_t)a.hkv * kD * 2;
  if (int rc = b200_store_kv(a.k_cache, a.v_cache, row_bytes, a.k, a.v, a.k_rs * 2, a.out_loc, 0, a.nnz,
                             row_bytes, a.stream))
    return rc;
  return a.dtype == B200_DTYPE_BF16 ? launch_prefill<__nv_bfloat16>(a) : launch_prefill<__half>(a);
}

}  // namespace b200
#endif  // B200_BRINGUP_KERNELS
