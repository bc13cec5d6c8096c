// cp.async / CUDA-core decode kernel: the cross-check of the wgmma product kernel (attn_decode_tc.cu), compiled
// into B200_BUILD_BRINGUP=1 builds only and selected with b200_set_option("decode_impl", 0).
//
// Batched single-token decode over per-request slot tables with the KV append fused into the
// same launch (replaces store_kv + BatchDecodeWithPagedKVCacheWrapper.run of the reference,
// python/minisgl/attention/fi.py:185-188), plus the split-KV combine.
//
// Shape of the work: HBM-bound.  Algorithmic bytes per launch =
//   sum_r kv_len_r * 2*Hkv*D*2  (K and V rows, once per KV head; GQA group shares them)
//   + bs * 2*Hkv*D*2 (append) + bs * 2*Hq*D*2 (q, o).
// Design: persistent grid (2 CTAs per SM), work unit = (request, chunk of the KV range,
// kv head) taken from the device-side plan (metadata.cu); K/V rows are gathered with 16-byte
// cp.async into a 3-stage XOR-swizzled shared-memory ring (96 KB in flight per CTA); scores are
// computed thread-per-key, PV thread-per-dim, online softmax with warp shuffles; partial
// (o, m, l) per chunk go to the workspace and are merged by the combine kernel.
// The new token's K/V row is never read back from the pool in the same launch: the unit that
// owns position kv_len-1 copies k/v into the pool (the append) and sources that row straight
// from the k/v inputs.
#ifdef B200_BRINGUP_KERNELS
#include "attn.cuh"
#include "combine.cuh"

namespace b200 {

constexpr int kD = kHeadDim;
constexpr int kTile = 64;        // kv tokens per pipeline stage
constexpr int kStages = 3;
constexpr int kThreads = 128;
constexpr int kRowBytes = kD * 2;  // 256 B per (token, head) row
constexpr int kSlotRing = 4;       // slot-id prefetch ring (tiles)
constexpr int kMaxBsSmem = 512;    // chunk_start / seq_lens are staged in smem up to this batch size

template <typename T>
struct DecodeParams {
  const T* q;
  int64_t q_rs;
  const T* k_new;
  int64_t k_rs;
  const T* v_new;
  int64_t v_rs;
  T* k_cache;
  T* v_cache;
  const int32_t* out_loc;
  const int32_t* slot_table;
  int64_t st_stride;
  const int32_t* seq_lens;
  const int32_t* plan;
  int bs, hq, hkv;
  float scale_log2;
  T* out;
  float* part_o;   // [bs][kMaxSplits][hq][kD]
  float* part_ml;  // [bs][kMaxSplits][hq][2]
};

template <typename T, int G>
__global__ void __launch_bounds__(kThreads, 2) attn_decode_kernel(const DecodeParams<T> p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sK = smem;                                   // kStages * kTile * 256
  uint8_t* sV = smem + kStages * kTile * kRowBytes;     // kStages * kTile * 256
  float* sQ = reinterpret_cast<float*>(sV + kStages * kTile * kRowBytes);  // [G][kD]
  float* sS = sQ + G * kD;                              // [2][G][kTile] partial scores
  float* sP = sS + 2 * G * kTile;                       // [G][kTile]
  float* sAlpha = sP + G * kTile;                       // [G]
  float* sL = sAlpha + 8;                               // [G]
  float* sM = sL + 8;                                   // [G]
  int32_t* sSlot = reinterpret_cast<int32_t*>(sM + 8);  // [kSlotRing][kTile]
  int32_t* sChunk = sSlot + kSlotRing * kTile;          // [kMaxBsSmem + 1]
  int32_t* sSeq = sChunk + kMaxBsSmem + 1;              // [kMaxBsSmem]

  const int tid = threadIdx.x;
  const int lane = tid % kWarp, warp = tid / kWarp;
  const int chunk_tokens = p.plan[0];
  const int total_units = p.plan[1] * p.hkv;
  const int32_t* chunk_start_g = p.plan + kPlanHeader;
  const uint32_t sK_u = smem_u32(sK), sV_u = smem_u32(sV), sSlot_u = smem_u32(sSlot);
  // per-request tables are read many times per CTA with dependent loads: stage them once
  const bool staged = p.bs <= kMaxBsSmem;
  if (staged) {
    for (int i = tid; i <= p.bs; i += kThreads) sChunk[i] = chunk_start_g[i];
    for (int i = tid; i < p.bs; i += kThreads) sSeq[i] = p.seq_lens[i];
  }
  __syncthreads();
  const int32_t* chunk_start = staged ? sChunk : chunk_start_g;
  const int32_t* seq_lens = staged ? sSeq : p.seq_lens;

  for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
    const int cg = unit / p.hkv;
    const int h = unit % p.hkv;
    // request owning global chunk cg: largest r with chunk_start[r] <= cg
    int lo = 0, hi = p.bs;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (chunk_start[mid] <= cg) lo = mid; else hi = mid;
    }
    const int r = lo;
    const int c = cg - chunk_start[r];
    const int n_chunks = chunk_start[r + 1] - chunk_start[r];
    const int kv_len = seq_lens[r];
    const int kv_begin = c * chunk_tokens;
    const int kv_end = min(kv_len, kv_begin + chunk_tokens);
    const int n_tiles = (kv_end - kv_begin + kTile - 1) / kTile;
    const int32_t* slots = p.slot_table + (int64_t)r * p.st_stride;
    const T* k_new_row = p.k_new + (int64_t)r * p.k_rs + h * kD;
    const T* v_new_row = p.v_new + (int64_t)r * p.v_rs + h * kD;
    const int64_t head_off = (int64_t)h * kD;
    const int64_t slot_stride = (int64_t)p.hkv * kD;

    // ---- fused KV append: the unit holding the newest position writes the pool row
    if (c == n_chunks - 1 && tid < 32) {
      const int64_t dst_slot = p.out_loc[r];
      const int cc = tid & 15;
      if (tid < 16) {
        Vec8 x = *reinterpret_cast<const Vec8*>(k_new_row + cc * 8);
        *reinterpret_cast<Vec8*>(p.k_cache + dst_slot * slot_stride + head_off + cc * 8) = x;
      } else {
        Vec8 x = *reinterpret_cast<const Vec8*>(v_new_row + cc * 8);
        *reinterpret_cast<Vec8*>(p.v_cache + dst_slot * slot_stride + head_off + cc * 8) = x;
      }
    }

    // ---- q (G heads of this kv head) -> smem fp32, pre-scaled by scale*log2(e)
    for (int i = tid; i < G * kD; i += kThreads) {
      const int g = i / kD, d = i % kD;
      sQ[i] = DTypeTraits<T>::to_float(p.q[(int64_t)r * p.q_rs + (int64_t)(h * G + g) * kD + d]) *
              p.scale_log2;
    }
    if (tid < G) {
      sM[tid] = -INFINITY;
      sL[tid] = 0.f;
    }

    // slot ids of tile t -> ring entry t % kSlotRing, asynchronously (joins the next commit group)
    auto fetch_slots = [&](int t) {
      if (t < n_tiles && tid < kTile) {
        const int pos = kv_begin + t * kTile + tid;
        if (pos < kv_end)
          asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(
                           sSlot_u + (uint32_t)(((t % kSlotRing) * kTile + tid) * 4)),
                       "l"(slots + pos)
                       : "memory");
      }
    };
    // K/V rows of tile t (slot ids must already be visible in the ring) + slot ids of tile t+2
    auto issue_tile = [&](int t) {
      if (t < n_tiles) {
        const int stage = t % kStages;
        const int tile_begin = kv_begin + t * kTile;
        const int32_t* ring = sSlot + (t % kSlotRing) * kTile;
#pragma unroll
        for (int i = 0; i < (kTile * 16) / kThreads; ++i) {
          const int idx = tid + i * kThreads;
          const int row = idx >> 4, cc = idx & 15;
          const int pos = tile_begin + row;
          const bool valid = pos < kv_end;
          const T* ksrc = p.k_cache;
          const T* vsrc = p.v_cache;
          if (valid) {
            if (pos == kv_len - 1) {  // the token appended by this very launch
              ksrc = k_new_row + cc * 8;
              vsrc = v_new_row + cc * 8;
            } else {
              const int64_t off = (int64_t)ring[row] * slot_stride + head_off + cc * 8;
              ksrc = p.k_cache + off;
              vsrc = p.v_cache + off;
            }
          }
          const uint32_t o = stage * (kTile * kRowBytes) + swz(row, cc);
          cp_async16_zfill(sK_u + o, ksrc, valid);
          cp_async16_zfill(sV_u + o, vsrc, valid);
        }
      }
      fetch_slots(t + 2);
      cp_async_commit();
    };

    fetch_slots(0);
    fetch_slots(1);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
#pragma unroll
    for (int t = 0; t < kStages - 1; ++t) issue_tile(t);

    float acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = 0.f;

    for (int t = 0; t < n_tiles; ++t) {
      cp_async_wait<kStages - 2>();
      __syncthreads();  // tile t visible to all; everyone is done with tile t-1's stage
      issue_tile(t + kStages - 1);
      const int stage = t % kStages;
      const uint8_t* kt = sK + stage * (kTile * kRowBytes);
      const uint8_t* vt = sV + stage * (kTile * kRowBytes);
      const int tile_begin = kv_begin + t * kTile;

      // ---- scores: thread = (key, half of D)
      {
        const int key = tid & (kTile - 1);
        const int half = tid / kTile;
        float part[G];
#pragma unroll
        for (int g = 0; g < G; ++g) part[g] = 0.f;
#pragma unroll
        for (int cc = 0; cc < 8; ++cc) {
          const int cidx = half * 8 + cc;
          const Vec8 kv = *reinterpret_cast<const Vec8*>(kt + swz(key, cidx));
          float kf[8];
          unpack8<T>(kv, kf);
#pragma unroll
          for (int g = 0; g < G; ++g) {
            const float4 q0 = *reinterpret_cast<const float4*>(sQ + g * kD + cidx * 8);
            const float4 q1 = *reinterpret_cast<const float4*>(sQ + g * kD + cidx * 8 + 4);
            part[g] += kf[0] * q0.x + kf[1] * q0.y + kf[2] * q0.z + kf[3] * q0.w + kf[4] * q1.x +
                       kf[5] * q1.y + kf[6] * q1.z + kf[7] * q1.w;
          }
        }
#pragma unroll
        for (int g = 0; g < G; ++g) sS[(half * G + g) * kTile + key] = part[g];
      }
      __syncthreads();

      // ---- online softmax: warp w owns heads w, w+4 ; lane owns keys lane, lane+32
      for (int g = warp; g < G; g += kThreads / kWarp) {
        const int k0 = lane, k1 = lane + 32;
        float s0 = sS[g * kTile + k0] + sS[(G + g) * kTile + k0];
        float s1 = sS[g * kTile + k1] + sS[(G + g) * kTile + k1];
        if (tile_begin + k0 >= kv_end) s0 = -INFINITY;
        if (tile_begin + k1 >= kv_end) s1 = -INFINITY;
        const float m_old = sM[g];
        const float m_new = fmaxf(m_old, warp_max(fmaxf(s0, s1)));
        const float p0 = fast_exp2(s0 - m_new), p1 = fast_exp2(s1 - m_new);
        const float alpha = fast_exp2(m_old - m_new);
        const float psum = warp_sum(p0 + p1);
        sP[g * kTile + k0] = p0;
        sP[g * kTile + k1] = p1;
        __syncwarp();
        if (lane == 0) {
          sM[g] = m_new;
          sL[g] = sL[g] * alpha + psum;
          sAlpha[g] = alpha;
        }
      }
      __syncthreads();

      // ---- PV: thread = output dim d
      {
        const int d = tid;
        const int cidx = d >> 3, e = d & 7;
#pragma unroll
        for (int g = 0; g < G; ++g) acc[g] *= sAlpha[g];
#pragma unroll 4
        for (int j = 0; j < kTile; j += 4) {
          float vf[4];
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
            vf[jj] = DTypeTraits<T>::to_float(
                *reinterpret_cast<const T*>(vt + swz(j + jj, cidx) + e * 2));
#pragma unroll
          for (int g = 0; g < G; ++g) {
            const float4 pp = *reinterpret_cast<const float4*>(sP + g * kTile + j);
            acc[g] += pp.x * vf[0] + pp.y * vf[1] + pp.z * vf[2] + pp.w * vf[3];
          }
        }
      }
    }
    __syncthreads();  // sM/sL final; all smem reads of this unit done

    // ---- epilogue
    if (n_chunks == 1) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float inv = 1.f / sL[g];
        p.out[((int64_t)r * p.hq + h * G + g) * kD + tid] =
            DTypeTraits<T>::from_float(acc[g] * inv);
      }
    } else {
      const int64_t base = ((int64_t)r * kMaxSplits + c) * p.hq + h * G;
#pragma unroll
      for (int g = 0; g < G; ++g) p.part_o[(base + g) * kD + tid] = acc[g];
      if (tid < G) {
        p.part_ml[(base + tid) * 2 + 0] = sM[tid];
        p.part_ml[(base + tid) * 2 + 1] = sL[tid];
      }
    }
    __syncthreads();  // before the next unit overwrites sQ / sM / sL / stages
  }
}

template <typename T, int G>
static int launch_decode_g(const DecodeParams<T>& p, cudaStream_t st) {
  const size_t smem = 2 * kStages * kTile * kRowBytes +
                      sizeof(float) * (G * kD + 2 * G * kTile + G * kTile + 24) +
                      sizeof(int32_t) * (kSlotRing * kTile + 2 * kMaxBsSmem + 1);
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(attn_decode_kernel<T, G>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  const int grid = 2 * num_sms();
  attn_decode_kernel<T, G><<<grid, kThreads, smem, st>>>(p);
  B200_POST_LAUNCH();
  attn_combine_kernel<T><<<dim3(p.bs, p.hq), kHeadDim, 0, st>>>(p.part_o, p.part_ml, p.plan, p.hq, p.out);
  B200_POST_LAUNCH();
  return 0;
}

template <typename T>
static int launch_decode(const DecodeArgs& a) {
  const DecodeWorkspace ws = carve_decode_workspace(a.workspace, a.workspace_bytes, a.bs, a.hq);
  const DecodeParams<T> p{(const T*)a.q, a.q_rs, (const T*)a.k, a.k_rs, (const T*)a.v, a.v_rs, (T*)a.k_cache,
                          (T*)a.v_cache, a.out_loc, a.slot_table, a.st_stride, a.seq_lens, a.plan, a.bs, a.hq,
                          a.hkv, a.scale * kLog2e, (T*)a.out, ws.part_o, ws.part_ml};
  switch (a.hq / a.hkv) {
    case 1: return launch_decode_g<T, 1>(p, a.stream);
    case 2: return launch_decode_g<T, 2>(p, a.stream);
    case 3: return launch_decode_g<T, 3>(p, a.stream);
    case 4: return launch_decode_g<T, 4>(p, a.stream);
    case 5: return launch_decode_g<T, 5>(p, a.stream);
    case 6: return launch_decode_g<T, 6>(p, a.stream);
    case 7: return launch_decode_g<T, 7>(p, a.stream);
    case 8: return launch_decode_g<T, 8>(p, a.stream);
    default:
      set_error("attn_decode: GQA group size %d not supported (1..8)", a.hq / a.hkv);
      return 1;
  }
}

int launch_decode_bringup(const DecodeArgs& a) {
  return a.dtype == B200_DTYPE_BF16 ? launch_decode<__nv_bfloat16>(a) : launch_decode<__half>(a);
}

}  // namespace b200
#endif  // B200_BRINGUP_KERNELS
