// Device-side replacement of the host loops in the reference's prepare_metadata
// (python/minisgl/attention/fa.py:67-105, fi.py:190-225): one call turns the per-request
// triples (table_idx, cached_len, device_len) into seq_lens / cu_seqlens_q / cu_seqlens_k,
// a token-granular slot-table snapshot (one row per request) and the split-KV decode plan.
// Integer work only -- results must be bit-identical to the reference's host arithmetic.
#include "attn.cuh"

namespace b200 {

constexpr int kOrderBins = 128; // counting-sort bins (tiles per work item, clamped)

// ---- row snapshot: slot_table[r][0:width] = page_table[table_idx_r][0:width]
__global__ void __launch_bounds__(256) meta_rows_kernel(const int32_t* __restrict__ req_info,
                                                        const int32_t* __restrict__ page_table,
                                                        int64_t pt_stride,
                                                        int32_t* __restrict__ slot_table,
                                                        int64_t st_stride, int width, int vec_ok) {
  const int r = blockIdx.x;
  const int64_t row = req_info[3 * r + 0];
  const int32_t* src = page_table + row * pt_stride;
  int32_t* dst = slot_table + (int64_t)r * st_stride;
  if (vec_ok) {
    const int n4 = (width + 3) / 4;
    const int4* s4 = reinterpret_cast<const int4*>(src);
    int4* d4 = reinterpret_cast<int4*>(dst);
    for (int i = threadIdx.x + blockIdx.y * blockDim.x; i < n4; i += blockDim.x * gridDim.y)
      d4[i] = __ldg(s4 + i);
  } else {
    for (int i = threadIdx.x + blockIdx.y * blockDim.x; i < width; i += blockDim.x * gridDim.y)
      dst[i] = __ldg(src + i);
  }
}

// inclusive block scan of one int per thread (blockDim.x == 1024), returns inclusive prefix;
// *total receives the block sum.
__device__ __forceinline__ int block_scan_incl(int v, int* smem /* [33] */, int* total) {
  const int lane = threadIdx.x % kWarp, wid = threadIdx.x / kWarp;
#pragma unroll
  for (int o = 1; o < kWarp; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == kWarp - 1) smem[wid] = v;
  __syncthreads();
  if (wid == 0) {
    int w = smem[lane];
#pragma unroll
    for (int o = 1; o < kWarp; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    smem[lane] = w;
  }
  __syncthreads();
  const int base = wid > 0 ? smem[wid - 1] : 0;
  *total = smem[kWarp - 1];
  __syncthreads();
  return v + base;
}

// ---- scans + decode plan, single CTA of 1024 threads, requests processed in passes of 1024
__global__ void __launch_bounds__(1024) meta_scan_kernel(const int32_t* __restrict__ req_info,
                                                         int bs, int32_t* __restrict__ seq_lens,
                                                         int32_t* __restrict__ cu_q,
                                                         int32_t* __restrict__ cu_k,
                                                         int32_t* __restrict__ plan,
                                                         int target_items, int nosplit) {
  __shared__ int sm[33];
  __shared__ int s_max;
  const int tid = threadIdx.x;
  if (tid == 0) s_max = 0;
  __syncthreads();
  int carry_q = 0, carry_k = 0;
  for (int base = 0; base < bs; base += 1024) {
    const int r = base + tid;
    int ql = 0, kl = 0;
    if (r < bs) {
      const int cached = req_info[3 * r + 1];
      kl = req_info[3 * r + 2];
      ql = kl - cached;
      seq_lens[r] = kl;
      atomicMax(&s_max, kl);
    }
    int tq, tk;
    const int iq = block_scan_incl(ql, sm, &tq);
    const int ik = block_scan_incl(kl, sm, &tk);
    if (r < bs) {
      cu_q[r + 1] = carry_q + iq;
      cu_k[r + 1] = carry_k + ik;
    }
    carry_q += tq;
    carry_k += tk;
  }
  if (tid == 0) {
    cu_q[0] = 0;
    cu_k[0] = 0;
  }
  __syncthreads();
  if (plan == nullptr) return;
  // chunk size: aim at `target_items` (request, chunk) items, whole tiles of 128 tokens,
  // never more than kMaxSplits chunks per request.
  const int total_kv = carry_k;
  const int max_kv = s_max;
  int chunk = (total_kv + target_items - 1) / target_items;
  // With enough whole requests to fill the persistent grid splitting buys nothing: the size-sorted
  // snake order balances them, and unsplit requests need no partial (o, m, l) round trip and no
  // combine work (the host decides from bs alone, so the launcher can drop the combine launch).
  if (nosplit) chunk = max_kv;
  const int min_chunk = (max_kv + kMaxSplits - 1) / kMaxSplits;
  if (chunk < min_chunk) chunk = min_chunk;
  chunk = ((chunk + 127) / 128) * 128;  // whole 128-token tiles
  if (chunk < 128) chunk = 128;
  int carry_c = 0;
  for (int base = 0; base < bs; base += 1024) {
    const int r = base + tid;
    int nc = 0;
    if (r < bs) nc = (req_info[3 * r + 2] + chunk - 1) / chunk;
    int tc;
    const int ic = block_scan_incl(nc, sm, &tc);
    if (r < bs) plan[kPlanHeader + r + 1] = carry_c + ic;
    carry_c += tc;
  }
  if (tid == 0) {
    plan[0] = chunk;
    plan[1] = carry_c;
    plan[2] = bs;
    plan[3] = 0;
    plan[kPlanHeader] = 0;
  }
  // ---- work order: (request, chunk) items sorted by size, largest first (counting sort on the
  // number of 128-token tiles).  The decode kernel deals them to its persistent CTAs in snake
  // order, which balances the per-CTA work to within about one tile.
  __shared__ int hist[kOrderBins];
  for (int i = tid; i < kOrderBins; i += 1024) hist[i] = 0;
  __syncthreads();
  int32_t* order = plan + kPlanHeader + bs + 1;
  auto tiles_of = [&](int kl, int nc, int c) {
    int len = min(chunk, kl - c * chunk);
    if (c == nc - 1) len -= 1;  // the appended token is not part of the tiled range
    int t = (len + 127) / 128;
    return t < kOrderBins - 1 ? t : kOrderBins - 1;
  };
  for (int r = tid; r < bs; r += 1024) {
    const int kl = req_info[3 * r + 2];
    const int nc = (kl + chunk - 1) / chunk;
    for (int c = 0; c < nc; ++c) atomicAdd(&hist[tiles_of(kl, nc, c)], 1);
  }
  __syncthreads();
  if (tid == 0) {  // descending exclusive prefix: largest items first
    int run = 0;
    for (int b = kOrderBins - 1; b >= 0; --b) {
      const int n = hist[b];
      hist[b] = run;
      run += n;
    }
  }
  __syncthreads();
  for (int r = tid; r < bs; r += 1024) {
    const int kl = req_info[3 * r + 2];
    const int nc = (kl + chunk - 1) / chunk;
    for (int c = 0; c < nc; ++c) {
      const int pos = atomicAdd(&hist[tiles_of(kl, nc, c)], 1);
      order[pos] = pack_plan_entry(r, c, nc);
    }
  }
}

// ---- prefill plan: (request, 128-row q tile) items, heaviest (most KV tiles under the causal mask)
// first; the prefill kernel deals them to its persistent CTAs in snake order.
constexpr int kPrefillBins = 1024;
__global__ void __launch_bounds__(1024) meta_prefill_plan_kernel(const int32_t* __restrict__ req_info,
                                                                 int bs, int32_t* __restrict__ plan,
                                                                 int capacity, int request_major) {
  __shared__ int hist[kPrefillBins];
  __shared__ int s_total;
  __shared__ int sm[33];
  const int tid = threadIdx.x;
  if (request_major) {
    // request-major order (query tiles of a request adjacent, heaviest first): the units that share
    // a request's K/V run at the same time on neighbouring CTAs, so the re-reads hit in L2
    int carry = 0;
    for (int base = 0; base < bs; base += 1024) {
      const int r = base + tid;
      int nq = 0;
      if (r < bs) nq = (req_info[3 * r + 2] - req_info[3 * r + 1] + 127) / 128;
      int tot;
      const int incl = block_scan_incl(nq, sm, &tot);
      const int start = carry + incl - nq;
      if (r < bs && carry + tot <= capacity)
        for (int qt = 0; qt < nq; ++qt) plan[4 + start + (nq - 1 - qt)] = pack_prefill_item(r, qt);
      carry += tot;
    }
    if (tid == 0) {
      plan[0] = carry <= capacity ? carry : -1;
      plan[1] = plan[2] = plan[3] = 0;
    }
    return;
  }
  for (int i = tid; i < kPrefillBins; i += 1024) hist[i] = 0;
  if (tid == 0) s_total = 0;
  __syncthreads();
  auto work_of = [&](int cached, int kl, int qt) {
    const int ql = kl - cached;
    const int kv_hi = min(kl, cached + min(ql, (qt + 1) * 128));
    const int t = (kv_hi + 127) / 128;
    return t < kPrefillBins - 1 ? t : kPrefillBins - 1;
  };
  for (int r = tid; r < bs; r += 1024) {
    const int cached = req_info[3 * r + 1], kl = req_info[3 * r + 2];
    const int nq = (kl - cached + 127) / 128;
    for (int qt = 0; qt < nq; ++qt) atomicAdd(&hist[work_of(cached, kl, qt)], 1);
    atomicAdd(&s_total, nq);
  }
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int b = kPrefillBins - 1; b >= 0; --b) {
      const int n = hist[b];
      hist[b] = run;
      run += n;
    }
    plan[0] = s_total <= capacity ? s_total : -1;  // -1: the caller's buffer is too small
    plan[1] = plan[2] = plan[3] = 0;
  }
  __syncthreads();
  if (s_total > capacity) return;
  for (int r = tid; r < bs; r += 1024) {
    const int cached = req_info[3 * r + 1], kl = req_info[3 * r + 2];
    const int nq = (kl - cached + 127) / 128;
    for (int qt = 0; qt < nq; ++qt) {
      const int pos = atomicAdd(&hist[work_of(cached, kl, qt)], 1);
      plan[4 + pos] = pack_prefill_item(r, qt);
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_build_prefill_plan(const int32_t* req_info, int bs, int32_t* prefill_plan,
                                       int capacity_items, void* stream) {
  B200_CHECK_ARG(bs > 0 && bs < 65536, "build_prefill_plan: batch size %d out of range", bs);
  B200_CHECK_ARG(capacity_items > 0 && prefill_plan != nullptr, "build_prefill_plan: no buffer");
  meta_prefill_plan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(req_info, bs, prefill_plan,
                                                                  capacity_items, g_prefill_order.load());
  B200_POST_LAUNCH();
  return 0;
}

extern "C" size_t b200_decode_plan_ints(int bs) {
  return (size_t)kPlanHeader + (size_t)bs + 1 + (size_t)kMaxSplits * bs;
}

namespace b200 {
// the one place that decides "this batch is not split" -- shared with the decode launcher
bool decode_plan_is_unsplit(int bs, int num_kv_heads, int ctas) {
  const int pct = g_decode_plan_nosplit.load();
  return pct > 0 && (int64_t)bs * num_kv_heads * 100 >= (int64_t)pct * ctas;
}
}  // namespace b200

extern "C" int b200_build_metadata(const int32_t* req_info, int bs, const int32_t* page_table,
                                   int64_t page_table_stride, int32_t* seq_lens,
                                   int32_t* cu_seqlens_q, int32_t* cu_seqlens_k,
                                   int32_t* slot_table, int64_t slot_table_stride, int width,
                                   int32_t* decode_plan, int num_kv_heads, int num_ctas_hint,
                                   void* stream) {
  B200_CHECK_ARG(bs > 0 && bs < 65536, "build_metadata: batch size %d out of range [1, 65535]", bs);
  B200_CHECK_ARG(width >= 0 && width <= page_table_stride && width <= slot_table_stride,
                 "build_metadata: width %d exceeds a table stride (%lld / %lld)", width,
                 (long long)page_table_stride, (long long)slot_table_stride);
  B200_CHECK_ARG(num_kv_heads >= 1, "build_metadata: num_kv_heads must be >= 1");
  auto st = (cudaStream_t)stream;
  if (slot_table != nullptr && width > 0) {
    const int w4 = ((width + 3) / 4) * 4;
    const int vec_ok = (page_table_stride % 4 == 0) && (slot_table_stride % 4 == 0) &&
                       (w4 <= page_table_stride) && (w4 <= slot_table_stride) &&
                       ((uintptr_t)page_table % 16 == 0) && ((uintptr_t)slot_table % 16 == 0);
    const int per_row = ceil_div(ceil_div(width, 4), 256);
    dim3 grid(bs, per_row > 4 ? 4 : (per_row < 1 ? 1 : per_row));
    meta_rows_kernel<<<grid, 256, 0, st>>>(req_info, page_table, page_table_stride, slot_table,
                                           slot_table_stride, width, vec_ok);
    B200_POST_LAUNCH();
  }
  const int ctas = num_ctas_hint > 0 ? num_ctas_hint : 2 * num_sms();
  // (request, chunk) items to aim at when splitting: g_decode_plan_target x CTA-hint / kv heads for the full
  // model (8 kv heads per rank); TP shards (<= 4 kv heads per rank: every unit is short) get half as many,
  // larger chunks
  int tgt = g_decode_plan_target.load();
  if (num_kv_heads <= 4 && tgt > 1) tgt /= 2;
  int target = (ctas * tgt) / num_kv_heads;
  if (target < 1) target = 1;
  meta_scan_kernel<<<1, 1024, 0, st>>>(req_info, bs, seq_lens, cu_seqlens_q, cu_seqlens_k,
                                       decode_plan, target, decode_plan_is_unsplit(bs, num_kv_heads, ctas) ? 1 : 0);
  B200_POST_LAUNCH();
  return 0;
}
