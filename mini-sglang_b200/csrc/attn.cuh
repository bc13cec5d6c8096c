// The attention contract: what metadata.cu, the decode / prefill kernels and their entry points must agree on
// (head dim, plan formats, decode workspace layout, TMA boxes over the KV pool), the arguments an entry
// point hands to a launcher, and the device skeleton the two wgmma kernels share.
#pragma once
#include <cuda.h>

#include "b200attn.h"
#include "common.cuh"
#include "sm90.cuh"

namespace b200 {

constexpr int kHeadDim = 128;

// ------------------------------------------------------------------------------- decode plan
// decode_plan = {chunk_tokens, total_chunks, bs, 0, chunk_start[bs + 1], order[total_chunks]}
constexpr int kPlanHeader = 4;
constexpr int kMaxSplits = 16;  // chunks per request: metadata.cu never exceeds it, the workspace is sized by it

// order[] entry: r | chunk << 16 | n_chunks << 20   (r < 65536, chunk < 16, n_chunks <= 16)
struct PlanEntry {
  int r, c, n_chunks;
};
__host__ __device__ __forceinline__ int32_t pack_plan_entry(int r, int c, int n_chunks) {
  return r | (c << 16) | (n_chunks << 20);
}
__host__ __device__ __forceinline__ PlanEntry unpack_plan_entry(int32_t e) {
  return {e & 0xffff, (e >> 16) & 0xf, (e >> 20) & 0x1f};
}

// prefill_plan = {n_items, 0, 0, 0, item[n_items]},  item = r | q_tile << 16
__host__ __device__ __forceinline__ int32_t pack_prefill_item(int r, int q_tile) { return r | (q_tile << 16); }
__host__ __device__ __forceinline__ int prefill_item_request(int32_t e) { return e & 0xffff; }
__host__ __device__ __forceinline__ int prefill_item_q_tile(int32_t e) { return (e >> 16) & 0xffff; }

bool decode_plan_is_unsplit(int bs, int num_kv_heads, int ctas);  // metadata.cu: the plan policy's split decision

// -------------------------------------------------------------------------- decode workspace
// partial o [bs][kMaxSplits][hq][128] | partial (m, l) [bs][kMaxSplits][hq][2] (fp32), the two rounded up to
// 256 B together, then the split-KV arrival counters [bs][hq] (zero between launches) at the END of the
// workspace: their place does not depend on bs and they can never overlap the last partials.
inline size_t decode_workspace_bytes(int max_bs, int hq, int head_dim) {
  const size_t items = (size_t)max_bs * kMaxSplits * hq;
  const size_t partials = items * head_dim * sizeof(float) + items * 2 * sizeof(float);
  const size_t counters = (size_t)max_bs * hq * sizeof(int);
  return (partials + 255) / 256 * 256 + (counters + 255) / 256 * 256 + 256;
}

struct DecodeWorkspace {
  float* part_o;
  float* part_ml;
  int* counters;
};
inline DecodeWorkspace carve_decode_workspace(void* workspace, size_t workspace_bytes, int bs, int hq) {
  const size_t items = (size_t)bs * kMaxSplits * hq;
  float* part_o = reinterpret_cast<float*>(workspace);
  const size_t cnt_bytes = ((size_t)bs * hq * sizeof(int) + 255) / 256 * 256;
  char* end = static_cast<char*>(workspace) + workspace_bytes / 256 * 256;
  return {part_o, part_o + items * kHeadDim, reinterpret_cast<int*>(end - cnt_bytes)};
}

// ------------------------------------------------------------------------ TMA over the KV pool
// Rows per tiled TMA box: the largest power of two <= min(page_size, 64) that divides page_size, if that is at
// least 8 (the slots of a page are consecutive pool rows); 0 = row mode, the pool rows are gathered with cp.async.
inline int box_rows_for(int page_size) {
  if (page_size < 8) return 0;
  int rows = 64;
  while (rows > 8 && page_size % rows != 0) rows >>= 1;
  return page_size % rows == 0 ? rows : 0;
}

// Cached tensor map of a 2-D 16-bit [rows, cols] tensor with {box_cols, box_rows} boxes (tma_host.cu).
int get_tensor_map_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t row_stride_bytes, uint32_t box_cols, uint32_t box_rows, bool is_bf16);

// Maps of one layer's K and V pool, [num_slots, hkv * 128] contiguous rows, in boxes of 64 columns x box_rows.
inline int kv_pool_maps(CUtensorMap* mk, CUtensorMap* mv, const void* k_cache, const void* v_cache,
                        int64_t num_slots, int hkv, uint32_t box_rows, bool bf16) {
  const uint64_t cols = (uint64_t)hkv * kHeadDim;
  if (int rc = get_tensor_map_2d(mk, k_cache, num_slots, cols, cols * 2, 64, box_rows, bf16)) return rc;
  return get_tensor_map_2d(mv, v_cache, num_slots, cols, cols * 2, 64, box_rows, bf16);
}

// ------------------------------------------------------------------------- launcher arguments
// The arguments of b200_attn_decode / b200_attn_decode_fused / b200_attn_prefill in their C ABI order
// (include/b200attn.h), as the phase's entry point has checked them.
struct DecodeArgs {
  const void *q; int64_t q_rs; const void* k; int64_t k_rs; const void* v; int64_t v_rs;
  void *k_cache, *v_cache; int64_t num_slots; int page_size;
  const int32_t *out_loc, *slot_table; int64_t st_stride; const int32_t *seq_lens, *plan;
  int bs, hq, hkv, head_dim; float scale; void* out; void* workspace; size_t workspace_bytes; int dtype;
  cudaStream_t stream;
  // b200_attn_decode_fused: q / k are the raw projection rows, normed (weights may be NULL) and roped in the kernel
  int fuse = 0; const void *qw = nullptr, *kw = nullptr; float eps = 0.f;
  const int32_t* positions = nullptr; const float* cos_sin = nullptr;
};

struct PrefillArgs {  // without the workspace, which prefill does not use
  const void *q; int64_t q_rs; const void* k; int64_t k_rs; const void* v; int64_t v_rs;
  void *k_cache, *v_cache; int64_t num_slots; int page_size;
  const int32_t *out_loc, *slot_table; int64_t st_stride; const int32_t *seq_lens, *cu_q, *plan;
  int bs; int64_t nnz; int max_q; int hq, hkv, head_dim; float scale; void* out; int dtype;
  cudaStream_t stream;
};

// Cross-check kernels of B200_BUILD_BRINGUP=1 builds (attn_decode_bringup.cu, attn_prefill_bringup.cu).
int launch_decode_bringup(const DecodeArgs& a);
int launch_prefill_bringup(const PrefillArgs& a);

// Swizzled byte offset of 16-byte chunk c (0..15) of row `row` in a bring-up kernel's [rows][256 B] tile.
__device__ __forceinline__ uint32_t swz(int row, int c) {
  return (uint32_t)(row * (kHeadDim * 2) + (((c & 8) | ((c ^ row) & 7)) << 4));
}

// ------------------------------------------------- device skeleton of the persistent wgmma kernels
// Work dealing: the size-sorted units (metadata.cu) go to the persistent CTAs in snake order, the k-th unit of a
// CTA being position k*grid + (k even ? cta : grid-1-cta), which balances per-CTA work to within about one unit.
// Every role walks the same list: stage() decodes the first kCap units once, with the whole CTA, into smem
// slots; at(k) reads them back, or decodes from global memory past the cap.  get(pos) is the kernel's decode.
template <typename Unit, int kSlotBytes, int kCap, typename GetUnit>
struct UnitList {
  static_assert(sizeof(Unit) <= kSlotBytes, "Unit must fit its smem slot");
  uint8_t* slots;
  GetUnit get;
  int total, n_rounds, grid, cta;
  __device__ __forceinline__ static bool none(const Unit& u) { return u.n_tiles < 0; }  // no unit this round (the last)
  __device__ __forceinline__ Unit decode(int k) const {
    const int pos = k * grid + ((k & 1) ? grid - 1 - cta : cta);
    Unit u;
    u.n_tiles = -1;
    if (pos < total) u = get(pos);
    return u;
  }
  __device__ __forceinline__ void stage(int tid, int n_threads) const {
    for (int k = tid; k < kCap && k < n_rounds; k += n_threads) *reinterpret_cast<Unit*>(slots + k * kSlotBytes) = decode(k);
  }
  __device__ __forceinline__ Unit at(int k) const {
    return k < kCap ? *reinterpret_cast<const Unit*>(slots + k * kSlotBytes) : decode(k);
  }
};
template <typename Unit, int kSlotBytes, int kCap, typename GetUnit>
__device__ __forceinline__ UnitList<Unit, kSlotBytes, kCap, GetUnit> deal_units(uint8_t* slots, int total, GetUnit get) {
  return {slots, get, total, (total + (int)gridDim.x - 1) / (int)gridDim.x, (int)gridDim.x, (int)blockIdx.x};
}

// K/V tile geometry: a K or V tile is 128 keys x 128 dims, two 64-column halves of [128 rows x 128 B], 128B-swizzled.
// In box mode (page_size >= 8) TMA writes it in place, one box of rb consecutive keys of one page per producer lane,
// lane = (box, half).  In row mode the pool keys are gathered with cp.async into the same layout (gather_part).
constexpr int kKvTileRows = 128, kKvHalfBytes = kKvTileRows * 128, kKvTileBytes = 2 * kKvHalfBytes;
struct KvLane {
  int row, half;  // first key of the run within the tile, 64-column half
  __device__ __forceinline__ static KvLane box(int lane, int rb) { return {(lane >> 1) * rb, lane & 1}; }
  __device__ __forceinline__ static int box_lanes(int rb) { return (kKvTileRows / rb) * 2; }  // lanes with a box
  __device__ __forceinline__ uint32_t dst(uint32_t ring, uint32_t stage) const { return ring + stage * kKvTileBytes + half * kKvHalfBytes + row * 128; }
  __device__ __forceinline__ int col(int col0) const { return col0 + half * 64; }
};
// Slots of keys pos0 .. pos0+3 (16-byte aligned); keys at or past `end` map to num_slots, out of range.
__device__ __forceinline__ int4 kv_slot_group(const int32_t* slots, int pos0, int end, int num_slots) {
  if (pos0 + 3 < end) return __ldg(reinterpret_cast<const int4*>(slots + pos0));
  auto slot = [&](int i) { return pos0 + i < end ? __ldg(slots + pos0 + i) : num_slots; };
  return make_int4(slot(0), slot(1), slot(2), slot(3));
}
// Row-mode gather (page_size < 8): keys 64 part + r, r < n, of the K or V stage at `stage` are copied from the pool
// rows `src` + slot * row_elems (the head's 128 columns) with 16-byte cp.async, into the 128B-swizzled layout TMA
// writes.  One warp instruction moves two 256-byte rows, keys r = i (lanes 0-15) and r = 32 + i (lanes 16-31), lane
// & 15 being the 16-byte chunk, so eight lanes cover a 128-byte half row.  `slots` = kv_slot_group of keys 64 part +
// 4 (lane & 15) ..: lane 8 (r / 32) + (r % 32) / 4 holds the slot of key r in component r % 4, one shuffle per
// instruction.  A key whose slot is num_slots (past the end of the range) is zero filled and never read; keys r >= n
// are not written.  Completion is the caller's cp_async_mbar_arrive_noinc.
template <typename T>
__device__ __forceinline__ void gather_part(uint32_t stage, int part, const T* src, int row_elems, int4 slots,
                                            int num_slots, int n, int lane) {
  // Rolled over 8-key atoms (a full unroll costs the producers registers they do not have): key r = r_hi + 8 a + k
  // sits at byte (part 64 + r) 128 of its half, chunk j ^ k (sw128_offset with row & 7 = k).
  const int j = lane & 15, r_hi = (lane >> 4) * 32, lane0 = (lane >> 4) * 8;
  const uint32_t dst0 = stage + (j >> 3) * kKvHalfBytes + (part * 64 + r_hi) * 128;
  const T* src_j = src + j * 8;
#pragma unroll 1
  for (int a = 0; a < 4; ++a) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = (k & 3) == 0 ? slots.x : (k & 3) == 1 ? slots.y : (k & 3) == 2 ? slots.z : slots.w;
      const int s = __shfl_sync(0xffffffffu, c, lane0 + 2 * a + (k >> 2));
      if (r_hi + 8 * a + k < n) {
        const bool in = s < num_slots;
        sm90::cp_async_16(dst0 + a * 1024 + k * 128 + (((j ^ k) & 7) << 4), src_j + (in ? (int64_t)s * row_elems : 0),
                          in ? 16u : 0u);
      }
    }
  }
}

// ------------------------------------------------------------------------------ event trace
// b200_attn_trace_set registers a device buffer; each traced launch gets one region of it (mini-sglang_b200/trace.py
// decodes the same layout):
//   TraceHeader (64 B) | u32 count[grid][warps], rounded up to 16 B | TraceRecord rec[grid][warps][events_per_warp]
// Lane 0 of every warp records the events of its warp with plain stores; past events_per_warp it only counts, and
// writes the count (which then exceeds events_per_warp) when the CTA ends.  Only the kTrace = true instantiations of
// the two wgmma kernels contain any of it.
constexpr uint32_t kTraceMagic = 0x52545441u;  // "ATTR"
constexpr uint32_t kTraceVersion = 1;
constexpr int kTracePhaseDecode = 0, kTracePhasePrefill = 1;
constexpr int kDecodeWarps = 10, kPrefillWarps = 12;
enum TraceFlag : uint32_t { kTraceFused = 1, kTraceInKernelCombine = 2, kTraceEarlyKv = 4 };

// Event codes; arg is %smid, the unit's position k in the CTA's list, or the tile's index within its unit.
enum TraceCode : uint32_t {
  kEvBegin = 1,        // first event of every warp, arg = %smid
  kEvPdlWait = 2,      // past griddepcontrol.wait
  kEvUnitBegin = 3,    // arg = k (every unit of the CTA's list, in every role, also those the role skips)
  kEvUnitEnd = 4,      // arg = k
  kEvEmptyWait = 5,    // producer: waits for a free ring slot, arg = tile
  kEvEmptyDone = 6,    // producer: the slot is free, arg = tile
  kEvIssued = 7,       // producer: the tile's loads are issued, arg = tile
  kEvQIssued = 8,      // prefill K producer: the unit's Q tile load is issued, arg = k
  kEvAppend = 9,       // prefill producers: the append stores of a tile are issued, arg = tile
  kEvQReady = 10,      // decode Q loader: operand (and fused epilogue rows) written; consumer: Q operand landed
  kEvKFull = 11,       // consumer: K tile landed, arg = tile
  kEvQK = 12,          // consumer: S = QK^T complete
  kEvSoftmax = 13,     // consumer: P written / in registers
  kEvVFull = 14,       // consumer: V tile landed
  kEvPV = 15,          // consumer: O += PV complete
  kEvSkip = 16,        // prefill consumer: tile fully masked for the warpgroup, no MMA
  kEvEpiBegin = 17,    // consumer epilogue (decode: new-token score, append, output or partial store), arg = k
  kEvEpiEnd = 18,
  kEvArrive = 19,      // decode combiner: counted in, another chunk merges, arg = k
  kEvArriveLast = 20,  // decode combiner: counted in last, merges, arg = k
  kEvMergeBegin = 21,
  kEvMergeEnd = 22,
  kEvEnd = 31,         // last event of every warp: past the kernel's final __syncthreads
};

struct TraceHeader {
  uint32_t magic, version, phase, grid, threads, warps, bs, hq, hkv, group, page_size, box_rows, events_per_warp,
      plan_kind, seq, flags;
};
static_assert(sizeof(TraceHeader) == 64, "trace header is 64 bytes");
struct TraceRecord {  // 16 bytes, one st.global.v4
  uint64_t globaltimer_ns;
  uint32_t clock;
  uint8_t code, warp;
  uint16_t arg;
};
static_assert(sizeof(TraceRecord) == 16, "trace record is 16 bytes");

__host__ __device__ inline size_t trace_counts_bytes(int grid, int warps) { return ((size_t)grid * warps * 4 + 15) / 16 * 16; }
inline size_t trace_region_bytes(int grid, int warps, int events_per_warp) {
  return sizeof(TraceHeader) + trace_counts_bytes(grid, warps) + (size_t)grid * warps * events_per_warp * sizeof(TraceRecord);
}

// What a traced launch is handed: its region (nullptr = not traced), the record capacity, its sequence number, and
// header fields the kernel does not know.  The header's plan_kind is 1 for a decode plan that splits, else 0.
struct TraceArgs {
  uint8_t* region;
  int events_per_warp, seq, page_size;
  uint32_t flags;
};
// capi.cu: the next region for a launch of `phase` with `grid` CTAs; false (and counted as untraced) when no buffer
// is registered or the regions are used up.
bool trace_next_region(int phase, int grid, TraceArgs* out);

// One warp's event writer, kWarps warps per CTA: WarpTrace<false, .> is empty and compiles to nothing.  The traced
// state is three registers (lane 0's record pointer, nullptr in the other lanes, and the event count); everything
// else is read from the kernel parameters when needed, so the producer warps' small register budget holds it.
template <bool kOn, int kWarps>
struct WarpTrace {
  __device__ __forceinline__ explicit WarpTrace(const TraceArgs&) {}
  __device__ __forceinline__ void ev(uint32_t, int) {}
  __device__ __forceinline__ void begin() {}
  __device__ __forceinline__ void header(int, int, int, int, int, int) {}
  __device__ __forceinline__ void finish() {}
};
template <int kWarps>
struct WarpTrace<true, kWarps> {
  const TraceArgs& t;
  TraceRecord* rec;
  uint32_t n;
  __device__ __forceinline__ static size_t slot() { return (size_t)blockIdx.x * kWarps + threadIdx.x / kWarp; }
  __device__ __forceinline__ explicit WarpTrace(const TraceArgs& args) : t(args), rec(nullptr), n(0) {
    if (threadIdx.x % kWarp == 0)
      rec = reinterpret_cast<TraceRecord*>(t.region + sizeof(TraceHeader) + trace_counts_bytes(gridDim.x, kWarps)) +
            slot() * t.events_per_warp;
  }
  __device__ __forceinline__ void ev(uint32_t code, int arg) {
    if (rec == nullptr) return;
    if (n < (uint32_t)t.events_per_warp) {
      uint64_t ns;
      uint32_t clk;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
      asm volatile("mov.u32 %0, %%clock;" : "=r"(clk));
      const uint32_t tag = code | ((threadIdx.x / kWarp) << 8) | ((uint32_t)arg << 16);
      asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(rec + n), "r"((uint32_t)ns),
                   "r"((uint32_t)(ns >> 32)), "r"(clk), "r"(tag));
    }
    ++n;
  }
  __device__ __forceinline__ void begin() {
    uint32_t sm;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
    ev(kEvBegin, (int)sm);
  }
  // CTA 0, warp 0: the launch's header
  __device__ __forceinline__ void header(int phase, int bs, int hq, int hkv, int box_rows, int plan_kind) {
    if (rec == nullptr || blockIdx.x != 0 || threadIdx.x != 0) return;
    *reinterpret_cast<TraceHeader*>(t.region) =
        TraceHeader{kTraceMagic, kTraceVersion, (uint32_t)phase, gridDim.x, blockDim.x, (uint32_t)kWarps,
                    (uint32_t)bs, (uint32_t)hq, (uint32_t)hkv, (uint32_t)(hq / hkv), (uint32_t)t.page_size,
                    (uint32_t)box_rows, (uint32_t)t.events_per_warp, (uint32_t)plan_kind, (uint32_t)t.seq, t.flags};
  }
  __device__ __forceinline__ void finish() {
    if (rec != nullptr) reinterpret_cast<uint32_t*>(t.region + sizeof(TraceHeader))[slot()] = n;
  }
};

}  // namespace b200
