// Hopper-native ragged prefill / extend attention: TMA -> swizzled smem -> wgmma with S, P and O in
// registers (replaces BatchPrefillWithPagedKVCacheWrapper.run, python/minisgl/attention/fi.py:150-165,188;
// causal, bottom-right aligned).
//
// Compute-bound: exact causal flops = 4*Hq*D*sum_r[q*cached + q(q+1)/2].
// Persistent, one CTA per SM, 384 threads = three warpgroups.  A work unit is (request, 128-row query
// tile, query head); the query heads of one kv head are adjacent units, so neighbouring CTAs stream the
// same K/V rows and the re-reads hit in L2.
//
//   warp 0      K producer (+ the unit's Q tile): TMA boxes per page piece / single-row boxes
//   warp 1      V producer
//   (append)    fused KV append: the producers write the tile of a unit that holds the unit's own new
//               tokens to the pool straight from shared memory (TMA store); the attention reads this
//               forward's tokens from the k / v inputs, never back from the pool, so no ordering is needed
//   warps 4-7   consumer warpgroup 0: query rows 0-63 of the tile;  warps 8-11: rows 64-127
//               S = Q . K^T      wgmma m64n128k16, A and B from smem (K-major, 128B swizzle), fp32 registers
//               O += P . V       wgmma m64n128k16, A = P from registers (16-bit), B = V tile read MN-major
//               online softmax on the score fragments: a query row lives in one quad of lanes, so the row
//               max / sum need two shuffles; K/V tiles that are fully masked for all 64 rows are skipped.
// The producer warpgroup hands registers to the consumers (setmaxnreg): 128 x 40 + 256 x 232 = 384 x 168.
#include "b200attn.h"
#include "common.cuh"
#include "sm90.cuh"

#include <type_traits>

namespace b200 {

int get_tensor_map_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t row_stride_bytes, uint32_t box_cols, uint32_t box_rows, bool is_bf16);

namespace ptc {

using namespace sm90;

constexpr int kD = 128;
constexpr int kBM = 128;                   // query rows per unit (two consumer warpgroups x 64)
constexpr int kBN = 128;                   // keys per tile
constexpr int kStages = 2;                 // K ring depth = V ring depth
constexpr int kThreads = 384;
constexpr int kHalfBytes = 128 * 128;      // [128 rows x 64 cols] 16-bit, 128B-swizzled: 16 KB
constexpr int kTileBytes = 2 * kHalfBytes; // 32 KB
constexpr int kMaxUnitsSmem = 64;

struct Smem {
  static constexpr int q = 0;                                // one 128-row Q tile: 32 KB
  static constexpr int kring = kTileBytes;                   // kStages x 32 KB
  static constexpr int vring = kring + kStages * kTileBytes;
  static constexpr int bars = vring + kStages * kTileBytes;  // 10 mbarriers
  static constexpr int units = bars + 16 * 8;
  static constexpr int total = units + kMaxUnitsSmem * 48;
};
static_assert(Smem::total + 1024 <= 232448, "prefill kernel shared memory exceeds the 227 KB per-CTA limit");
enum Bar { kFullK = 0, kEmptyK = 2, kFullV = 4, kEmptyV = 6, kQFull = 8, kQEmpty = 9 };

template <typename T>
struct Params {
  const int32_t* slot_table;
  int64_t st_stride;
  const int32_t* seq_lens;
  const int32_t* cu_q;
  const int32_t* plan;  // {n_items, 0,0,0, item[...]}
  int bs, hq, hkv;
  int num_slots;
  int box_rows;
  float scale_log2;
  T* out;
  // fused KV append (rows of the new tokens -> pool); attention never reads them back from the pool
  const T* k_new;
  const T* v_new;
  int64_t kv_rs;      // row stride of k_new / v_new (elements)
  T* k_cache;
  T* v_cache;
  const int32_t* out_loc;
  int64_t nnz;
  int skip_append;  // debug: measure the attention without the fused append
};

struct Unit {
  int r, q_start, q_len, q_begin, kv_len, cached, kv_hi, n_tiles, h, head, owner;
};
static_assert(sizeof(Unit) <= 48, "Unit must fit its smem slot");

__device__ __forceinline__ Unit get_unit(int pos, int hq, int group, const int32_t* items,
                                         const int32_t* seq_lens, const int32_t* cu_q) {
  Unit u;
  const int item = pos / hq;
  u.head = pos - item * hq;
  u.h = u.head / group;
  u.owner = (u.head == u.h * group);  // the first query head of a kv head appends its rows
  const int e = items[item];
  u.r = e & 0xffff;
  u.q_start = ((e >> 16) & 0xffff) * kBM;
  u.q_begin = cu_q[u.r];
  u.q_len = cu_q[u.r + 1] - u.q_begin;
  u.kv_len = seq_lens[u.r];
  u.cached = u.kv_len - u.q_len;
  u.kv_hi = min(u.kv_len, u.cached + min(u.q_len, u.q_start + kBM));
  u.n_tiles = (u.kv_hi + kBN - 1) / kBN;
  return u;
}

template <typename T>
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  typename DTypeTraits<T>::T2 v = DTypeTraits<T>::from_float2(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <typename T>
__global__ void __launch_bounds__(kThreads, 1)
attn_prefill_tc_kernel(const Params<T> p, const __grid_constant__ CUtensorMap map_q,
                       const __grid_constant__ CUtensorMap map_k,
                       const __grid_constant__ CUtensorMap map_v,
                       const __grid_constant__ CUtensorMap box_k,
                       const __grid_constant__ CUtensorMap box_v,
                       const __grid_constant__ CUtensorMap new_k,    // k input rows, box {64, 1}
                       const __grid_constant__ CUtensorMap new_v,
                       const __grid_constant__ CUtensorMap newbox_k, // k input rows, box {64, box_rows}
                       const __grid_constant__ CUtensorMap newbox_v) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid / kWarp, lane = tid % kWarp;
  auto bar = [&](int i) { return sbase + Smem::bars + i * 8; };
  uint8_t* sUnits = smem + Smem::units;

  const int group = p.hq / p.hkv;
  const int total_units = p.plan[0] * p.hq;
  const int32_t* items = p.plan + 4;
  const int grid = gridDim.x, cta = blockIdx.x;
  const int n_rounds = (total_units + grid - 1) / grid;
  auto pos_of = [&](int k) { return k * grid + ((k & 1) ? grid - 1 - cta : cta); };

  // ---------------------------------------------------------------- one-time setup
  for (int k = tid; k < kMaxUnitsSmem && k < n_rounds; k += kThreads) {
    const int pos = pos_of(k);
    Unit u;
    u.n_tiles = -1;
    if (pos < total_units) u = get_unit(pos, p.hq, group, items, p.seq_lens, p.cu_q);
    *reinterpret_cast<Unit*>(sUnits + k * 48) = u;
  }
  auto unit_at = [&](int k) {
    if (k < kMaxUnitsSmem) return *reinterpret_cast<const Unit*>(sUnits + k * 48);
    const int pos = pos_of(k);
    Unit u;
    u.n_tiles = -1;
    if (pos < total_units) u = get_unit(pos, p.hq, group, items, p.seq_lens, p.cu_q);
    return u;
  };
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(bar(kFullK + s), 1);
      mbar_init(bar(kEmptyK + s), 8);  // one elected arrival per consumer warp
      mbar_init(bar(kFullV + s), 1);
      mbar_init(bar(kEmptyV + s), 8);
    }
    mbar_init(bar(kQFull), 1);
    mbar_init(bar(kQEmpty), 8);
    fence_barrier_init();
    prefetch_tensormap(&map_q);
    prefetch_tensormap(&map_k);
    prefetch_tensormap(&map_v);
    prefetch_tensormap(&box_k);
    prefetch_tensormap(&box_v);
    prefetch_tensormap(&new_k);
    prefetch_tensormap(&new_v);
    prefetch_tensormap(&newbox_k);
    prefetch_tensormap(&newbox_v);
  }
  __syncthreads();

  // Register budget: the producer warpgroup gives registers up, the consumer warpgroups take them.  Each
  // setmaxnreg sits at the top of its own branch so that ptxas allocates per role.  The pool is what the CTA
  // was launched with (384 threads x 168 registers = 64 512): 128 x 40 + 256 x 232 = 64 512.
  if (warp < 4) {
   asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
   if (warp < 2) {
    // ============================================================ TMA producers: warp 0 = K (+Q), warp 1 = V
    const int kind = warp;
    const int rb = p.box_rows;
    const CUtensorMap* gmap = kind == 0 ? &map_k : &map_v;
    const CUtensorMap* bmap = kind == 0 ? &box_k : &box_v;
    const int full0 = kind == 0 ? kFullK : kFullV, empty0 = kind == 0 ? kEmptyK : kEmptyV;
    const uint32_t ring = sbase + (kind == 0 ? Smem::kring : Smem::vring);
    uint32_t tile_count = 0, unit_count = 0;
    // ---- fused KV append: the tile of a unit that holds the unit's own new tokens is written to the
    // pool straight from shared memory (TMA store) when its ring slot is recycled -- no extra loads,
    // no extra launch.  Ownership: positions [cached + q_start, cached + min(q_len, q_start + 128)) of
    // kv head h belong to the unit of query tile q_start and the first query head of the group.
    struct Pending {
      int valid, lo, hi, tile_begin, col0;
      uint32_t phase;
      const int32_t* slots;
    } pend[kStages];
    for (int s = 0; s < kStages; ++s) pend[s].valid = 0;
    const CUtensorMap* smap_box = bmap;   // pool, box_rows x 64 columns
    const CUtensorMap* smap_row = gmap;   // pool, 1 x 64 columns (row-exact)
    // valid: 0 = nothing, 1 = tile issued (append once it has landed), 2 = stores issued
    auto issue_stores = [&](int stage) {  // whole warp; the tile has landed
      Pending& pd = pend[stage];
      const uint32_t base = ring + stage * kTileBytes;
      if (rb > 0) {
        const int n_instr = (kBN / rb) * 2;
        if (lane < n_instr) {
          const int box = lane >> 1, half = lane & 1;
          const int pb = pd.tile_begin + box * rb;
          const uint32_t src = base + half * kHalfBytes + box * rb * 128;
          const int col = pd.col0 + half * 64;
          if (pb >= pd.lo && pb + rb <= pd.hi) {
            tma_store_2d(smap_box, src, col, __ldg(pd.slots + pb));
          } else {
            for (int i = 0; i < rb; ++i)
              if (pb + i >= pd.lo && pb + i < pd.hi) tma_store_2d(smap_row, src + i * 128, col, __ldg(pd.slots + pb + i));
          }
        }
      } else {
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          const int grp = (lane >> 1) + it * 16, half = lane & 1;
          const int pos0 = pd.tile_begin + grp * 4;
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (pos0 + i >= pd.lo && pos0 + i < pd.hi)
              tma_store_2d(smap_row, base + half * kHalfBytes + (grp * 4 + i) * 128, pd.col0 + half * 64,
                           __ldg(pd.slots + pos0 + i));
        }
      }
      bulk_commit();
      pd.valid = 2;
      __syncwarp();
    };
    // opportunistic: append a tile as soon as it has landed (the tensor core may still be reading it)
    auto try_store = [&](int stage) {
      if (pend[stage].valid == 1 && mbar_test_wait(bar(full0 + stage), pend[stage].phase)) issue_stores(stage);
    };
    // before a ring slot is overwritten: its tile has landed and been consumed
    auto flush_stage = [&](int stage) {
      if (pend[stage].valid == 1) issue_stores(stage);
      if (pend[stage].valid == 2) {
        bulk_wait_read0();  // the stores have read the slot (normally long ago)
        pend[stage].valid = 0;
      }
    };
    for (int k = 0; k < n_rounds; ++k) {
      const Unit u = unit_at(k);
      if (u.n_tiles <= 0) continue;
      const int32_t* slots = p.slot_table + (int64_t)u.r * p.st_stride;
      const int col0 = u.h * kD;
      const bool owner = !p.skip_append && u.owner;
      const int own_lo = u.cached + u.q_start, own_hi = u.cached + min(u.q_len, u.q_start + kBM);
      // The unit's query tile is requested right AFTER its first K tile (see the tile loop): the Q
      // buffer only becomes free once the previous unit's last QK^T has completed, whereas a K ring slot is
      // usually free earlier -- so the first K tile of the next unit does not queue behind the Q wait.
      auto load_q = [&]() {
        // rows past the tensor end are zero filled, rows past the request's end belong to the next
        // request: computed, never stored
        mbar_wait(bar(kQEmpty), (unit_count & 1) ^ 1);
        if (lane == 0) {
          mbar_arrive_expect_tx(bar(kQFull), (uint32_t)kTileBytes);
          for (int half = 0; half < 2; ++half)
            tma_load_2d(sbase + Smem::q + half * kHalfBytes, &map_q, bar(kQFull), u.head * kD + half * 64,
                        u.q_begin + u.q_start);
        }
        __syncwarp();
      };
      // Positions < cached come from the pool through the slot table; positions >= cached are the
      // tokens of this very forward and are read straight from the k / v inputs (row q_begin + pos -
      // cached), so the attention never depends on the append performed concurrently.
      // Rows past the end of the request are other requests' tokens or out of range (zeros): finite,
      // and masked by position.
      const CUtensorMap* nmap = kind == 0 ? &new_k : &new_v;
      const CUtensorMap* nbmap = kind == 0 ? &newbox_k : &newbox_v;
      auto load_rows_one_by_one = [&](uint32_t dst, uint32_t fb, int col, int pos0, int n) {
        for (int i = 0; i < n; ++i) {
          const int pos = pos0 + i;
          if (pos < u.cached) tma_load_2d(dst + i * 128, gmap, fb, col, __ldg(slots + pos));
          else tma_load_2d(dst + i * 128, nmap, fb, col, u.q_begin + pos - u.cached);
        }
      };
      for (int t = 0; t < u.n_tiles; ++t, ++tile_count) {
        const uint32_t stage = tile_count % kStages, phase = (tile_count / kStages) & 1;
        const int tile_begin = t * kBN;
        if (rb > 0) {
          const int n_instr = (kBN / rb) * 2;
          const int box = lane >> 1, half = lane & 1;
          const int pb = tile_begin + box * rb;
          const bool old_box = pb + rb <= u.cached, new_box = pb >= u.cached;
          int first_slot = p.num_slots;
          if (lane < n_instr && old_box) first_slot = __ldg(slots + pb);
          mbar_wait(bar(empty0 + stage), phase ^ 1);
          flush_stage(stage);
          if (lane == 0) mbar_arrive_expect_tx(bar(full0 + stage), kTileBytes);
          __syncwarp();
          if (lane < n_instr) {
            const uint32_t dst = ring + stage * kTileBytes + half * kHalfBytes + box * rb * 128;
            const uint32_t fb = bar(full0 + stage);
            const int col = col0 + half * 64;
            if (old_box) tma_load_2d(dst, bmap, fb, col, first_slot);
            else if (new_box) tma_load_2d(dst, nbmap, fb, col, u.q_begin + pb - u.cached);
            else load_rows_one_by_one(dst, fb, col, pb, rb);  // the box straddling cached_len
          }
        } else {
          // row mode: 32 row groups of four x 2 halves = 2 groups per lane, one single-row box per row
          mbar_wait(bar(empty0 + stage), phase ^ 1);
          flush_stage(stage);
          if (lane == 0) mbar_arrive_expect_tx(bar(full0 + stage), kTileBytes);
          __syncwarp();
#pragma unroll
          for (int it = 0; it < 2; ++it) {
            const int grp = (lane >> 1) + it * 16, half = lane & 1;
            const int pos0 = tile_begin + grp * 4;
            const uint32_t dst = ring + stage * kTileBytes + half * kHalfBytes + grp * 512;
            const uint32_t fb = bar(full0 + stage);
            const int col = col0 + half * 64;
            if (pos0 + 4 <= u.cached) {
              const int4 rr = __ldg(reinterpret_cast<const int4*>(slots + pos0));
              tma_load_2d(dst, gmap, fb, col, rr.x);
              tma_load_2d(dst + 128, gmap, fb, col, rr.y);
              tma_load_2d(dst + 256, gmap, fb, col, rr.z);
              tma_load_2d(dst + 384, gmap, fb, col, rr.w);
            } else {
              load_rows_one_by_one(dst, fb, col, pos0, 4);
            }
          }
        }
        if (kind == 0 && t == 0) load_q();
        // tiles issued earlier may have landed by now
        for (int s2 = 0; s2 < kStages; ++s2)
          if (s2 != (int)stage) try_store(s2);
        // does this tile hold rows this unit has to append?
        const int lo = max(own_lo, tile_begin), hi = min(own_hi, tile_begin + kBN);
        if (owner && lo < hi) {
          pend[stage].valid = 1;
          pend[stage].lo = lo;
          pend[stage].hi = hi;
          pend[stage].tile_begin = tile_begin;
          pend[stage].col0 = col0;
          pend[stage].phase = phase;
          pend[stage].slots = slots;
        }
      }
      ++unit_count;
    }
    // tiles still waiting for their append: wait until they have landed, store, drain
    for (int s = 0; s < kStages; ++s)
      if (pend[s].valid == 1) {
        mbar_wait(bar(full0 + s), pend[s].phase);
        issue_stores(s);
      }
    bulk_wait0();
   }
  } else {
    // ============================================================ consumer warpgroups (64 query rows each)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    T* const tsel = nullptr;              // selects the bf16 / fp16 wgmma overload
    const int wg = (warp - 4) >> 2;       // rows wg*64 .. wg*64+63 of the unit's query tile
    const int cw = warp & 3;
    // accumulator fragment (see sm90.cuh): rows ra = 16*cw + lane/4 and ra + 8 of the warpgroup's 64,
    // columns 8i + 2*(lane%4) (+1), i = 0..15
    const int ra = wg * 64 + 16 * cw + (lane >> 2);
    const int cq = 2 * (lane & 3);
    uint32_t tile_count = 0, unit_count = 0;
    for (int k = 0; k < n_rounds; ++k) {
      const Unit u = unit_at(k);
      if (u.n_tiles <= 0) continue;
      // keys [0, vis_end) are visible to a query row; the warpgroup's last row bounds the tiles it needs
      const int vis0 = min(u.cached + u.q_start + ra + 1, u.kv_len);
      const int vis1 = min(u.cached + u.q_start + ra + 9, u.kv_len);
      const int wg_vis = min(u.cached + u.q_start + wg * 64 + 64, u.kv_len);
      float o[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] = 0.f;
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
      mbar_wait(bar(kQFull), unit_count & 1);
      ++unit_count;
      const uint32_t qa = sbase + Smem::q + wg * 8192;  // 64 rows x 128 B into each half
      for (int j = 0; j < u.n_tiles; ++j, ++tile_count) {
        const uint32_t stage = tile_count % kStages, phase = (tile_count / kStages) & 1;
        const int tile_begin = j * kBN;
        const bool active = tile_begin < wg_vis;  // warpgroup-uniform
        mbar_wait(bar(kFullK + stage), phase);
        float s[64];
        if (active) {
          const uint32_t kb = sbase + Smem::kring + stage * kTileBytes;
#pragma unroll
          for (int i = 0; i < 64; ++i) s[i] = 0.f;
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) {
            const uint64_t da = make_smem_desc(qa + (kk >> 2) * kHalfBytes + (kk & 3) * 32, 16, 1024, kLayoutSW128);
            const uint64_t db = make_smem_desc(kb + (kk >> 2) * kHalfBytes + (kk & 3) * 32, 16, 1024, kLayoutSW128);
            wgmma_m64n128k16_ss(s, da, db, kk > 0, tsel);
          }
          wgmma_commit();
          wgmma_wait0();
        }
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(bar(kEmptyK + stage));
          if (j + 1 == u.n_tiles) mbar_arrive(bar(kQEmpty));  // last QK of the unit
        }
        uint32_t pa[8][4];
        if (active) {
          // ---- scale, causal mask, online softmax (a row's 128 columns live in one quad of lanes)
          float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
          for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int x = 0; x < 4; ++x) {
              const int key = tile_begin + 8 * i + cq + (x & 1);
              const float v = key < ((x >> 1) ? vis1 : vis0) ? s[4 * i + x] * p.scale_log2 : -INFINITY;
              s[4 * i + x] = v;
              mx[x >> 1] = fmaxf(mx[x >> 1], v);
            }
          float alpha[2], m_use[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 1));
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 2));
            const float m_new = fmaxf(m_run[e], mx[e]);
            m_use[e] = (m_new == -INFINITY) ? 0.f : m_new;
            alpha[e] = fast_exp2(m_run[e] - m_use[e]);
            m_run[e] = m_new;
          }
          float ps[2] = {0.f, 0.f};
#pragma unroll
          for (int i = 0; i < 64; ++i) {
            const float e = fast_exp2(s[i] - m_use[(i >> 1) & 1]);
            s[i] = e;
            ps[(i >> 1) & 1] += e;
            o[i] *= alpha[(i >> 1) & 1];
          }
#pragma unroll
          for (int e = 0; e < 2; ++e) l_run[e] = l_run[e] * alpha[e] + ps[e];
          // P as the 16-bit A fragment of k-block kb (keys 16kb .. 16kb+15)
#pragma unroll
          for (int kb = 0; kb < 8; ++kb) {
            pa[kb][0] = pack2<T>(s[8 * kb + 0], s[8 * kb + 1]);
            pa[kb][1] = pack2<T>(s[8 * kb + 2], s[8 * kb + 3]);
            pa[kb][2] = pack2<T>(s[8 * kb + 4], s[8 * kb + 5]);
            pa[kb][3] = pack2<T>(s[8 * kb + 6], s[8 * kb + 7]);
          }
        }
        mbar_wait(bar(kFullV + stage), phase);
        if (active) {
          const uint32_t vb = sbase + Smem::vring + stage * kTileBytes;
          wgmma_fence();
#pragma unroll
          for (int kb = 0; kb < 8; ++kb) {
            // B = V (MN-major): 16 keys = two 8-key swizzle atoms (1024 B each); dims 64..127 at +16 KB
            const uint64_t db = make_smem_desc(vb + kb * 2048, kHalfBytes, 1024, kLayoutSW128);
            wgmma_m64n128k16_rs(o, pa[kb], db, 1u, tsel);
          }
          wgmma_commit();
          wgmma_wait0();
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(kEmptyV + stage));
      }
      // ---- epilogue: O / l -> out, rows ra and ra + 8 (row sums reduced over the quad)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        l_run[e] += __shfl_xor_sync(0xffffffffu, l_run[e], 1);
        l_run[e] += __shfl_xor_sync(0xffffffffu, l_run[e], 2);
      }
      const float inv[2] = {1.f / l_run[0], 1.f / l_run[1]};
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int q_row = u.q_start + ra + 8 * e;
        if (q_row < u.q_len) {
          T* orow = p.out + ((int64_t)(u.q_begin + q_row) * p.hq + u.head) * kD + cq;
#pragma unroll
          for (int i = 0; i < 16; ++i)
            *reinterpret_cast<uint32_t*>(orow + 8 * i) = pack2<T>(o[4 * i + 2 * e] * inv[e], o[4 * i + 2 * e + 1] * inv[e]);
        }
      }
    }
  }

  // ---------------------------------------------------------------- teardown
  __syncthreads();
}

template <typename T>
static int launch(const Params<T>& p, const void* q, int64_t q_rs, int64_t nnz, const void* k_cache,
                  const void* v_cache, cudaStream_t st) {
  CUtensorMap nk, nv, nbk, nbv;
  const bool bf16 = std::is_same<T, __nv_bfloat16>::value;
  CUtensorMap mq, mk, mv, bk, bv;
  const uint64_t cols = (uint64_t)p.hkv * kD;
  if (int rc = encode_tensor_map_2d(&mq, q, nnz, (uint64_t)p.hq * kD, q_rs * 2, 64, kBM, bf16)) return rc;
  if (int rc = get_tensor_map_2d(&mk, k_cache, p.num_slots, cols, cols * 2, 64, 1, bf16)) return rc;
  if (int rc = get_tensor_map_2d(&mv, v_cache, p.num_slots, cols, cols * 2, 64, 1, bf16)) return rc;
  bk = mk;
  bv = mv;
  if (p.box_rows > 0) {
    if (int rc = get_tensor_map_2d(&bk, k_cache, p.num_slots, cols, cols * 2, 64, p.box_rows, bf16)) return rc;
    if (int rc = get_tensor_map_2d(&bv, v_cache, p.num_slots, cols, cols * 2, 64, p.box_rows, bf16)) return rc;
  }
  // the k / v inputs of this forward as [nnz, hkv*128] row-strided tensors (not cached: activations
  // move between forwards)
  if (int rc = encode_tensor_map_2d(&nk, p.k_new, nnz, cols, p.kv_rs * 2, 64, 1, bf16)) return rc;
  if (int rc = encode_tensor_map_2d(&nv, p.v_new, nnz, cols, p.kv_rs * 2, 64, 1, bf16)) return rc;
  nbk = nk;
  nbv = nv;
  if (p.box_rows > 0) {
    if (int rc = encode_tensor_map_2d(&nbk, p.k_new, nnz, cols, p.kv_rs * 2, 64, p.box_rows, bf16)) return rc;
    if (int rc = encode_tensor_map_2d(&nbv, p.v_new, nnz, cols, p.kv_rs * 2, 64, p.box_rows, bf16)) return rc;
  }
  const size_t smem = Smem::total + 1024;
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(attn_prefill_tc_kernel<T>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  attn_prefill_tc_kernel<T><<<num_sms(), kThreads, smem, st>>>(p, mq, mk, mv, bk, bv, nk, nv, nbk, nbv);
  B200_POST_LAUNCH();
  return 0;
}

}  // namespace ptc

extern std::atomic<int> g_prefill_skip_append;

// entry used by b200_attn_prefill (attn_prefill.cu)
int launch_prefill_tc(const void* q, int64_t q_rs, int64_t nnz, const void* k, const void* v, int64_t kv_rs,
                      void* k_cache, void* v_cache, const int32_t* out_loc, const int32_t* slot_table, int64_t st_stride, const int32_t* seq_lens,
                      const int32_t* cu_q, const int32_t* prefill_plan, int bs, int hq, int hkv,
                      int64_t num_slots, int page_size, float scale_log2, void* out, int dtype,
                      cudaStream_t st) {
  B200_CHECK_ARG(num_slots > 0 && num_slots < (1ll << 31), "attn_prefill: bad num_slots");
  B200_CHECK_ARG(st_stride % 4 == 0 && ((uintptr_t)slot_table % 16) == 0,
                 "attn_prefill: slot table rows must be 16-byte aligned");
  B200_CHECK_ARG(prefill_plan != nullptr, "attn_prefill: prefill_plan is NULL (b200_build_prefill_plan)");
  int box_rows = 0;
  if (page_size >= 8) {
    box_rows = 64;
    while (box_rows > 8 && (page_size % box_rows) != 0) box_rows >>= 1;
    if (page_size % box_rows != 0) box_rows = 0;
  }
#define RUN(T_)                                                                                    \
  ptc::Params<T_> p{slot_table, st_stride, seq_lens, cu_q, prefill_plan, bs, hq, hkv, (int)num_slots, \
                    box_rows, scale_log2, (T_*)out, (const T_*)k, (const T_*)v, kv_rs, (T_*)k_cache,  \
                    (T_*)v_cache, out_loc, nnz, g_prefill_skip_append.load()};                                                   \
  return ptc::launch<T_>(p, q, q_rs, nnz, k_cache, v_cache, st)
  if (dtype == B200_DTYPE_BF16) {
    RUN(__nv_bfloat16);
  }
  RUN(__half);
#undef RUN
}

}  // namespace b200
