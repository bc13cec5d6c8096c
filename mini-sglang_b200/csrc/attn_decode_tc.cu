// Hopper-native batched decode: TMA -> 128B-swizzled smem -> wgmma (register accumulators).
//
// Replaces store_kv + BatchDecodeWithPagedKVCacheWrapper.run (python/minisgl/attention/fi.py:185-188)
// with one persistent launch (+ the split-KV combine).  HBM-bound; algorithmic bytes as in
// attn_decode.cu.  One CTA per SM, 320 threads, warp-specialised:
//
//   warps 0-3 TMA producers, 3-stage rings of 32 KB K and 32 KB V tiles (two 64-column halves of a
//            128-key tile), data lands directly in the 128-byte-swizzled layout wgmma consumes.
//            * page_size >= 8 ("box mode", warp 0 = K, warp 1 = V): the slots of a page are contiguous
//              rows of the pool, so one tiled TMA box of min(page_size, 64) rows x 128 B is issued per
//              page piece -- 4 instructions per tile and half at page_size 64.
//            * page_size < 8 ("row mode", all four warps): one single-row TMA box per token row and
//              half; rows past the end of the KV range are out-of-range rows (zero filled), so stale
//              pool memory is never multiplied in.
//   warps 4-7 one consumer warpgroup: S^T[128 keys x 8] = K_tile . Q^T and O^T[128 dims x 8] += V_tile^T . P^T
//            as wgmma m64n8k16 (two 64-row blocks each): the keys / head dims fill M and the <= 8 query
//            heads of the GQA group sit in N = 8, so no tensor-core row is spent on padding.  Softmax on
//            the score fragments (tile max across the four warps through smem + a named barrier), P^T to
//            smem as the 16-bit B operand, O^T stays in registers with the online-softmax rescale.
//   warp 8   Q loader: the group's q rows -> swizzled smem operand (double buffered across units).
//   warp 9   split-KV combiner: the last-arriving chunk of a (request, kv head) merges the partials.
//
// Fused pre-attention (p.fuse, b200_attn_decode_fused): q and the new k row arrive RAW (straight from the
// qkv projection); the Q loader applies the per-head RMSNorm + neox RoPE of layers/attention.py:50-54 with
// the arithmetic of qknorm_rope_kernel (qknorm_rope.cuh, bit for bit) while it builds the swizzled Q
// operand, and hands the roped q / k rows the epilogue needs (new-token score, append payload) to the
// consumer warps through a small smem ring -- the separate qk-norm + RoPE launch disappears and q / k are
// never written back to global memory (only the pool row of the new token is).
//
// The token appended by this launch is handled without touching the pool copy that is being
// written: its score / value come straight from the k/v inputs on CUDA cores in the epilogue of
// the unit that owns position kv_len-1 (which also performs the append).
#include "b200attn.h"
#include "combine.cuh"
#include "common.cuh"
#include "qknorm_rope.cuh"
#include "sm90.cuh"

#include <type_traits>

namespace b200 {

int get_tensor_map_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t row_stride_bytes, uint32_t box_cols, uint32_t box_rows, bool is_bf16);

namespace dtc {

using namespace sm90;

constexpr int kD = 128;
constexpr int kTileN = 128;                 // keys per tile
constexpr int kStages = 3;
constexpr int kThreads = 320;
constexpr int kWarpQ = 8, kWarpCombine = 9;
constexpr int kHalfBytes = kTileN * 128;    // one 64-column half of a K or V tile: 16 KB
constexpr int kStageBytes = 2 * kHalfBytes; // one K (or V) tile: half 0 | half 1 = 32 KB
constexpr int kNPad = 8;                    // wgmma N (query heads of the group, padded)
constexpr int kQBufBytes = 2 * 1024;        // two halves of [8 rows x 128 B], 128B-swizzled
constexpr int kPBufBytes = kNPad * kTileN * 2;  // P^T [8 x 128] 16-bit, no-swizzle K-major
constexpr int kMaxUnitsSmem = 96;           // per-CTA work units decoded once into smem
constexpr int kEpiSlots = 4;                // fused mode: roped (q heads, new k) rows in flight to the epilogue
constexpr int kEpiSlotBytes = 9 * kD * 2;   // up to 8 q heads + the k row, 128 x 16-bit each

struct Smem {
  // offsets from the 1024-aligned base
  static constexpr int kring = 0;                          // K tiles, released right after QK
  static constexpr int vring = kStages * kStageBytes;      // V tiles, released after PV
  static constexpr int qbuf = 2 * kStages * kStageBytes;
  static constexpr int pbuf = qbuf + 2 * kQBufBytes;
  static constexpr int bars = pbuf + kPBufBytes;           // 32 mbarriers
  static constexpr int red = bars + 32 * 8;                // floats: tile max [4][8], [2][4][8] row sums, [2][4][8] new-token dots
  static constexpr int units = red + (32 + 64 + 64) * 4;   // decoded work units
  static constexpr int epi = units + kMaxUnitsSmem * 40;   // fused mode: kEpiSlots x [9][128] 16-bit
  static constexpr int total = epi + kEpiSlots * kEpiSlotBytes;
};
static_assert(Smem::total + 1024 <= 232448, "decode kernel shared memory exceeds the 227 KB per-CTA limit");
enum Bar { kFullK = 0, kEmptyK = 3, kFullV = 6, kEmptyV = 9, kQFull = 12, kQEmpty = 14, kFinFull = 16, kFinEmpty = 20, kEpiFull = 24, kEpiEmpty = 28 };
constexpr int kFinRing = 4;  // units in flight between the consumer warps and the combiner warp

template <typename T>
struct Params {
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
  int num_slots;
  int box_rows;  // rows per tiled TMA box (8..64, divides page_size); 0 = row mode
  int fused_combine;  // 1: last-arriving unit merges the split-KV partials in this launch
  float scale_log2;
  T* out;
  float* part_o;
  float* part_ml;
  int* counters;  // [bs][hkv] split-KV arrival counters, zero between launches
  // fused pre-attention (fuse = 1): q / k_new are raw; norm weights may be NULL (models without qk-norm)
  int early;  // 1: captured launch -- TMA producers do not wait for the predecessor (see the kernel prologue)
  int fuse;
  const T* qw;
  const T* kw;
  float eps;
  const int32_t* positions;
  const float* cos_sin;  // fp32 [max_pos][128] = cos | sin
};

struct Unit {
  int r, c, h, n_chunks, kv_len, kv_begin, kv_end_tc, n_tiles;
  int last_chunk;
};
static_assert(sizeof(Unit) <= 40, "Unit must fit its smem slot");

// Work unit `pos` of the size-sorted order (metadata.cu): entry = r | chunk << 16 | n_chunks << 20,
// the hkv heads of an item are adjacent positions (neighbouring CTAs stream the same token rows).
__device__ __forceinline__ Unit get_unit(int pos, int hkv, int chunk_tokens, const int32_t* order,
                                         const int32_t* seq_lens) {
  Unit u;
  const int item = pos / hkv;
  u.h = pos - item * hkv;
  const int e = order[item];
  u.r = e & 0xffff;
  u.c = (e >> 16) & 0xf;
  u.n_chunks = (e >> 20) & 0x1f;
  u.kv_len = seq_lens[u.r];
  u.kv_begin = u.c * chunk_tokens;
  const int kv_end = min(u.kv_len, u.kv_begin + chunk_tokens);
  u.last_chunk = (u.c == u.n_chunks - 1);
  u.kv_end_tc = u.last_chunk ? kv_end - 1 : kv_end;  // the appended token is handled on CUDA cores
  const int n = u.kv_end_tc - u.kv_begin;
  u.n_tiles = n > 0 ? (n + kTileN - 1) / kTileN : 0;
  return u;
}

template <typename T, int G>
__global__ void __launch_bounds__(kThreads, 1)
attn_decode_tc_kernel(const Params<T> p, const __grid_constant__ CUtensorMap map_k,
                      const __grid_constant__ CUtensorMap map_v,
                      const __grid_constant__ CUtensorMap box_k,
                      const __grid_constant__ CUtensorMap box_v) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B-swizzled tiles
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid / kWarp, lane = tid % kWarp;
  auto bar = [&](int i) { return sbase + Smem::bars + i * 8; };
  float* red = reinterpret_cast<float*>(smem + Smem::red);
  uint8_t* sUnits = smem + Smem::units;

  // ---------------------------------------------------------------- setup that touches no global memory
  // zero the Q operand buffers whose padding rows (heads >= G) are never written again
  for (int i = tid; i < (2 * kQBufBytes) / 16; i += kThreads)
    reinterpret_cast<uint4*>(smem + Smem::qbuf)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(bar(kFullK + s), 1);
      mbar_init(bar(kEmptyK + s), 4);  // one elected arrival per consumer warp
      mbar_init(bar(kFullV + s), 1);
      mbar_init(bar(kEmptyV + s), 4);
    }
    for (int b = 0; b < kFinRing; ++b) {
      mbar_init(bar(kFinFull + b), 128);
      mbar_init(bar(kFinEmpty + b), 1);
    }
    for (int b = 0; b < kEpiSlots; ++b) {
      mbar_init(bar(kEpiFull + b), 1);
      mbar_init(bar(kEpiEmpty + b), 1);
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(bar(kQFull + b), 1);
      mbar_init(bar(kQEmpty + b), 4);
    }
    fence_barrier_init();
    prefetch_tensormap(&map_k);
    prefetch_tensormap(&map_v);
    prefetch_tensormap(&box_k);
    prefetch_tensormap(&box_v);
  }
  // PDL: everything above may overlap the tail of the previous kernel in the stream.
  //  * p.early == 0 (eager launches): wait here -- from here on the results of every kernel before this one
  //    (in particular the metadata kernel's plan / seq_lens / slot table) are complete and visible.
  //  * p.early == 1 (launch captured into a CUDA graph): the metadata was written BEFORE the graph started
  //    (prepare_for_replay), and the K/V rows this launch streams belong to this layer's pool slice, which
  //    no other kernel of the graph writes -- so only the roles that consume the predecessor's outputs
  //    (Q loader: q / k_new; consumer warps: v_new, out_loc operands, output / partial stores; combiner)
  //    wait, while the TMA producers start streaming K/V at once: prologue, pipeline fill and the
  //    predecessor's tail (or a small kernel in between, e.g. the TP all-reduce) overlap.
  if (!p.early) pdl_wait();
  pdl_launch_dependents();
  const int chunk_tokens = p.plan[0];
  const int total_units = p.plan[1] * p.hkv;
  const int32_t* order = p.plan + kPlanHeader + p.bs + 1;
  const int32_t* seq_lens = p.seq_lens;
  // This CTA's k-th unit is position k*grid + (k even ? cta : grid-1-cta) of the size-sorted order
  // ("snake" dealing): per-CTA work is balanced to within about one tile.
  const int grid = gridDim.x, cta = blockIdx.x;
  const int n_rounds = (total_units + grid - 1) / grid;
  auto pos_of = [&](int k) { return k * grid + ((k & 1) ? grid - 1 - cta : cta); };

  // ---------------------------------------------------------------- one-time setup
  // every role walks the same unit list: decode it once, in parallel, into smem
  for (int k = tid; k < kMaxUnitsSmem && k < n_rounds; k += kThreads) {
    const int pos = pos_of(k);
    Unit u;
    u.n_tiles = -1;  // marks "no unit in this round"
    if (pos < total_units) u = get_unit(pos, p.hkv, chunk_tokens, order, seq_lens);
    *reinterpret_cast<Unit*>(sUnits + k * 40) = u;
  }
  auto unit_at = [&](int k) {
    if (k < kMaxUnitsSmem) return *reinterpret_cast<const Unit*>(sUnits + k * 40);
    const int pos = pos_of(k);
    Unit u;
    u.n_tiles = -1;
    if (pos < total_units) u = get_unit(pos, p.hkv, chunk_tokens, order, seq_lens);
    return u;
  };
  fence_proxy_async_smem();  // zero-fill above must be visible to wgmma operand reads
  __syncthreads();
  if (warp < 4) {
    // ============================================================ TMA producers
    // K and V travel in separate rings (a K tile is dead as soon as QK^T has completed, a V
    // tile only after PV), so each has its own producers: box mode warp 0 = K, warp 1 = V;
    // row mode warps 0,1 = K rows 0-63 / 64-127, warps 2,3 = V.
    const int rb = p.box_rows;
    const int kind = rb > 0 ? warp : (warp >> 1);  // 0 = K, 1 = V
    if (rb > 0 && warp >= 2) {
      // box mode needs a handful of instructions per tile: two warps are plenty
    } else {
      const CUtensorMap* gmap = kind == 0 ? &map_k : &map_v;
      const CUtensorMap* bmap = kind == 0 ? &box_k : &box_v;
      const int full0 = kind == 0 ? kFullK : kFullV, empty0 = kind == 0 ? kEmptyK : kEmptyV;
      const uint32_t ring = sbase + (kind == 0 ? Smem::kring : Smem::vring);
      uint32_t tile_count = 0;
      for (int k = 0; k < n_rounds; ++k) {
        const Unit u = unit_at(k);
        if (u.n_tiles <= 0) continue;
        const int32_t* slots = p.slot_table + (int64_t)u.r * p.st_stride;
        const int col0 = u.h * kD;
        // four slots of row group `grp` (rows 4*grp..4*grp+3 of tile t); invalid rows -> out of range
        auto load_group = [&](int t, int grp) {
          int4 rr;
          const int pos0 = u.kv_begin + t * kTileN + grp * 4;
          if (pos0 + 3 < u.kv_end_tc) {
            rr = __ldg(reinterpret_cast<const int4*>(slots + pos0));
          } else {
            rr.x = pos0 + 0 < u.kv_end_tc ? __ldg(slots + pos0 + 0) : p.num_slots;
            rr.y = pos0 + 1 < u.kv_end_tc ? __ldg(slots + pos0 + 1) : p.num_slots;
            rr.z = pos0 + 2 < u.kv_end_tc ? __ldg(slots + pos0 + 2) : p.num_slots;
            rr.w = pos0 + 3 < u.kv_end_tc ? __ldg(slots + pos0 + 3) : p.num_slots;
          }
          return rr;
        };
        if (rb == 0) {
          // ---- row mode: this warp owns 64 rows; lane = (row group of four, half)
          const int grp = (warp & 1) * 16 + (lane >> 1), half = lane & 1;
          int4 nxt = make_int4(0, 0, 0, 0);
          if (u.n_tiles > 0) nxt = load_group(0, grp);
          for (int t = 0; t < u.n_tiles; ++t, ++tile_count) {
            const int4 cur = nxt;
            if (t + 1 < u.n_tiles) nxt = load_group(t + 1, grp);
            const uint32_t stage = tile_count % kStages, phase = (tile_count / kStages) & 1;
            mbar_wait(bar(empty0 + stage), phase ^ 1);
            if ((warp & 1) == 0 && lane == 0) mbar_arrive_expect_tx(bar(full0 + stage), kStageBytes);
            __syncwarp();
            const uint32_t dst = ring + stage * kStageBytes + half * kHalfBytes + grp * 512;
            const uint32_t fb = bar(full0 + stage);
            const int col = col0 + half * 64;
            tma_load_2d(dst, gmap, fb, col, cur.x);
            tma_load_2d(dst + 128, gmap, fb, col, cur.y);
            tma_load_2d(dst + 256, gmap, fb, col, cur.z);
            tma_load_2d(dst + 384, gmap, fb, col, cur.w);
          }
        } else {
          // ---- box mode: instruction idx = (box, half); a box is rb consecutive positions of one page
          const int n_instr = (kTileN / rb) * 2;  // <= 32
          for (int t = 0; t < u.n_tiles; ++t, ++tile_count) {
            const uint32_t stage = tile_count % kStages, phase = (tile_count / kStages) & 1;
            const int tile_begin = u.kv_begin + t * kTileN;
            const int box = lane >> 1, half = lane & 1;
            const int pb = tile_begin + box * rb;
            // slot of the box's first row, loaded before the wait so its latency overlaps
            int first_slot = p.num_slots;
            if (lane < n_instr && pb < u.kv_end_tc) first_slot = __ldg(slots + pb);
            mbar_wait(bar(empty0 + stage), phase ^ 1);
            if (lane == 0) mbar_arrive_expect_tx(bar(full0 + stage), kStageBytes);
            __syncwarp();
            if (lane < n_instr) {
              const uint32_t dst = ring + stage * kStageBytes + half * kHalfBytes + box * rb * 128;
              const uint32_t fb = bar(full0 + stage);
              const int col = col0 + half * 64;
              // A box reaching past the end of the range still lies inside the request's page; the
              // extra K rows are masked by position and the extra V rows are zeroed in smem by the
              // consumer warps before PV.  A box wholly past the end gets an out-of-range row => zeros.
              tma_load_2d(dst, bmap, fb, col, first_slot);
            }
          }
        }
      }
    }
  } else if (warp == kWarpQ) {
    // ============================================================ Q loader
    if (p.early) pdl_wait();
    uint32_t unit_count = 0, epi_count = 0;
    for (int k = 0; k < n_rounds; ++k) {
      const Unit u = unit_at(k);
      if (u.n_tiles < 0) continue;
      const bool need_q = u.n_tiles > 0;                 // the tensor core needs the Q operand
      const bool need_epi = p.fuse && u.last_chunk;      // the epilogue needs roped q / k rows
      if (!need_q && !need_epi) continue;
      const uint32_t qb = unit_count & 1, es = epi_count % kEpiSlots;
      if (need_q) mbar_wait(bar(kQEmpty + qb), ((unit_count >> 1) & 1) ^ 1);
      if (need_epi) mbar_wait(bar(kEpiEmpty + es), ((epi_count / kEpiSlots) & 1) ^ 1);
      uint8_t* qdst = smem + Smem::qbuf + qb * kQBufBytes;
      if (!p.fuse) {
        for (int idx = lane; idx < G * 16; idx += kWarp) {
          const int g = idx >> 4, cc = idx & 15;
          const Vec8 v = *reinterpret_cast<const Vec8*>(p.q + (int64_t)u.r * p.q_rs +
                                                        (int64_t)(u.h * G + g) * kD + cc * 8);
          *reinterpret_cast<Vec8*>(qdst + (cc >> 3) * 1024 + sw128_offset(g, cc & 7)) = v;
        }
      } else {
        // per-head RMSNorm + RoPE on 16-lane groups, two rows per pass: the G q heads of the group and,
        // for the unit that owns the new token, its k row (row index G).  Uniform trip count: the
        // shuffles inside qknorm_rope_lanes need the whole warp.
        uint8_t* edst = smem + Smem::epi + es * kEpiSlotBytes;
        const float* cs_row = p.cos_sin + (int64_t)__ldg(p.positions + u.r) * kD;
        const int n_rows = G + (need_epi ? 1 : 0);
        for (int base = 0; base < n_rows; base += 2) {
          const int g = base + (lane >> 4), cc = lane & 15;
          const bool active = g < n_rows, is_k = (g == G);
          Vec8 xv = {};
          if (active)
            xv = is_k ? *reinterpret_cast<const Vec8*>(p.k_new + (int64_t)u.r * p.k_rs + u.h * kD + cc * 8)
                      : *reinterpret_cast<const Vec8*>(p.q + (int64_t)u.r * p.q_rs + (int64_t)(u.h * G + g) * kD + cc * 8);
          const Vec8 rv = qknorm_rope_lanes<T, 16, true>(xv, cc, is_k ? p.kw : p.qw, p.eps, cs_row, active);
          if (active) {
            if (!is_k && need_q) *reinterpret_cast<Vec8*>(qdst + (cc >> 3) * 1024 + sw128_offset(g, cc & 7)) = rv;
            if (need_epi) *reinterpret_cast<Vec8*>(edst + g * (kD * 2) + cc * 16) = rv;
          }
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        if (need_q) mbar_arrive(bar(kQFull + qb));
        if (need_epi) mbar_arrive(bar(kEpiFull + es));
      }
      if (need_q) ++unit_count;
      if (need_epi) ++epi_count;
    }
  } else if (warp >= 4 && warp < 8) {
    // ============================================================ consumer warpgroup (128 threads)
    if (p.early) pdl_wait();
    constexpr bool kTransV = true;  // A = V^T: the head dims (M) are the contiguous axis of a V tile
    T* const tsel = nullptr;        // selects the bf16 / fp16 wgmma overload
    const int ct = tid - 128;       // 0..127
    const int cw = warp - 4;        // warp of the group
    // accumulator fragment (see sm90.cuh): element i of 64-row block mb is row mb*64 + r0 + (i>>1)*8,
    // column h0 + (i&1).  Rows are keys (S^T) or head dims (O^T), columns are the group's query heads.
    const int r0 = 16 * cw + (lane >> 2), h0 = 2 * (lane & 3);
    auto row_of = [&](int mb, int i) { return mb * 64 + r0 + ((i >> 1) << 3); };
    float* red_max = red;          // [4 warps][8 heads]
    float* red_sum0 = red + 32;    // [2 parity][4][8]
    float* red_new0 = red + 96;    // [2 parity][4][8]
    uint32_t tile_count = 0, q_count = 0, fin_count = 0, epi_fin = 0, unit_par = 0;
    for (int k = 0; k < n_rounds; ++k) {
      const Unit u = unit_at(k);
      if (u.n_tiles < 0) continue;  // no unit for this CTA in the last round
      float acc[2][4], l_thr[2], m_run[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        l_thr[e] = 0.f;
        m_run[e] = -INFINITY;
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[e][i] = 0.f;
      }
      // operands of the appended token's score / value (x = mb*2 + (i>>1) indexes this thread's four dims):
      // issue the loads now, use them in the epilogue -- their latency hides behind the tile loop
      float q_new[2][4], kn[4], vn[4];
      int app_loc = 0;
      Vec8 app_x = Vec8{{0u, 0u, 0u, 0u}};
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        kn[x] = vn[x] = 0.f;
        q_new[0][x] = q_new[1][x] = 0.f;
      }
      if (u.last_chunk) {
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          const int dim = row_of(x >> 1, (x & 1) << 1);
          if (!p.fuse) {  // fused mode: roped q / k come from the Q loader's ring in the epilogue
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (h0 + e < G)
                q_new[e][x] = DTypeTraits<T>::to_float(p.q[(int64_t)u.r * p.q_rs + (int64_t)(u.h * G + h0 + e) * kD + dim]);
            kn[x] = DTypeTraits<T>::to_float(p.k_new[(int64_t)u.r * p.k_rs + u.h * kD + dim]);
          }
          vn[x] = DTypeTraits<T>::to_float(p.v_new[(int64_t)u.r * p.v_rs + u.h * kD + dim]);
        }
        // fused KV append (threads 0-15: K row, 16-31: V row, 16 bytes each): destination slot and
        // payload are fetched here as well, so the epilogue only issues the store
        if (ct < 32) {
          app_loc = p.out_loc[u.r];
          const T* src = ct < 16 ? p.k_new + (int64_t)u.r * p.k_rs : p.v_new + (int64_t)u.r * p.v_rs;
          if (!(p.fuse && ct < 16)) app_x = *reinterpret_cast<const Vec8*>(src + u.h * kD + (ct & 15) * 8);
        }
      }
      if (u.n_tiles > 0) {
        const uint32_t qb = q_count & 1;
        mbar_wait(bar(kQFull + qb), (q_count >> 1) & 1);
        const uint32_t qa = sbase + Smem::qbuf + qb * kQBufBytes;
        for (int j = 0; j < u.n_tiles; ++j, ++tile_count) {
          const uint32_t stage = tile_count % kStages, sphase = (tile_count / kStages) & 1;
          // ---- S^T = K_tile . Q^T: A = K rows (K-major, 128B swizzle), B = Q rows (K-major)
          mbar_wait(bar(kFullK + stage), sphase);
          const uint32_t kb = sbase + Smem::kring + stage * kStageBytes;
          float s[2][4];
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int i = 0; i < 4; ++i) s[mb][i] = 0.f;
          wgmma_fence();
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
              const uint64_t da = make_smem_desc(kb + mb * 8192 + (kk >> 2) * kHalfBytes + (kk & 3) * 32, 16, 1024, kLayoutSW128);
              const uint64_t db = make_smem_desc(qa + (kk >> 2) * 1024 + (kk & 3) * 32, 16, 1024, kLayoutSW128);
              wgmma_m64n8k16_ss<0>(s[mb], da, db, kk > 0, tsel);
            }
          wgmma_commit();
          wgmma_wait0();
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(bar(kEmptyK + stage));                      // the K tile is dead
            if (j + 1 == u.n_tiles) mbar_arrive(bar(kQEmpty + qb));  // last QK of the unit
          }
          const int n_valid = u.kv_end_tc - (u.kv_begin + j * kTileN);  // >= 1
          if (p.box_rows > 0 && n_valid < kTileN) {
            // box mode, last tile of the range: the V rows past the end hold whatever the page holds
            // (possibly NaN bit patterns): zero them so that 0 * garbage cannot reach the output
            mbar_wait(bar(kFullV + stage), sphase);
            uint8_t* vt = smem + Smem::vring + stage * kStageBytes;
            for (int idx = ct; idx < (kTileN - n_valid) * 16; idx += 128) {
              const int row = n_valid + (idx >> 4), c16 = idx & 15;
              *reinterpret_cast<uint4*>(vt + (c16 >> 3) * kHalfBytes + row * 128 + (c16 & 7) * 16) = make_uint4(0, 0, 0, 0);
            }
            fence_proxy_async_smem();
          }
          // ---- online softmax: per head (column) max over the 128 keys of the tile
          float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float v = row_of(mb, i) < n_valid ? s[mb][i] * p.scale_log2 : -INFINITY;
              s[mb][i] = v;
              mx[i & 1] = fmaxf(mx[i & 1], v);
            }
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 4));
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 8));
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 16));
          }
          if (lane < 4) {
            red_max[cw * 8 + h0] = mx[0];
            red_max[cw * 8 + h0 + 1] = mx[1];
          }
          named_bar_sync(1, 128);
          float alpha[2], psum[2] = {0.f, 0.f};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int hh = h0 + e;
            const float mt = fmaxf(fmaxf(red_max[hh], red_max[8 + hh]), fmaxf(red_max[16 + hh], red_max[24 + hh]));
            const float m_new = fmaxf(m_run[e], mt);  // finite: every tile has >= 1 valid key
            alpha[e] = fast_exp2(m_run[e] - m_new);
            m_run[e] = m_new;
          }
          // P^T [head][key] as 8x8 core matrices (no swizzle, K-major): key chunks of 8 are 128 B apart
          uint8_t* pdst = smem + Smem::pbuf;
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int key = row_of(mb, i), hh = h0 + (i & 1);
              const float pv = fast_exp2(s[mb][i] - m_run[i & 1]);
              psum[i & 1] += pv;
              *reinterpret_cast<T*>(pdst + (key >> 3) * 128 + hh * 16 + (key & 7) * 2) = DTypeTraits<T>::from_float(pv);
              acc[mb][i] *= alpha[i & 1];
            }
#pragma unroll
          for (int e = 0; e < 2; ++e) l_thr[e] = l_thr[e] * alpha[e] + psum[e];
          fence_proxy_async_smem();  // P^T (and zeroed V rows) visible to the tensor core
          named_bar_sync(1, 128);    // every warp's P^T is written; the tile maxima may be overwritten
          // ---- O^T += V_tile^T . P^T: A = V rows read MN-major, B = P^T (K-major, no swizzle)
          mbar_wait(bar(kFullV + stage), sphase);
          const uint32_t vb = sbase + Smem::vring + stage * kStageBytes;
          const uint32_t pb = sbase + Smem::pbuf;
          wgmma_fence();
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
              // 16 keys = two 8-key swizzle atoms of 1024 B; dims 64..127 in the second half (+16 KB)
              const uint64_t da = make_smem_desc(vb + mb * kHalfBytes + kk * 2048, kHalfBytes, 1024, kLayoutSW128);
              const uint64_t db = make_smem_desc(pb + kk * 256, 128, 1024, kLayoutNone);
              wgmma_m64n8k16_ss<kTransV ? 1 : 0>(acc[mb], da, db, 1u, tsel);
            }
          wgmma_commit();
          wgmma_wait0();
          __syncwarp();
          if (lane == 0) mbar_arrive(bar(kEmptyV + stage));
        }
        ++q_count;
      }

      // ---- unit epilogue on CUDA cores: row sums, the appended token (score, value, pool append), output.
      // Reduction scratch double buffered by unit parity: the next unit may write its slots while
      // stragglers still read this unit's (every unit passes a named barrier in between).
      float* red_sum = red_sum0 + unit_par * 32;
      float* red_new = red_new0 + unit_par * 32;
      unit_par ^= 1;
      const bool epi = p.fuse && u.last_chunk;
      const uint32_t es = epi_fin % kEpiSlots;
      if (epi) {
        // fused mode: the Q loader left the roped q rows of the group and the roped new k row in the ring
        mbar_wait(bar(kEpiFull + es), (epi_fin / kEpiSlots) & 1);
        ++epi_fin;
        const uint8_t* esrc = smem + Smem::epi + es * kEpiSlotBytes;
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          const int dim = row_of(x >> 1, (x & 1) << 1);
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (h0 + e < G) q_new[e][x] = DTypeTraits<T>::to_float(*reinterpret_cast<const T*>(esrc + (h0 + e) * (kD * 2) + dim * 2));
          kn[x] = DTypeTraits<T>::to_float(*reinterpret_cast<const T*>(esrc + G * (kD * 2) + dim * 2));
        }
        if (ct < 16) app_x = *reinterpret_cast<const Vec8*>(esrc + G * (kD * 2) + ct * 16);
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float ls = l_thr[e], sn = 0.f;
        if (u.last_chunk) sn = (q_new[e][0] * kn[0] + q_new[e][1] * kn[1]) + (q_new[e][2] * kn[2] + q_new[e][3] * kn[3]);
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          ls += __shfl_xor_sync(0xffffffffu, ls, o);
          sn += __shfl_xor_sync(0xffffffffu, sn, o);
        }
        if (lane < 4) {
          red_sum[cw * 8 + h0 + e] = ls;
          red_new[cw * 8 + h0 + e] = sn;
        }
      }
      named_bar_sync(1, 128);
      if (epi && ct == 0) mbar_arrive(bar(kEpiEmpty + es));  // every thread has read its ring values
      float l_tot[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int hh = h0 + e;
        l_tot[e] = red_sum[hh] + red_sum[8 + hh] + red_sum[16 + hh] + red_sum[24 + hh];
      }
      if (u.last_chunk) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int hh = h0 + e;
          const float s_new = (red_new[hh] + red_new[8 + hh] + red_new[16 + hh] + red_new[24 + hh]) * p.scale_log2;
          const float m_new = fmaxf(m_run[e], s_new);
          const float a = fast_exp2(m_run[e] - m_new);
          const float pnew = fast_exp2(s_new - m_new);
#pragma unroll
          for (int mb = 0; mb < 2; ++mb) {
            acc[mb][e] = acc[mb][e] * a + pnew * vn[mb * 2];
            acc[mb][2 + e] = acc[mb][2 + e] * a + pnew * vn[mb * 2 + 1];
          }
          l_tot[e] = l_tot[e] * a + pnew;
          m_run[e] = m_new;
        }
        // fused KV append: this head's new K and V rows go into the pool (operands fetched at unit start)
        if (ct < 32) {
          T* dst = (ct < 16 ? p.k_cache : p.v_cache) + (int64_t)app_loc * p.hkv * kD + u.h * kD + (ct & 15) * 8;
          *reinterpret_cast<Vec8*>(dst) = app_x;
        }
      }
      // ---- write out
      if (u.n_chunks == 1) {
        const float inv[2] = {1.f / l_tot[0], 1.f / l_tot[1]};
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (h0 + (i & 1) < G)
              p.out[((int64_t)u.r * p.hq + u.h * G + h0 + (i & 1)) * kD + row_of(mb, i)] =
                  DTypeTraits<T>::from_float(acc[mb][i] * inv[i & 1]);
      } else {
        const int64_t base = ((int64_t)u.r * kMaxSplits + u.c) * p.hq + u.h * G;
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (h0 + (i & 1) < G) p.part_o[(base + h0 + (i & 1)) * kD + row_of(mb, i)] = acc[mb][i];
        if (cw == 0 && lane < 4) {
          // m_run / l_tot of a head are uniform across threads; lanes 0-3 of warp 0 store heads h0, h0+1
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (h0 + e < G) {
              p.part_ml[(base + h0 + e) * 2 + 0] = m_run[e];
              p.part_ml[(base + h0 + e) * 2 + 1] = l_tot[e];
            }
        }
        // ---- hand the unit to the combiner warp (asynchronous split-KV merge): the consumer warps
        // only pay an mbarrier arrive; the release/acquire pair orders the partial stores above
        // before the combiner's device-scope fence + arrival counter.
        if (p.fused_combine) {
          const uint32_t slot = fin_count % kFinRing;
          mbar_wait(bar(kFinEmpty + slot), ((fin_count / kFinRing) & 1) ^ 1);
          mbar_arrive(bar(kFinFull + slot));
          ++fin_count;
        }
      }
    }
  } else if (warp == kWarpCombine) {
    // ============================================================ split-KV combiner (one warp)
    // For every multi-chunk unit of this CTA: count in on the (request, kv head) arrival counter;
    // whoever arrives last merges all partials (flash-decoding reduction) and writes the output.
    if (p.early) pdl_wait();
    if (p.fused_combine) {
      uint32_t fin_count = 0;
      for (int k = 0; k < n_rounds; ++k) {
        const Unit u = unit_at(k);
        if (u.n_tiles < 0 || u.n_chunks == 1) continue;
        const uint32_t slot = fin_count % kFinRing;
        mbar_wait(bar(kFinFull + slot), (fin_count / kFinRing) & 1);
        ++fin_count;
        __threadfence();
        int last = 0;
        if (lane == 0) {
          const int old = atomicAdd(p.counters + u.r * p.hkv + u.h, 1);
          last = (old == u.n_chunks - 1);
          if (last) p.counters[u.r * p.hkv + u.h] = 0;  // zero again for the next launch
        }
        last = __shfl_sync(0xffffffffu, last, 0);
        if (last) {
          __threadfence();  // acquire the other chunks' partials
          // The merge is pure latency (partials sit in L2, written by other SMs): every load whose address
          // is known is issued before anything is consumed -- (m, l) of all G heads at once, then the
          // partial outputs kMergeBatch chunks x G heads at a time.
          const int64_t b0 = ((int64_t)u.r * kMaxSplits) * p.hq + u.h * G;
          float mc[G], lc[G];
#pragma unroll
          for (int g = 0; g < G; ++g) {  // lane c holds (m, l) of chunk c
            mc[g] = -INFINITY;
            lc[g] = 0.f;
            if (lane < u.n_chunks) {
              const float2 ml = __ldcg(reinterpret_cast<const float2*>(p.part_ml + (b0 + (int64_t)lane * p.hq + g) * 2));
              mc[g] = ml.x;
              lc[g] = ml.y;
            }
          }
          constexpr int kMergeBatch = G <= 2 ? 8 : (G <= 4 ? 4 : 2);
          float4 o[G];
          float wc[G], inv[G];
#pragma unroll
          for (int g = 0; g < G; ++g) o[g] = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int c0 = 0; c0 < u.n_chunks; c0 += kMergeBatch) {
            float4 po[G][kMergeBatch];
#pragma unroll
            for (int g = 0; g < G; ++g)
#pragma unroll
              for (int j = 0; j < kMergeBatch; ++j)
                po[g][j] = c0 + j < u.n_chunks
                               ? __ldcg(reinterpret_cast<const float4*>(p.part_o + (b0 + (int64_t)(c0 + j) * p.hq + g) * kD) + lane)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
            if (c0 == 0) {
#pragma unroll
              for (int g = 0; g < G; ++g) {
                const float mx = warp_max(mc[g]);
                wc[g] = lane < u.n_chunks ? fast_exp2(mc[g] - mx) : 0.f;
                inv[g] = 1.f / warp_sum(wc[g] * lc[g]);
              }
            }
#pragma unroll
            for (int g = 0; g < G; ++g)
#pragma unroll
              for (int j = 0; j < kMergeBatch; ++j) {  // chunk order 0, 1, ... as in combine.cuh
                const float w = __shfl_sync(0xffffffffu, wc[g], (c0 + j) & 31);
                o[g].x += w * po[g][j].x;
                o[g].y += w * po[g][j].y;
                o[g].z += w * po[g][j].z;
                o[g].w += w * po[g][j].w;
              }
          }
#pragma unroll
          for (int g = 0; g < G; ++g) {
            typename DTypeTraits<T>::T2 lo = DTypeTraits<T>::from_float2(o[g].x * inv[g], o[g].y * inv[g]);
            typename DTypeTraits<T>::T2 hi = DTypeTraits<T>::from_float2(o[g].z * inv[g], o[g].w * inv[g]);
            uint2 pk;
            pk.x = *reinterpret_cast<uint32_t*>(&lo);
            pk.y = *reinterpret_cast<uint32_t*>(&hi);
            *reinterpret_cast<uint2*>(p.out + ((int64_t)u.r * p.hq + u.h * G + g) * kD + lane * 4) = pk;
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(kFinEmpty + slot));
      }
    }
  }

  // ---------------------------------------------------------------- teardown
  __syncthreads();
}

template <typename T, int G>
static int launch_g(const Params<T>& p, const CUtensorMap& mk, const CUtensorMap& mv,
                    const CUtensorMap& bk, const CUtensorMap& bv, cudaStream_t st) {
  const size_t smem = Smem::total + 1024;
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(attn_decode_tc_kernel<T, G>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  B200_CHECK_CUDA(launch_pdl(attn_decode_tc_kernel<T, G>, dim3(num_sms()), dim3(kThreads), smem, st, p, mk, mv, bk, bv));
  B200_POST_LAUNCH();
  if (!p.fused_combine) {
    B200_CHECK_CUDA(launch_pdl(attn_combine_kernel<T>, dim3(p.bs, p.hq), dim3(kHeadDim), 0, st,
                               (const float*)p.part_o, (const float*)p.part_ml, p.plan, p.hq, p.out));
    B200_POST_LAUNCH();
  }
  return 0;
}

template <typename T>
static int launch(const Params<T>& p, cudaStream_t st) {
  CUtensorMap mk, mv;
  const bool bf16 = std::is_same<T, __nv_bfloat16>::value;
  const uint64_t cols = (uint64_t)p.hkv * kD;
  if (int rc = get_tensor_map_2d(&mk, p.k_cache, p.num_slots, cols, cols * 2, 64, 1, bf16)) return rc;
  if (int rc = get_tensor_map_2d(&mv, p.v_cache, p.num_slots, cols, cols * 2, 64, 1, bf16)) return rc;
  CUtensorMap bk = mk, bv = mv;
  if (p.box_rows > 0) {
    if (int rc = get_tensor_map_2d(&bk, p.k_cache, p.num_slots, cols, cols * 2, 64, p.box_rows, bf16)) return rc;
    if (int rc = get_tensor_map_2d(&bv, p.v_cache, p.num_slots, cols, cols * 2, 64, p.box_rows, bf16)) return rc;
  }
  switch (p.hq / p.hkv) {
    case 1: return launch_g<T, 1>(p, mk, mv, bk, bv, st);
    case 2: return launch_g<T, 2>(p, mk, mv, bk, bv, st);
    case 3: return launch_g<T, 3>(p, mk, mv, bk, bv, st);
    case 4: return launch_g<T, 4>(p, mk, mv, bk, bv, st);
    case 5: return launch_g<T, 5>(p, mk, mv, bk, bv, st);
    case 6: return launch_g<T, 6>(p, mk, mv, bk, bv, st);
    case 7: return launch_g<T, 7>(p, mk, mv, bk, bv, st);
    case 8: return launch_g<T, 8>(p, mk, mv, bk, bv, st);
    default:
      set_error("attn_decode: GQA group size %d not supported (1..8)", p.hq / p.hkv);
      return 1;
  }
}

}  // namespace dtc

extern std::atomic<int> g_decode_fused_combine;
extern std::atomic<int> g_decode_early_kv;
bool decode_plan_is_unsplit(int bs, int num_kv_heads, int ctas);  // metadata.cu

// entry used by b200_attn_decode (attn_decode.cu)
int launch_decode_tc(const void* q, int64_t q_rs, const void* k, int64_t k_rs, const void* v,
                     int64_t v_rs, void* k_cache, void* v_cache, const int32_t* out_loc,
                     const int32_t* slot_table, int64_t st_stride, const int32_t* seq_lens,
                     const int32_t* plan, int bs, int hq, int hkv, int64_t num_slots, int page_size,
                     float scale_log2, void* out, float* part_o, float* part_ml, int* counters,
                     int dtype, cudaStream_t st, int fuse, const void* qw, const void* kw, float eps,
                     const int32_t* positions, const float* cos_sin) {
  // A batch the plan policy leaves unsplit needs no combine pass: run the in-kernel merge (a no-op
  // then; still correct for a foreign plan that does split) and skip the combine launch.
  int fused = g_decode_fused_combine.load();
  if (fused == 2) fused = decode_plan_is_unsplit(bs, hkv, 2 * num_sms()) ? 1 : 0;
  // rows per tiled TMA box: largest power of two <= min(page_size, 64) that divides page_size
  int box_rows = 0;
  if (page_size >= 8) {
    box_rows = 64;
    while (box_rows > 8 && (page_size % box_rows) != 0) box_rows >>= 1;
    if (page_size % box_rows != 0) box_rows = 0;
  }
  B200_CHECK_ARG(num_slots > 0 && num_slots < (1ll << 31), "attn_decode: bad num_slots %lld",
                 (long long)num_slots);
  // K/V streaming ahead of the predecessor: only for launches that are being captured into a graph
  int early = 0;
  if (g_decode_early_kv.load()) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs == cudaStreamCaptureStatusActive) early = 1;
  }
  B200_CHECK_ARG(st_stride % 4 == 0 && ((uintptr_t)slot_table % 16) == 0,
                 "attn_decode: slot table rows must be 16-byte aligned");
#define RUN(T_)                                                                                   \
  dtc::Params<T_> p{(const T_*)q, q_rs, (const T_*)k, k_rs, (const T_*)v, v_rs, (T_*)k_cache,     \
                    (T_*)v_cache, out_loc, slot_table, st_stride, seq_lens, plan, bs, hq, hkv,    \
                    (int)num_slots, box_rows, fused, scale_log2, (T_*)out,                        \
                    part_o, part_ml, counters, early, fuse, (const T_*)qw, (const T_*)kw, eps, positions, cos_sin};  \
  return dtc::launch<T_>(p, st)
  if (dtype == B200_DTYPE_BF16) {
    RUN(__nv_bfloat16);
  }
  RUN(__half);
#undef RUN
}

}  // namespace b200
