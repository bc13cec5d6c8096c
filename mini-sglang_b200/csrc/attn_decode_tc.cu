// Hopper-native batched decode: TMA -> 128B-swizzled smem -> wgmma (register accumulators).
//
// Replaces store_kv + BatchDecodeWithPagedKVCacheWrapper.run (python/minisgl/attention/fi.py:185-188)
// with one persistent launch (+ the split-KV combine).  HBM-bound; algorithmic bytes as in
// attn_decode_bringup.cu.  One CTA per SM, 320 threads, warp-specialised:
//
//   warps 0-3 producers, 3-stage rings of 32 KB K and 32 KB V tiles (two 64-column halves of a
//            128-key tile), data lands directly in the 128-byte-swizzled layout wgmma consumes.
//            * page_size >= 8 ("box mode", warp 0 = K, warp 1 = V): the slots of a page are contiguous
//              rows of the pool, so one tiled TMA box of min(page_size, 64) rows x 128 B is issued per
//              page piece -- 4 instructions per tile and half at page_size 64.  The piece holding the
//              end of the KV range is loaded as 8-row boxes up to its last valid row, and pieces past
//              the end are not loaded at all, so no more than 7 rows past the end come from HBM.
//            * page_size < 8 ("row mode", warps 0,1 = K keys 0-63 / 64-127, warps 2,3 = V): a warp-wide
//              cp.async gather, 16 bytes per lane, two 256-byte token rows per instruction (gather_part);
//              rows past the end of the KV range are zero filled and never read, so stale pool memory is
//              never multiplied in.  Every producer lane arrives on the stage's full barrier once its copies
//              have landed (cp.async.mbarrier.arrive.noinc: 64 arrivals, no transaction bytes), and every
//              consumer thread fences the generic-proxy writes for the tensor core after its wait.
//   warps 4-7 one consumer warpgroup: S^T[128 keys x N] = K_tile . Q^T and O^T[128 dims x N] += V_tile^T . P^T
//            as wgmma m64nNk16 (two 64-row blocks each): the keys / head dims fill M and the query heads of
//            the GQA group sit in N -- N = 8 for groups of 1-8, N = 16 for groups of 9-16, chosen at compile
//            time from the group size -- so no tensor-core row is spent on padding.  Softmax on the score
//            fragments (tile max across the four warps through smem + a named barrier), P^T to smem as the
//            16-bit B operand, O^T stays in registers with the online-softmax rescale.
//   warp 8   Q loader: the group's q rows -> swizzled smem operand (double buffered across units).
//   warp 9   split-KV combiner: the last-arriving chunk of a (request, kv head) merges the partials.
//
// Every unit is one (request, chunk, kv head): all G query heads of the group share each K/V tile, so the K/V
// bytes of a launch do not depend on G.
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
#include "attn.cuh"
#include "combine.cuh"
#include "qknorm_rope.cuh"

#include <type_traits>

namespace b200 {
namespace dtc {

using namespace sm90;

constexpr int kD = kHeadDim;
constexpr int kStages = 3;
constexpr int kThreads = 320;
constexpr int kWarpQ = 8, kWarpCombine = 9;
constexpr int kMaxGroup = 16;               // largest GQA group (query heads per kv head) of the kernel
template <int G>
constexpr int kNOf = G <= 8 ? 8 : 16;       // wgmma N: the query heads of the group, padded
constexpr int kUnitSlotBytes = 40, kMaxUnitsSmem = 96;  // per-CTA work units decoded once into smem

template <int N>
struct Smem {
  static_assert(N == 8 || N == 16, "wgmma N of the decode kernel is 8 or 16");
  static constexpr int kQHalfBytes = N * 128;            // one 64-column half of [N rows x 128 B], 128B-swizzled
  static constexpr int kQBufBytes = 2 * kQHalfBytes;
  static constexpr int kPBufBytes = N * kKvTileRows * 2;  // P^T [N x 128] 16-bit, no-swizzle K-major
  // fused mode: roped (q heads, new k) rows in flight to the epilogue, up to N q heads + the k row of 128 x 16 bit.
  // N = 16 keeps three slots instead of four: with the doubled Q, P^T and reduction buffers and 17-row slots, four
  // would need 232704 B with the alignment slack, over the 232448 B a CTA may have.  The ring only lets the Q
  // loader run ahead of the consumers' epilogues; three slots still cover its two-deep Q ring plus one unit.  The
  // unit cache keeps its 96 slots, so no batch moves onto the slower decode-from-global path.
  static constexpr int kEpiSlots = N == 8 ? 4 : 3;
  static constexpr int kEpiSlotBytes = (N + 1) * kD * 2;
  // offsets from the 1024-aligned base
  static constexpr int kring = 0;                          // K tiles, released right after QK
  static constexpr int vring = kStages * kKvTileBytes;     // V tiles, released after PV
  static constexpr int qbuf = 2 * kStages * kKvTileBytes;
  static constexpr int pbuf = qbuf + 2 * kQBufBytes;
  static constexpr int bars = pbuf + kPBufBytes;           // 32 mbarriers
  static constexpr int red = bars + 32 * 8;                // floats: tile max [4][N], [2][4][N] row sums, [2][4][N] new-token dots
  static constexpr int units = red + 20 * N * 4;           // decoded work units
  static constexpr int epi = units + kMaxUnitsSmem * kUnitSlotBytes;  // fused mode: kEpiSlots x [N + 1][128] 16-bit
  static constexpr int total = epi + kEpiSlots * kEpiSlotBytes;
};
static_assert(Smem<8>::total + 1024 <= 232448, "decode kernel shared memory exceeds the 227 KB per-CTA limit");
static_assert(Smem<16>::total + 1024 <= 232448, "decode kernel shared memory exceeds the 227 KB per-CTA limit");
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
  int exact_tail;  // box mode: the box holding the end of a range loads only its valid rows (8-row granules)
  int fused_combine;  // 1: last-arriving unit merges the split-KV partials in this launch
  float scale_log2;
  T* out;
  float* part_o;
  float* part_ml;
  int* counters;  // [bs][hkv] split-KV arrival counters, zero between launches
  // fused pre-attention (fuse = 1): q / k_new are raw; norm weights may be NULL (models without qk-norm)
  int early;  // 1: captured launch -- K/V producers do not wait for the predecessor (see the kernel prologue)
  int fuse;
  const T* qw;
  const T* kw;
  float eps;
  const int32_t* positions;
  const float* cos_sin;  // fp32 [max_pos][128] = cos | sin
  TraceArgs trace;       // read by the kTrace = true instantiation only
};

struct Unit {
  int r, c, h, n_chunks, kv_len, kv_begin, kv_end_tc, n_tiles;
  int last_chunk;
};

// Work unit `pos` of the size-sorted order (metadata.cu): the hkv heads of an item are adjacent positions
// (neighbouring CTAs stream the same token rows).
__device__ __forceinline__ Unit get_unit(int pos, int hkv, int chunk_tokens, const int32_t* order,
                                         const int32_t* seq_lens) {
  Unit u;
  const int item = pos / hkv;
  u.h = pos - item * hkv;
  const PlanEntry e = unpack_plan_entry(order[item]);
  u.r = e.r;
  u.c = e.c;
  u.n_chunks = e.n_chunks;
  u.kv_len = seq_lens[u.r];
  u.kv_begin = u.c * chunk_tokens;
  const int kv_end = min(u.kv_len, u.kv_begin + chunk_tokens);
  u.last_chunk = (u.c == u.n_chunks - 1);
  u.kv_end_tc = u.last_chunk ? kv_end - 1 : kv_end;  // the appended token is handled on CUDA cores
  const int n = u.kv_end_tc - u.kv_begin;
  u.n_tiles = n > 0 ? (n + kKvTileRows - 1) / kKvTileRows : 0;
  return u;
}

// wgmma m64nNk16 with both operands in shared memory, N = 8 or 16
template <int N, int kTransA, typename T>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d, T* tsel) {
  if constexpr (N == 8)
    wgmma_m64n8k16_ss<kTransA>(d, da, db, scale_d, tsel);
  else
    wgmma_m64n16k16_ss<kTransA>(d, da, db, scale_d, tsel);
}

// kTrace: each warp records its events into p.trace (attn.cuh); the false instantiation is the product kernel.
// kRows: row mode (p.box_rows == 0), a separate instantiation so that box mode's tile loop carries none of it.
template <typename T, int G, bool kTrace, bool kRows>
__global__ void __launch_bounds__(kThreads, 1)
attn_decode_tc_kernel(const Params<T> p, const __grid_constant__ CUtensorMap box_k,
                      const __grid_constant__ CUtensorMap box_v,
                      const __grid_constant__ CUtensorMap tail_k,
                      const __grid_constant__ CUtensorMap tail_v) {
  constexpr int N = kNOf<G>;
  using Smem = dtc::Smem<N>;
  constexpr int kE = N / 4;  // accumulator columns (query heads) per thread: h0, h0+1 and, at N = 16, h0+8, h0+9
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B-swizzled tiles
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid / kWarp, lane = tid % kWarp;
  auto bar = [&](int i) { return sbase + Smem::bars + i * 8; };
  float* red = reinterpret_cast<float*>(smem + Smem::red);
  WarpTrace<kTrace, kDecodeWarps> tr(p.trace);
  tr.begin();

  // ---------------------------------------------------------------- setup that touches no global memory
  // zero the Q operand buffers whose padding rows (heads >= G) are never written again
  for (int i = tid; i < (2 * Smem::kQBufBytes) / 16; i += kThreads)
    reinterpret_cast<uint4*>(smem + Smem::qbuf)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    // full: box mode, lane 0's expect_tx; row mode, every lane of the two warps that gather the tile
    const uint32_t n_fill = kRows ? 2 * kWarp : 1;
    for (int s = 0; s < kStages; ++s) {
      mbar_init(bar(kFullK + s), n_fill);
      mbar_init(bar(kEmptyK + s), 4);  // one elected arrival per consumer warp
      mbar_init(bar(kFullV + s), n_fill);
      mbar_init(bar(kEmptyV + s), 4);
    }
    for (int b = 0; b < kFinRing; ++b) {
      mbar_init(bar(kFinFull + b), 128);
      mbar_init(bar(kFinEmpty + b), 1);
    }
    for (int b = 0; b < Smem::kEpiSlots; ++b) {
      mbar_init(bar(kEpiFull + b), 1);
      mbar_init(bar(kEpiEmpty + b), 1);
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(bar(kQFull + b), 1);
      mbar_init(bar(kQEmpty + b), 4);
    }
    fence_barrier_init();
    if constexpr (!kRows) {  // row mode passes no tensor maps
      prefetch_tensormap(&box_k);
      prefetch_tensormap(&box_v);
      prefetch_tensormap(&tail_k);
      prefetch_tensormap(&tail_v);
    }
  }
  // PDL: everything above may overlap the tail of the previous kernel in the stream.
  //  * p.early == 0 (eager launches): wait here -- from here on the results of every kernel before this one
  //    (in particular the metadata kernel's plan / seq_lens / slot table) are complete and visible.
  //  * p.early == 1 (launch captured into a CUDA graph): the metadata was written BEFORE the graph started
  //    (prepare_for_replay), and the K/V rows this launch streams belong to this layer's pool slice, which
  //    no other kernel of the graph writes -- so only the roles that consume the predecessor's outputs
  //    (Q loader: q / k_new; consumer warps: v_new, out_loc operands, output / partial stores; combiner)
  //    wait, while the K/V producers start streaming K/V at once: prologue, pipeline fill and the
  //    predecessor's tail (or a small kernel in between, e.g. the TP all-reduce) overlap.
  if (!p.early) pdl_wait();
  pdl_launch_dependents();
  if (!p.early) tr.ev(kEvPdlWait, 0);
  const int chunk_tokens = p.plan[0];
  tr.header(kTracePhaseDecode, p.bs, p.hq, p.hkv, p.box_rows, p.plan[1] != p.bs);
  const int32_t* order = p.plan + kPlanHeader + p.bs + 1;
  const auto units = deal_units<Unit, kUnitSlotBytes, kMaxUnitsSmem>(
      smem + Smem::units, p.plan[1] * p.hkv,
      [&](int pos) { return get_unit(pos, p.hkv, chunk_tokens, order, p.seq_lens); });

  // ---------------------------------------------------------------- one-time setup
  units.stage(tid, kThreads);
  fence_proxy_async_smem();  // zero-fill above must be visible to wgmma operand reads
  __syncthreads();
  if (warp < 4) {
    // ============================================================ K/V producers
    // K and V travel in separate rings (a K tile is dead as soon as QK^T has completed, a V
    // tile only after PV), so each has its own producers: box mode warp 0 = K, warp 1 = V;
    // row mode warps 0,1 = K rows 0-63 / 64-127, warps 2,3 = V.
    const int rb = p.box_rows;
    const int kind = rb > 0 ? warp : (warp >> 1);  // 0 = K, 1 = V
    if (rb > 0 && warp >= 2) {
      // box mode needs a handful of instructions per tile: two warps are plenty
    } else {
      const CUtensorMap* bmap = kind == 0 ? &box_k : &box_v;
      const int full0 = kind == 0 ? kFullK : kFullV, empty0 = kind == 0 ? kEmptyK : kEmptyV;
      const uint32_t ring = sbase + (kind == 0 ? Smem::kring : Smem::vring);
      RingCursor<kStages> kv;
      for (int k = 0; k < units.n_rounds; ++k) {
        const Unit u = units.at(k);
        if constexpr (kTrace)
          if (!units.none(u)) tr.ev(kEvUnitBegin, k);
        if (u.n_tiles <= 0) {
          if constexpr (kTrace)
            if (!units.none(u)) tr.ev(kEvUnitEnd, k);
          continue;
        }
        const int32_t* slots = p.slot_table + (int64_t)u.r * p.st_stride;
        const int col0 = u.h * kD;
        if constexpr (kRows) {
          // ---- row mode: this warp gathers keys 64 part .. 64 part + 63 of every tile
          const int part = warp & 1;
          const T* src = (kind == 0 ? p.k_cache : p.v_cache) + col0;
          auto load_slots = [&](int t) {
            return kv_slot_group(slots, u.kv_begin + t * kKvTileRows + part * 64 + 4 * (lane & 15), u.kv_end_tc,
                                 p.num_slots);
          };
          int4 nxt = load_slots(0);
          for (int t = 0; t < u.n_tiles; ++t, kv.advance()) {
            const int4 cur = nxt;
            if (t + 1 < u.n_tiles) nxt = load_slots(t + 1);
            tr.ev(kEvEmptyWait, t);
            kv.wait_empty(bar(empty0));
            tr.ev(kEvEmptyDone, t);
            gather_part(ring + kv.stage() * kKvTileBytes, part, src, p.hkv * kD, cur, p.num_slots, 64, lane);
            cp_async_mbar_arrive_noinc(bar(full0 + kv.stage()));
            tr.ev(kEvIssued, t);
          }
        } else {
          // ---- box mode
          const KvLane L = KvLane::box(lane, rb);
          const int n_instr = KvLane::box_lanes(rb);  // <= 32
          const CUtensorMap* tmap = kind == 0 ? &tail_k : &tail_v;
          for (int t = 0; t < u.n_tiles; ++t, kv.advance()) {
            const int pb = u.kv_begin + t * kKvTileRows + L.row;
            // Rows this lane loads.  Exact tail: a box wholly inside the range is one rb-row box, the box
            // holding the end of the range is cut to its valid rows rounded up to 8-row boxes, and a box
            // wholly past the end is not issued.  Otherwise every box is loaded whole: one reaching past
            // the end reads the rest of its page from HBM, one wholly past the end gets out-of-range rows.
            // Rows of the stage that are not loaded keep older contents: the consumer warps mask those K
            // rows by position and zero those V rows before PV.
            const int left = u.kv_end_tc - pb;
            int rows = 0;
            if (lane < n_instr) rows = !p.exact_tail ? rb : (left <= 0 ? 0 : min(rb, (left + 7) & ~7));
            // slot of the box's first row, loaded before the wait so its latency overlaps
            int first_slot = p.num_slots;
            if (lane < n_instr && left > 0) first_slot = __ldg(slots + pb);
            // the stage's transaction bytes are exactly the rows the lanes issue below
            const uint32_t tx_bytes = __reduce_add_sync(0xffffffffu, (uint32_t)rows) * 128u;
            tr.ev(kEvEmptyWait, t);
            kv.wait_empty(bar(empty0));
            tr.ev(kEvEmptyDone, t);
            const uint32_t fb = bar(full0 + kv.stage());
            if (lane == 0) mbar_arrive_expect_tx(fb, tx_bytes);
            __syncwarp();
            if (rows > 0) {
              const uint32_t dst = L.dst(ring, kv.stage());
              const int col = L.col(col0);
              if (rows == rb) {
                tma_load_2d(dst, bmap, fb, col, first_slot);
              } else {
                // the rows of a box are consecutive slots of one page
                for (int r = 0; r < rows; r += 8) tma_load_2d(dst + r * 128, tmap, fb, col, first_slot + r);
              }
            }
            tr.ev(kEvIssued, t);
          }
        }
        tr.ev(kEvUnitEnd, k);
      }
    }
  } else if (warp == kWarpQ) {
    // ============================================================ Q loader
    if (p.early) {
      pdl_wait();
      tr.ev(kEvPdlWait, 0);
    }
    RingCursor<2> qr;
    RingCursor<Smem::kEpiSlots> er;
    for (int k = 0; k < units.n_rounds; ++k) {
      const Unit u = units.at(k);
      if (units.none(u)) continue;
      tr.ev(kEvUnitBegin, k);
      const bool need_q = u.n_tiles > 0;                 // the tensor core needs the Q operand
      const bool need_epi = p.fuse && u.last_chunk;      // the epilogue needs roped q / k rows
      if (!need_q && !need_epi) {
        tr.ev(kEvUnitEnd, k);
        continue;
      }
      const uint32_t qb = qr.stage(), es = er.stage();
      if (need_q) qr.wait_empty(bar(kQEmpty));
      if (need_epi) er.wait_empty(bar(kEpiEmpty));
      uint8_t* qdst = smem + Smem::qbuf + qb * Smem::kQBufBytes;
      if (!p.fuse) {
        for (int idx = lane; idx < G * 16; idx += kWarp) {
          const int g = idx >> 4, cc = idx & 15;
          const Vec8 v = *reinterpret_cast<const Vec8*>(p.q + (int64_t)u.r * p.q_rs +
                                                        (int64_t)(u.h * G + g) * kD + cc * 8);
          *reinterpret_cast<Vec8*>(qdst + (cc >> 3) * Smem::kQHalfBytes + sw128_offset(g, cc & 7)) = v;
        }
      } else {
        // per-head RMSNorm + RoPE on 16-lane groups, two rows per pass: the G q heads of the group and,
        // for the unit that owns the new token, its k row (row index G).  Uniform trip count: the
        // shuffles inside qknorm_rope_lanes need the whole warp.
        uint8_t* edst = smem + Smem::epi + es * Smem::kEpiSlotBytes;
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
            if (!is_k && need_q) *reinterpret_cast<Vec8*>(qdst + (cc >> 3) * Smem::kQHalfBytes + sw128_offset(g, cc & 7)) = rv;
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
      tr.ev(kEvQReady, k);
      if (need_q) qr.advance();
      if (need_epi) er.advance();
      tr.ev(kEvUnitEnd, k);
    }
  } else if (warp >= 4 && warp < 8) {
    // ============================================================ consumer warpgroup (128 threads)
    if (p.early) {
      pdl_wait();
      tr.ev(kEvPdlWait, 0);
    }
    constexpr bool kTransV = true;  // A = V^T: the head dims (M) are the contiguous axis of a V tile
    T* const tsel = nullptr;        // selects the bf16 / fp16 wgmma overload
    const int ct = tid - 128;       // 0..127
    const int cw = warp - 4;        // warp of the group
    // accumulator fragment (see sm90.cuh): element i of 64-row block mb is row mb*64 + r0 + ((i>>1)&1)*8,
    // column (i>>2)*8 + h0 + (i&1).  Rows are keys (S^T) or head dims (O^T), columns are the group's query
    // heads.  A thread owns kE columns; column slot e is column col_of(e), fragment element i is in slot_of(i).
    const int r0 = 16 * cw + (lane >> 2), h0 = 2 * (lane & 3);
    auto row_of = [&](int mb, int i) { return mb * 64 + r0 + (((i >> 1) & 1) << 3); };
    auto col_of = [&](int e) { return (e >> 1) * 8 + h0 + (e & 1); };
    auto slot_of = [](int i) { return ((i >> 2) << 1) | (i & 1); };
    float* red_max = red;            // [4 warps][N heads]
    float* red_sum0 = red + 4 * N;   // [2 parity][4][N]
    float* red_new0 = red + 12 * N;  // [2 parity][4][N]
    RingCursor<kStages> kv;
    RingCursor<2> qr;
    RingCursor<kFinRing> fr;
    RingCursor<Smem::kEpiSlots> er;
    uint32_t unit_par = 0;
    for (int k = 0; k < units.n_rounds; ++k) {
      const Unit u = units.at(k);
      if (units.none(u)) continue;
      tr.ev(kEvUnitBegin, k);
      float acc[2][N / 2], l_thr[kE], m_run[kE];
#pragma unroll
      for (int e = 0; e < kE; ++e) {
        l_thr[e] = 0.f;
        m_run[e] = -INFINITY;
      }
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[mb][i] = 0.f;
      // operands of the appended token's score / value (x = mb*2 + (i>>1) indexes this thread's four dims):
      // issue the loads now, use them in the epilogue -- their latency hides behind the tile loop
      float q_new[kE][4], kn[4], vn[4];
      int app_loc = 0;
      Vec8 app_x = Vec8{{0u, 0u, 0u, 0u}};
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        kn[x] = vn[x] = 0.f;
#pragma unroll
        for (int e = 0; e < kE; ++e) q_new[e][x] = 0.f;
      }
      if (u.last_chunk) {
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          const int dim = row_of(x >> 1, (x & 1) << 1);
          if (!p.fuse) {  // fused mode: roped q / k come from the Q loader's ring in the epilogue
#pragma unroll
            for (int e = 0; e < kE; ++e)
              if (col_of(e) < G)
                q_new[e][x] = DTypeTraits<T>::to_float(p.q[(int64_t)u.r * p.q_rs + (int64_t)(u.h * G + h0 + (e & 1) + (e >> 1) * 8) * kD + dim]);
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
        const uint32_t qb = qr.stage();
        qr.wait_full(bar(kQFull));
        tr.ev(kEvQReady, k);
        const uint32_t qa = sbase + Smem::qbuf + qb * Smem::kQBufBytes;
        for (int j = 0; j < u.n_tiles; ++j, kv.advance()) {
          const uint32_t stage = kv.stage();
          // ---- S^T = K_tile . Q^T: A = K rows (K-major, 128B swizzle), B = Q rows (K-major, 8-row atoms 1024 B apart)
          kv.wait_full(bar(kFullK));
          // Row mode: the tile was written by cp.async, generic-proxy writes, and wgmma reads it through the async
          // proxy.  The full barrier's phase completes only after every copy of the tile has landed (each producer
          // lane's arrival waits for its own copies), so the writes happen before this thread's wait returns; the
          // fence then orders them before this thread's async-proxy reads.  The producers cannot fence: they never
          // wait for their copies.  (Overwriting a slot after the release below needs no fence: wgmma_wait0 has
          // completed the reads before the release, and the next copies are issued after it.)
          if constexpr (kRows) fence_proxy_async_smem();
          tr.ev(kEvKFull, j);
          const uint32_t kb = sbase + Smem::kring + stage * kKvTileBytes;
          float s[2][N / 2];
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int i = 0; i < N / 2; ++i) s[mb][i] = 0.f;
          wgmma_fence();
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
              const uint64_t da = make_smem_desc(kb + mb * 8192 + (kk >> 2) * kKvHalfBytes + (kk & 3) * 32, 16, 1024, kLayoutSW128);
              const uint64_t db = make_smem_desc(qa + (kk >> 2) * Smem::kQHalfBytes + (kk & 3) * 32, 16, 1024, kLayoutSW128);
              wgmma_ss<N, 0>(s[mb], da, db, kk > 0, tsel);
            }
          wgmma_commit();
          wgmma_wait0();
          tr.ev(kEvQK, j);
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(bar(kEmptyK + stage));                      // the K tile is dead
            if (j + 1 == u.n_tiles) mbar_arrive(bar(kQEmpty + qb));  // last QK of the unit
          }
          const int n_valid = u.kv_end_tc - (u.kv_begin + j * kKvTileRows);  // >= 1
          if (p.box_rows > 0 && n_valid < kKvTileRows) {
            // box mode, last tile of the range: the V rows past the end hold the rest of the page or
            // an earlier tile of this stage (possibly NaN bit patterns): zero them so that 0 * garbage
            // cannot reach the output
            kv.wait_full(bar(kFullV));
            uint8_t* vt = smem + Smem::vring + stage * kKvTileBytes;
            for (int idx = ct; idx < (kKvTileRows - n_valid) * 16; idx += 128) {
              const int row = n_valid + (idx >> 4), c16 = idx & 15;
              *reinterpret_cast<uint4*>(vt + (c16 >> 3) * kKvHalfBytes + row * 128 + (c16 & 7) * 16) = make_uint4(0, 0, 0, 0);
            }
            fence_proxy_async_smem();
          }
          // ---- online softmax: per head (column) max over the 128 keys of the tile
          float mx[kE];
#pragma unroll
          for (int e = 0; e < kE; ++e) mx[e] = -INFINITY;
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int i = 0; i < N / 2; ++i) {
              const float v = row_of(mb, i) < n_valid ? s[mb][i] * p.scale_log2 : -INFINITY;
              s[mb][i] = v;
              mx[slot_of(i)] = fmaxf(mx[slot_of(i)], v);
            }
#pragma unroll
          for (int e = 0; e < kE; ++e) {
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 4));
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 8));
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 16));
          }
          if (lane < 4) {
#pragma unroll
            for (int e = 0; e < kE; ++e) red_max[cw * N + col_of(e)] = mx[e];
          }
          named_bar_sync(1, 128);
          float alpha[kE], psum[kE];
#pragma unroll
          for (int e = 0; e < kE; ++e) {
            const int hh = col_of(e);
            const float mt = fmaxf(fmaxf(red_max[hh], red_max[N + hh]), fmaxf(red_max[2 * N + hh], red_max[3 * N + hh]));
            const float m_new = fmaxf(m_run[e], mt);  // finite: every tile has >= 1 valid key
            alpha[e] = fast_exp2(m_run[e] - m_new);
            m_run[e] = m_new;
            psum[e] = 0.f;
          }
          // P^T [head][key] as 8x8 core matrices (no swizzle, K-major): key chunks of 8 are 128 B apart, and at
          // N = 16 heads 8-15 follow heads 0-7 as a second [8 x 128] block (kPBlockBytes)
          uint8_t* pdst = smem + Smem::pbuf;
          constexpr int kPBlockBytes = 8 * kKvTileRows * 2;
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int i = 0; i < N / 2; ++i) {
              const int key = row_of(mb, i), hh = h0 + (i & 1), e = slot_of(i);
              const float pv = fast_exp2(s[mb][i] - m_run[e]);
              psum[e] += pv;
              *reinterpret_cast<T*>(pdst + (i >> 2) * kPBlockBytes + (key >> 3) * 128 + hh * 16 + (key & 7) * 2) =
                  DTypeTraits<T>::from_float(pv);
              acc[mb][i] *= alpha[e];
            }
#pragma unroll
          for (int e = 0; e < kE; ++e) l_thr[e] = l_thr[e] * alpha[e] + psum[e];
          fence_proxy_async_smem();  // P^T (and zeroed V rows) visible to the tensor core
          named_bar_sync(1, 128);    // every warp's P^T is written; the tile maxima may be overwritten
          tr.ev(kEvSoftmax, j);
          // ---- O^T += V_tile^T . P^T: A = V rows read MN-major, B = P^T (K-major, no swizzle)
          kv.wait_full(bar(kFullV));
          if constexpr (kRows) fence_proxy_async_smem();  // as for the K tile
          tr.ev(kEvVFull, j);
          const uint32_t vb = sbase + Smem::vring + stage * kKvTileBytes;
          const uint32_t pb = sbase + Smem::pbuf;
          wgmma_fence();
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
              // 16 keys = two 8-key swizzle atoms of 1024 B; dims 64..127 in the second half (+16 KB)
              const uint64_t da = make_smem_desc(vb + mb * kKvHalfBytes + kk * 2048, kKvHalfBytes, 1024, kLayoutSW128);
              // P^T: LBO = 128 B between key chunks; SBO = the head-block stride (unused at N = 8: one block)
              const uint64_t db = make_smem_desc(pb + kk * 256, 128, N == 8 ? 1024 : kPBlockBytes, kLayoutNone);
              wgmma_ss<N, kTransV ? 1 : 0>(acc[mb], da, db, 1u, tsel);
            }
          wgmma_commit();
          wgmma_wait0();
          tr.ev(kEvPV, j);
          __syncwarp();
          if (lane == 0) mbar_arrive(bar(kEmptyV + stage));
        }
        qr.advance();
      }
      tr.ev(kEvEpiBegin, k);

      // ---- unit epilogue on CUDA cores: row sums, the appended token (score, value, pool append), output.
      // Reduction scratch double buffered by unit parity: the next unit may write its slots while
      // stragglers still read this unit's (every unit passes a named barrier in between).
      float* red_sum = red_sum0 + unit_par * (4 * N);
      float* red_new = red_new0 + unit_par * (4 * N);
      unit_par ^= 1;
      const bool epi = p.fuse && u.last_chunk;
      const uint32_t es = er.stage();
      if (epi) {
        // fused mode: the Q loader left the roped q rows of the group and the roped new k row in the ring
        er.wait_full(bar(kEpiFull));
        er.advance();
        const uint8_t* esrc = smem + Smem::epi + es * Smem::kEpiSlotBytes;
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          const int dim = row_of(x >> 1, (x & 1) << 1);
#pragma unroll
          for (int e = 0; e < kE; ++e)
            if (col_of(e) < G) q_new[e][x] = DTypeTraits<T>::to_float(*reinterpret_cast<const T*>(esrc + col_of(e) * (kD * 2) + dim * 2));
          kn[x] = DTypeTraits<T>::to_float(*reinterpret_cast<const T*>(esrc + G * (kD * 2) + dim * 2));
        }
        if (ct < 16) app_x = *reinterpret_cast<const Vec8*>(esrc + G * (kD * 2) + ct * 16);
      }
#pragma unroll
      for (int e = 0; e < kE; ++e) {
        float ls = l_thr[e], sn = 0.f;
        if (u.last_chunk) sn = (q_new[e][0] * kn[0] + q_new[e][1] * kn[1]) + (q_new[e][2] * kn[2] + q_new[e][3] * kn[3]);
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          ls += __shfl_xor_sync(0xffffffffu, ls, o);
          sn += __shfl_xor_sync(0xffffffffu, sn, o);
        }
        if (lane < 4) {
          red_sum[cw * N + col_of(e)] = ls;
          red_new[cw * N + col_of(e)] = sn;
        }
      }
      named_bar_sync(1, 128);
      if (epi && ct == 0) mbar_arrive(bar(kEpiEmpty + es));  // every thread has read its ring values
      float l_tot[kE];
#pragma unroll
      for (int e = 0; e < kE; ++e) {
        const int hh = col_of(e);
        l_tot[e] = red_sum[hh] + red_sum[N + hh] + red_sum[2 * N + hh] + red_sum[3 * N + hh];
      }
      if (u.last_chunk) {
#pragma unroll
        for (int e = 0; e < kE; ++e) {
          const int hh = col_of(e);
          const float s_new = (red_new[hh] + red_new[N + hh] + red_new[2 * N + hh] + red_new[3 * N + hh]) * p.scale_log2;
          const float m_new = fmaxf(m_run[e], s_new);
          const float a = fast_exp2(m_run[e] - m_new);
          const float pnew = fast_exp2(s_new - m_new);
          const int i0 = (e >> 1) * 4 + (e & 1);  // fragment elements of column slot e: i0 (row r0), i0 + 2 (row r0 + 8)
#pragma unroll
          for (int mb = 0; mb < 2; ++mb) {
            acc[mb][i0] = acc[mb][i0] * a + pnew * vn[mb * 2];
            acc[mb][i0 + 2] = acc[mb][i0 + 2] * a + pnew * vn[mb * 2 + 1];
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
        float inv[kE];
#pragma unroll
        for (int e = 0; e < kE; ++e) inv[e] = 1.f / l_tot[e];
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
          for (int i = 0; i < N / 2; ++i)
            if (col_of(slot_of(i)) < G)
              p.out[((int64_t)u.r * p.hq + u.h * G + h0 + (i & 1) + (i >> 2) * 8) * kD + row_of(mb, i)] =
                  DTypeTraits<T>::from_float(acc[mb][i] * inv[slot_of(i)]);
        tr.ev(kEvEpiEnd, k);
      } else {
        const int64_t base = ((int64_t)u.r * kMaxSplits + u.c) * p.hq + u.h * G;
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
          for (int i = 0; i < N / 2; ++i)
            if (col_of(slot_of(i)) < G) p.part_o[(base + h0 + (i & 1) + (i >> 2) * 8) * kD + row_of(mb, i)] = acc[mb][i];
        if (cw == 0 && lane < 4) {
          // m_run / l_tot of a head are uniform across threads; lanes 0-3 of warp 0 store their kE heads
#pragma unroll
          for (int e = 0; e < kE; ++e)
            if (col_of(e) < G) {
              p.part_ml[(base + h0 + (e & 1) + (e >> 1) * 8) * 2 + 0] = m_run[e];
              p.part_ml[(base + h0 + (e & 1) + (e >> 1) * 8) * 2 + 1] = l_tot[e];
            }
        }
        tr.ev(kEvEpiEnd, k);
        // ---- hand the unit to the combiner warp (asynchronous split-KV merge): the consumer warps
        // only pay an mbarrier arrive; the release/acquire pair orders the partial stores above
        // before the combiner's device-scope fence + arrival counter.
        if (p.fused_combine) {
          fr.wait_empty(bar(kFinEmpty));
          mbar_arrive(bar(kFinFull + fr.stage()));
          fr.advance();
        }
      }
      tr.ev(kEvUnitEnd, k);
    }
  } else if (warp == kWarpCombine) {
    // ============================================================ split-KV combiner (one warp)
    // For every multi-chunk unit of this CTA: count in on the (request, kv head) arrival counter;
    // whoever arrives last merges all partials (flash-decoding reduction) and writes the output.
    if (p.early) {
      pdl_wait();
      tr.ev(kEvPdlWait, 0);
    }
    if (p.fused_combine) {
      RingCursor<kFinRing> fr;
      for (int k = 0; k < units.n_rounds; ++k) {
        const Unit u = units.at(k);
        if constexpr (kTrace)
          if (!units.none(u)) {
            tr.ev(kEvUnitBegin, k);
            if (u.n_chunks == 1) tr.ev(kEvUnitEnd, k);
          }
        if (units.none(u) || u.n_chunks == 1) continue;
        const uint32_t slot = fr.stage();
        fr.wait_full(bar(kFinFull));
        fr.advance();
        __threadfence();
        int last = 0;
        if (lane == 0) {
          const int old = atomicAdd(p.counters + u.r * p.hkv + u.h, 1);
          last = (old == u.n_chunks - 1);
          if (last) p.counters[u.r * p.hkv + u.h] = 0;  // zero again for the next launch
        }
        last = __shfl_sync(0xffffffffu, last, 0);
        tr.ev(last ? kEvArriveLast : kEvArrive, k);
        if (last) {
          tr.ev(kEvMergeBegin, k);
          __threadfence();  // acquire the other chunks' partials
          // Heads in passes of GB <= 8: (o, m, l, weight, 1/l) of 9-16 heads plus their prefetched partials would
          // not fit one warp's registers.  A group of 9-15 ends its last pass at head G-1, so that pass merges some
          // heads of the first one again -- with the same bits, as a head's merge reads only its own partials.
          constexpr int GB = G <= 8 ? G : 8;
#pragma unroll
          for (int pass = 0; pass < (G + GB - 1) / GB; ++pass) {
            const int g0 = min(pass * GB, G - GB);  // first head of the pass
            // The merge is pure latency (partials sit in L2, written by other SMs): every load whose address
            // is known is issued before anything is consumed -- (m, l) of all GB heads at once, then the
            // partial outputs kMergeBatch chunks x GB heads at a time.
            const int64_t b0 = ((int64_t)u.r * kMaxSplits) * p.hq + u.h * G + g0;
            float mc[GB], lc[GB];
#pragma unroll
            for (int g = 0; g < GB; ++g) {  // lane c holds (m, l) of chunk c
              mc[g] = -INFINITY;
              lc[g] = 0.f;
              if (lane < u.n_chunks) {
                const float2 ml = __ldcg(reinterpret_cast<const float2*>(p.part_ml + (b0 + (int64_t)lane * p.hq + g) * 2));
                mc[g] = ml.x;
                lc[g] = ml.y;
              }
            }
            constexpr int kMergeBatch = GB <= 2 ? 8 : (GB <= 4 ? 4 : 2);
            float4 o[GB];
            float wc[GB], inv[GB];
#pragma unroll
            for (int g = 0; g < GB; ++g) o[g] = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int c0 = 0; c0 < u.n_chunks; c0 += kMergeBatch) {
              float4 po[GB][kMergeBatch];
#pragma unroll
              for (int g = 0; g < GB; ++g)
#pragma unroll
                for (int j = 0; j < kMergeBatch; ++j)
                  po[g][j] = c0 + j < u.n_chunks
                                 ? __ldcg(reinterpret_cast<const float4*>(p.part_o + (b0 + (int64_t)(c0 + j) * p.hq + g) * kD) + lane)
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
              if (c0 == 0) {
#pragma unroll
                for (int g = 0; g < GB; ++g) {
                  const float mx = warp_max(mc[g]);
                  wc[g] = lane < u.n_chunks ? fast_exp2(mc[g] - mx) : 0.f;
                  inv[g] = 1.f / warp_sum(wc[g] * lc[g]);
                }
              }
#pragma unroll
              for (int g = 0; g < GB; ++g)
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
            for (int g = 0; g < GB; ++g) {
              typename DTypeTraits<T>::T2 lo = DTypeTraits<T>::from_float2(o[g].x * inv[g], o[g].y * inv[g]);
              typename DTypeTraits<T>::T2 hi = DTypeTraits<T>::from_float2(o[g].z * inv[g], o[g].w * inv[g]);
              uint2 pk;
              pk.x = *reinterpret_cast<uint32_t*>(&lo);
              pk.y = *reinterpret_cast<uint32_t*>(&hi);
              *reinterpret_cast<uint2*>(p.out + ((int64_t)u.r * p.hq + u.h * G + g0 + g) * kD + lane * 4) = pk;
            }
          }
          tr.ev(kEvMergeEnd, k);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(kFinEmpty + slot));
        tr.ev(kEvUnitEnd, k);
      }
    }
  }

  // ---------------------------------------------------------------- teardown
  __syncthreads();
  tr.ev(kEvEnd, 0);
  tr.finish();
}

template <typename T, int G, bool kTrace, bool kRows>
static int launch_kernel(const Params<T>& p, const CUtensorMap& bk, const CUtensorMap& bv, const CUtensorMap& tk,
                         const CUtensorMap& tv, cudaStream_t st) {
  const size_t smem = Smem<kNOf<G>>::total + 1024;
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(attn_decode_tc_kernel<T, G, kTrace, kRows>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  B200_CHECK_CUDA(launch_pdl(attn_decode_tc_kernel<T, G, kTrace, kRows>, dim3(num_sms()), dim3(kThreads), smem, st, p, bk, bv,
                             tk, tv));
  return 0;
}

template <typename T, int G>
static int launch_g(Params<T> p, const CUtensorMap& bk, const CUtensorMap& bv, const CUtensorMap& tk,
                    const CUtensorMap& tv, cudaStream_t st) {
  // a registered trace buffer with a region left selects the instrumented instantiation (same launch otherwise)
  if (trace_next_region(kTracePhaseDecode, num_sms(), &p.trace)) {
    p.trace.flags = (p.fuse ? kTraceFused : 0u) | (p.fused_combine ? kTraceInKernelCombine : 0u) | (p.early ? kTraceEarlyKv : 0u);
    if (int rc = p.box_rows == 0 ? launch_kernel<T, G, true, true>(p, bk, bv, tk, tv, st)
                                 : launch_kernel<T, G, true, false>(p, bk, bv, tk, tv, st))
      return rc;
  } else {
    if (int rc = p.box_rows == 0 ? launch_kernel<T, G, false, true>(p, bk, bv, tk, tv, st)
                                 : launch_kernel<T, G, false, false>(p, bk, bv, tk, tv, st))
      return rc;
  }
  B200_POST_LAUNCH();
  if (!p.fused_combine) {
    B200_CHECK_CUDA(launch_pdl(attn_combine_kernel<T>, dim3(p.bs, p.hq), dim3(kHeadDim), 0, st,
                               (const float*)p.part_o, (const float*)p.part_ml, p.plan, p.hq, p.out));
    B200_POST_LAUNCH();
  }
  return 0;
}

template <typename T>
static int launch(const DecodeArgs& a) {
  // A batch the plan policy leaves unsplit needs no combine pass: run the in-kernel merge (a no-op
  // then; still correct for a foreign plan that does split) and skip the combine launch.
  int fused = g_decode_fused_combine.load();
  if (fused == 2) fused = decode_plan_is_unsplit(a.bs, a.hkv, 2 * num_sms()) ? 1 : 0;
  // K/V streaming ahead of the predecessor: only for launches that are being captured into a graph
  int early = 0;
  if (g_decode_early_kv.load()) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(a.stream, &cs) == cudaSuccess && cs == cudaStreamCaptureStatusActive) early = 1;
  }
  const DecodeWorkspace ws = carve_decode_workspace(a.workspace, a.workspace_bytes, a.bs, a.hq);
  const Params<T> p{(const T*)a.q, a.q_rs, (const T*)a.k, a.k_rs, (const T*)a.v, a.v_rs, (T*)a.k_cache,
                    (T*)a.v_cache, a.out_loc, a.slot_table, a.st_stride, a.seq_lens, a.plan, a.bs, a.hq, a.hkv,
                    (int)a.num_slots, box_rows_for(a.page_size), g_decode_exact_tail.load() ? 1 : 0, fused,
                    a.scale * kLog2e, (T*)a.out, ws.part_o, ws.part_ml, ws.counters, early, a.fuse,
                    (const T*)a.qw, (const T*)a.kw, a.eps, a.positions, a.cos_sin,
                    TraceArgs{nullptr, 0, 0, a.page_size, 0}};
  const bool bf16 = std::is_same<T, __nv_bfloat16>::value;
  CUtensorMap bk{}, bv{};  // row mode gathers with cp.async and needs no tensor map
  if (p.box_rows > 0)
    if (int rc = kv_pool_maps(&bk, &bv, a.k_cache, a.v_cache, a.num_slots, a.hkv, p.box_rows, bf16)) return rc;
  // 8-row boxes for the last page piece of a range (exact tail)
  CUtensorMap tk = bk, tv = bv;
  if (p.box_rows > 8)
    if (int rc = kv_pool_maps(&tk, &tv, a.k_cache, a.v_cache, a.num_slots, a.hkv, 8, bf16)) return rc;
  switch (p.hq / p.hkv) {
    case 1: return launch_g<T, 1>(p, bk, bv, tk, tv, a.stream);
    case 2: return launch_g<T, 2>(p, bk, bv, tk, tv, a.stream);
    case 3: return launch_g<T, 3>(p, bk, bv, tk, tv, a.stream);
    case 4: return launch_g<T, 4>(p, bk, bv, tk, tv, a.stream);
    case 5: return launch_g<T, 5>(p, bk, bv, tk, tv, a.stream);
    case 6: return launch_g<T, 6>(p, bk, bv, tk, tv, a.stream);
    case 7: return launch_g<T, 7>(p, bk, bv, tk, tv, a.stream);
    case 8: return launch_g<T, 8>(p, bk, bv, tk, tv, a.stream);
    case 9: return launch_g<T, 9>(p, bk, bv, tk, tv, a.stream);
    case 10: return launch_g<T, 10>(p, bk, bv, tk, tv, a.stream);
    case 11: return launch_g<T, 11>(p, bk, bv, tk, tv, a.stream);
    case 12: return launch_g<T, 12>(p, bk, bv, tk, tv, a.stream);
    case 13: return launch_g<T, 13>(p, bk, bv, tk, tv, a.stream);
    case 14: return launch_g<T, 14>(p, bk, bv, tk, tv, a.stream);
    case 15: return launch_g<T, 15>(p, bk, bv, tk, tv, a.stream);
    case 16: return launch_g<T, 16>(p, bk, bv, tk, tv, a.stream);
    default:  // attn_decode() has refused every other group size
      set_error("attn_decode: GQA group size %d not supported by the wgmma decode kernel (1..%d)", p.hq / p.hkv,
                kMaxGroup);
      return 1;
  }
}

}  // namespace dtc

// Every argument check of both decode entry points, then the kernel the options select.
static int attn_decode(const DecodeArgs& a) {
  if (a.fuse) {
    B200_CHECK_ARG(a.positions != nullptr && a.cos_sin != nullptr,
                   "attn_decode_fused: positions / cos_sin_cache must not be NULL");
    B200_CHECK_ARG(((uintptr_t)a.qw % 16) == 0 && ((uintptr_t)a.kw % 16) == 0 && ((uintptr_t)a.cos_sin % 16) == 0,
                   "attn_decode_fused: weights / cos_sin_cache must be 16-byte aligned");
  }
  B200_CHECK_ARG(a.head_dim == kHeadDim, "attn_decode: head_dim must be 128 (got %d)", a.head_dim);
  B200_CHECK_ARG(a.bs > 0 && a.hq > 0 && a.hkv > 0 && a.hq % a.hkv == 0, "attn_decode: bad bs/hq/hkv %d/%d/%d",
                 a.bs, a.hq, a.hkv);
  B200_CHECK_ARG(a.q_rs % 8 == 0 && a.k_rs % 8 == 0 && a.v_rs % 8 == 0,
                 "attn_decode: row strides must be multiples of 8 elements");
  B200_CHECK_ARG(((uintptr_t)a.q % 16) == 0 && ((uintptr_t)a.k % 16) == 0 && ((uintptr_t)a.v % 16) == 0 &&
                     ((uintptr_t)a.k_cache % 16) == 0 && ((uintptr_t)a.v_cache % 16) == 0 &&
                     ((uintptr_t)a.out % 16) == 0,
                 "attn_decode: pointers must be 16-byte aligned");
  const size_t ws_need = decode_workspace_bytes(a.bs, a.hq, a.head_dim);
  B200_CHECK_ARG(a.workspace_bytes >= ws_need, "attn_decode: workspace too small (%zu < %zu)", a.workspace_bytes,
                 ws_need);
  B200_CHECK_ARG(a.plan != nullptr, "attn_decode: decode_plan is NULL (b200_build_metadata)");
  B200_CHECK_ARG(a.page_size >= 1, "attn_decode: page_size must be >= 1");
  B200_CHECK_ARG(a.dtype == B200_DTYPE_BF16 || a.dtype == B200_DTYPE_FP16, "attn_decode: bad dtype %d", a.dtype);
  B200_CHECK_ARG(a.num_slots > 0 && a.num_slots < (1ll << 31), "attn_decode: bad num_slots %lld",
                 (long long)a.num_slots);
  B200_CHECK_ARG(a.st_stride % 4 == 0 && ((uintptr_t)a.slot_table % 16) == 0,
                 "attn_decode: slot table rows must be 16-byte aligned");
  const int group = a.hq / a.hkv;
  if (g_decode_impl.load() == 1) {
    B200_CHECK_ARG(group <= dtc::kMaxGroup,
                   "attn_decode: GQA group size %d (hq/hkv) not supported by the wgmma decode kernel (1..%d)", group,
                   dtc::kMaxGroup);
    return a.dtype == B200_DTYPE_BF16 ? dtc::launch<__nv_bfloat16>(a) : dtc::launch<__half>(a);
  }
  B200_CHECK_ARG(!a.fuse, "attn_decode_fused: only the wgmma kernel (decode_impl = 1) fuses qk-norm + RoPE");
  B200_CHECK_ARG(group <= 8,
                 "attn_decode: GQA group size %d (hq/hkv) not supported by the cp.async bring-up decode kernel (1..8)",
                 group);
#ifdef B200_BRINGUP_KERNELS
  return launch_decode_bringup(a);
#else
  set_error("attn_decode: decode_impl = 0 (cp.async bring-up kernel) is not part of this build (B200_BUILD_BRINGUP=1)");
  return 1;
#endif
}

}  // namespace b200

using namespace b200;

extern "C" size_t b200_attn_workspace_bytes(int max_bs, int hq, int head_dim) {
  return decode_workspace_bytes(max_bs, hq, head_dim);
}

extern "C" int b200_attn_decode(const void* q, int64_t q_row_stride, const void* k, int64_t k_row_stride,
                                const void* v, int64_t v_row_stride, void* k_cache, void* v_cache,
                                int64_t num_slots, int page_size, const int32_t* out_loc,
                                const int32_t* slot_table, int64_t slot_table_stride, const int32_t* seq_lens,
                                const int32_t* decode_plan, int bs, int hq, int hkv, int head_dim, float scale,
                                void* out, void* workspace, size_t workspace_bytes, int dtype, void* stream) {
  return attn_decode({q, q_row_stride, k, k_row_stride, v, v_row_stride, k_cache, v_cache, num_slots, page_size,
                      out_loc, slot_table, slot_table_stride, seq_lens, decode_plan, bs, hq, hkv, head_dim, scale,
                      out, workspace, workspace_bytes, dtype, (cudaStream_t)stream});
}

extern "C" int b200_attn_decode_fused(const void* q, int64_t q_row_stride, const void* k,
                                      int64_t k_row_stride, const void* v, int64_t v_row_stride,
                                      const void* q_weight, const void* k_weight, float eps,
                                      const int32_t* positions, const float* cos_sin_cache,
                                      void* k_cache, void* v_cache, int64_t num_slots, int page_size,
                                      const int32_t* out_loc, const int32_t* slot_table,
                                      int64_t slot_table_stride, const int32_t* seq_lens,
                                      const int32_t* decode_plan, int bs, int hq, int hkv, int head_dim,
                                      float scale, void* out, void* workspace, size_t workspace_bytes,
                                      int dtype, void* stream) {
  return attn_decode({q, q_row_stride, k, k_row_stride, v, v_row_stride, k_cache, v_cache, num_slots, page_size,
                      out_loc, slot_table, slot_table_stride, seq_lens, decode_plan, bs, hq, hkv, head_dim, scale,
                      out, workspace, workspace_bytes, dtype, (cudaStream_t)stream, 1, q_weight, k_weight, eps,
                      positions, cos_sin_cache});
}
