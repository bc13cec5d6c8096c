// Library-level entry points of the C ABI (include/b200attn.h): error reporting, launch
// accounting, device probe.  Errors follow the reference's convention of surfacing native
// failures as Python RuntimeError (python/minisgl/kernel/csrc/include/minisgl/utils.h:40-88):
// every entry point returns non-zero and leaves a message here.
#include "attn.cuh"
#include "b200attn.h"
#include "common.cuh"

#include <cstring>
#include <mutex>

namespace b200 {

static thread_local char t_error[512] = "";
std::atomic<uint64_t> g_launch_count{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_error, sizeof(t_error), fmt, ap);
  va_end(ap);
}

}  // namespace b200

namespace b200 {
std::atomic<int> g_use_pdl{1};
std::atomic<int> g_decode_impl{1};
std::atomic<int> g_prefill_impl{1};
std::atomic<int> g_prefill_order{0};  // 0 = size-sorted + snake dealing (balanced), 1 = request-major
std::atomic<int> g_prefill_skip_append{0};  // debug only
// Split-KV policy: splitting costs a partial (o, m, l) round trip plus the combine pass, so it only pays
// when whole requests cannot fill the grid.
std::atomic<int> g_decode_plan_target{2};    // when splitting, aim at target * CTA-hint / kv_heads (request, chunk) items
std::atomic<int> g_decode_plan_nosplit{75};  // no split once bs * kv_heads * 100 >= nosplit * CTA-hint (0 = always split)
// 0 = separate combine launch, 1 = the last-arriving chunk's CTA merges the partials in the decode launch (no
// combine launch at all), 2 = in-kernel exactly when the policy above does not split.
std::atomic<int> g_decode_fused_combine{1};
std::atomic<int> g_decode_early_kv{1};  // captured decode launches stream K/V without waiting for the predecessor
std::atomic<int> g_decode_exact_tail{1};  // box mode: the last page piece of a range loads only its valid rows

static const struct {
  const char* name;
  std::atomic<int>* value;
} kOptions[] = {
    {"use_pdl", &g_use_pdl},
    {"decode_impl", &g_decode_impl},
    {"prefill_skip_append", &g_prefill_skip_append},
    {"prefill_order", &g_prefill_order},
    {"prefill_impl", &g_prefill_impl},
    {"decode_plan_target", &g_decode_plan_target},
    {"decode_plan_nosplit", &g_decode_plan_nosplit},
    {"decode_early_kv", &g_decode_early_kv},
    {"decode_fused_combine", &g_decode_fused_combine},
    {"decode_exact_tail", &g_decode_exact_tail},
};
}  // namespace b200

// ------------------------------------------------------------------------------ event trace
// The registered buffer is handed out front to back, one region per traced launch (attn.cuh TraceHeader).
namespace b200 {
static std::mutex g_trace_mu;
static std::atomic<bool> g_trace_on{false};
static struct {
  uint8_t* buf = nullptr;
  size_t bytes = 0, used = 0;
  int events_per_warp = 0;
  uint64_t traced = 0, untraced = 0;
} g_trace;

static int trace_warps(int phase) { return phase == kTracePhaseDecode ? kDecodeWarps : kPrefillWarps; }

bool trace_next_region(int phase, int grid, TraceArgs* out) {
  if (!g_trace_on.load(std::memory_order_relaxed)) return false;
  std::lock_guard<std::mutex> lock(g_trace_mu);
  if (g_trace.buf == nullptr) return false;
  const size_t need = trace_region_bytes(grid, trace_warps(phase), g_trace.events_per_warp);
  if (g_trace.bytes - g_trace.used < need) {
    ++g_trace.untraced;
    return false;
  }
  out->region = g_trace.buf + g_trace.used;
  out->events_per_warp = g_trace.events_per_warp;
  out->seq = (int)g_trace.traced;
  g_trace.used += need;
  ++g_trace.traced;
  return true;
}
}  // namespace b200

extern "C" size_t b200_attn_trace_launch_bytes(int phase, int events_per_warp) {
  using namespace b200;
  if ((phase != kTracePhaseDecode && phase != kTracePhasePrefill) || events_per_warp <= 0) return 0;
  return trace_region_bytes(num_sms(), trace_warps(phase), events_per_warp);
}

extern "C" int b200_attn_trace_set(void* buf, size_t bytes, int events_per_warp) {
  using namespace b200;
  if (buf != nullptr) {
    B200_CHECK_ARG(events_per_warp > 0, "attn_trace_set: events_per_warp must be > 0 (got %d)", events_per_warp);
    B200_CHECK_ARG(((uintptr_t)buf % 16) == 0, "attn_trace_set: the buffer must be 16-byte aligned");
    // The region size depends on the grid: num_sms() queries the device's SM count once (cached).  That query
    // enqueues nothing; it is the only CUDA call made before every argument has been checked.
    const size_t one = b200_attn_trace_launch_bytes(kTracePhaseDecode, events_per_warp);
    B200_CHECK_ARG(bytes >= one, "attn_trace_set: buffer of %zu bytes is smaller than one launch region (%zu)", bytes,
                   one);
  }
  std::lock_guard<std::mutex> lock(g_trace_mu);
  if (buf == nullptr) {  // off; the counts stay readable until the next buffer is registered
    g_trace.buf = nullptr;
    g_trace_on.store(false);
    return 0;
  }
  g_trace.buf = static_cast<uint8_t*>(buf);
  g_trace.bytes = bytes;
  g_trace.used = 0;
  g_trace.events_per_warp = events_per_warp;
  g_trace.traced = g_trace.untraced = 0;
  g_trace_on.store(true);
  return 0;
}

extern "C" int b200_attn_trace_launches(uint64_t* traced, uint64_t* untraced) {
  using namespace b200;
  B200_CHECK_ARG(traced != nullptr && untraced != nullptr, "attn_trace_launches: NULL output pointer");
  std::lock_guard<std::mutex> lock(g_trace_mu);
  *traced = g_trace.traced;
  *untraced = g_trace.untraced;
  return 0;
}

extern "C" int b200_abi_version(void) { return 9; }

#ifndef B200_BUILD_DIGEST
#define B200_BUILD_DIGEST "B200DIGEST:unknown"
#endif
// the marker prefix lets build.py find the digest in the file without loading the library
extern "C" const char* b200_build_digest(void) { return B200_BUILD_DIGEST + 11; }

extern "C" int b200_set_option(const char* name, int value) {
  if (name == nullptr) return -1;
#ifndef B200_BRINGUP_KERNELS
  // the cross-check kernels are compiled into test builds only (B200_BUILD_BRINGUP=1)
  if (value == 0 && (std::strcmp(name, "decode_impl") == 0 || std::strcmp(name, "prefill_impl") == 0)) return -1;
#endif
  for (const auto& o : b200::kOptions)
    if (std::strcmp(name, o.name) == 0) return o.value->exchange(value);
  return -1;
}

extern "C" const char* b200_last_error(void) { return b200::t_error; }

extern "C" uint64_t b200_launch_count(void) { return b200::g_launch_count.load(); }

extern "C" int b200_device_supported(void) {
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  return major == 9 ? 1 : 0;
}
