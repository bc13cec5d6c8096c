// Library-level entry points of the C ABI (include/b200attn.h): error reporting, launch
// accounting, device probe.  Errors follow the reference's convention of surfacing native
// failures as Python RuntimeError (python/minisgl/kernel/csrc/include/minisgl/utils.h:40-88):
// every entry point returns non-zero and leaves a message here.
#include "b200attn.h"
#include "common.cuh"

#include <cstring>

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
}

extern "C" int b200_abi_version(void) { return 7; }

#ifndef B200_BUILD_DIGEST
#define B200_BUILD_DIGEST "B200DIGEST:unknown"
#endif
// the marker prefix lets build.py find the digest in the file without loading the library
extern "C" const char* b200_build_digest(void) { return B200_BUILD_DIGEST + 11; }

extern "C" int b200_set_option(const char* name, int value) {
#ifndef B200_BRINGUP_KERNELS
  // the cross-check kernels are compiled into test builds only (B200_BUILD_BRINGUP=1)
  if (name != nullptr && value == 0 && (std::strcmp(name, "decode_impl") == 0 || std::strcmp(name, "prefill_impl") == 0))
    return -1;
#endif
  if (name != nullptr && std::strcmp(name, "use_pdl") == 0) return b200::g_use_pdl.exchange(value);
  if (name != nullptr && std::strcmp(name, "decode_impl") == 0) return b200::g_decode_impl.exchange(value);
  if (name != nullptr && std::strcmp(name, "prefill_skip_append") == 0) return b200::g_prefill_skip_append.exchange(value);
  if (name != nullptr && std::strcmp(name, "prefill_order") == 0) return b200::g_prefill_order.exchange(value);
  if (name != nullptr && std::strcmp(name, "prefill_impl") == 0) return b200::g_prefill_impl.exchange(value);
  if (name != nullptr && std::strcmp(name, "decode_plan_target") == 0) return b200::g_decode_plan_target.exchange(value);
  if (name != nullptr && std::strcmp(name, "decode_plan_nosplit") == 0) return b200::g_decode_plan_nosplit.exchange(value);
  if (name != nullptr && std::strcmp(name, "decode_early_kv") == 0) return b200::g_decode_early_kv.exchange(value);
  if (name != nullptr && std::strcmp(name, "decode_fused_combine") == 0) return b200::g_decode_fused_combine.exchange(value);
  if (name != nullptr && std::strcmp(name, "decode_exact_tail") == 0) return b200::g_decode_exact_tail.exchange(value);
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
