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

extern "C" int b200_abi_version(void) { return 7; }

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
