// Host side of TMA: tensor-map encoding through the driver entry point (resolved at run time via
// the CUDA runtime, so libb200attn.so does not link against libcuda) and a small cache keyed by
// (base pointer, shape) -- the KV pool layers are the only tensors ever described.
#include "attn.cuh"
#include "sm90.cuh"

#include <cudaTypedefs.h>

#include <mutex>
#include <unordered_map>

namespace b200 {

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                              CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                              CUtensorMapFloatOOBfill);

static EncodeFn get_encode_fn() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(p);
  });
  return fn;
}

int encode_tensor_map_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                         uint64_t row_stride_bytes, uint32_t box_cols, uint32_t box_rows,
                         bool is_bf16) {
  EncodeFn fn = get_encode_fn();
  B200_CHECK_ARG(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (driver too old?)");
  B200_CHECK_ARG(((uintptr_t)base % 16) == 0 && row_stride_bytes % 16 == 0,
                 "tensor map: base / stride must be 16-byte aligned");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t elem[2] = {1, 1};
  CUresult rc = fn(out, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                   const_cast<void*>(base), dims, strides, box, elem, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_CHECK_ARG(rc == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d", (int)rc);
  return 0;
}

struct MapKey {
  const void* base;
  uint64_t rows, cols, stride;
  uint32_t box_cols, box_rows;
  bool bf16;
  bool operator==(const MapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && stride == o.stride &&
           box_cols == o.box_cols && box_rows == o.box_rows && bf16 == o.bf16;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.base);
    h = h * 1000003u ^ std::hash<uint64_t>()(k.rows * 31 + k.cols);
    h = h * 1000003u ^ std::hash<uint64_t>()(k.stride * 131 + k.box_cols * 7 + k.box_rows + (k.bf16 ? 1 : 0));
    return h;
  }
};

// Returns a cached tensor map (by value copy into *out).
int get_tensor_map_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t row_stride_bytes, uint32_t box_cols, uint32_t box_rows, bool is_bf16) {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  MapKey key{base, rows, cols, row_stride_bytes, box_cols, box_rows, is_bf16};
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it == cache.end()) {
    CUtensorMap m;
    if (int rc = encode_tensor_map_2d(&m, base, rows, cols, row_stride_bytes, box_cols, box_rows, is_bf16))
      return rc;
    it = cache.emplace(key, m).first;
  }
  *out = it->second;
  return 0;
}

}  // namespace b200
