#include "tensor_map.h"

#include <mutex>
#include <unordered_map>

#include "common.h"
#include "drv.h"

namespace b200 {
namespace {

struct MapKey {
  const void* ptr; uint64_t d[4]; uint64_t s[3]; uint32_t b[4]; int rank, dtype, swizzle;
  bool operator==(const MapKey& o) const {
    if (ptr != o.ptr || rank != o.rank || dtype != o.dtype || swizzle != o.swizzle) return false;
    for (int i = 0; i < 4; ++i) if (d[i] != o.d[i] || b[i] != o.b[i]) return false;
    for (int i = 0; i < 3; ++i) if (s[i] != o.s[i]) return false;
    return true;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr) ^ (size_t)k.rank ^ ((size_t)k.dtype << 8) ^ ((size_t)k.swizzle << 16);
    for (int i = 0; i < 4; ++i) h = (h * 1000003u) ^ (size_t)k.d[i] ^ ((size_t)k.b[i] << 20);
    for (int i = 0; i < 3; ++i) h = (h * 1000003u) ^ (size_t)k.s[i];
    return h;
  }
};

}  // namespace

CUtensorMap encode_tensor_map(const void* ptr, CUtensorMapDataType dtype, CUtensorMapSwizzle swizzle, int rank,
                              const uint64_t* dims, const uint64_t* strides, const uint32_t* box) {
  if (rank < 1 || rank > 4) throw std::runtime_error("tensor map: rank must be 1..4");
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  MapKey key{};
  key.ptr = ptr; key.rank = rank; key.dtype = (int)dtype; key.swizzle = (int)swizzle;
  for (int i = 0; i < rank; ++i) { key.d[i] = dims[i]; key.b[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) key.s[i] = strides[i];
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) return it->second;
  }
  auto& drv = Driver::get();
  if (!drv.TensorMapEncodeTiled) throw std::runtime_error("tensor map: cuTensorMapEncodeTiled unavailable");
  // driver-API calls need a current context; autograd worker threads only get one lazily from the runtime
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { B200_CUDA_CHECK(cudaFree(nullptr)); ctx_bound = true; }
  CUtensorMap map;
  cuuint64_t d[4], s[3];
  cuuint32_t b[4], es[4] = {1, 1, 1, 1};
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) s[i] = strides[i];
  B200_DRV_CHECK(drv.TensorMapEncodeTiled(&map, dtype, rank, const_cast<void*>(ptr), d, s, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                          swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
  std::lock_guard<std::mutex> g(mu);
  if (cache.size() > 4096) cache.clear();      // freed-and-reallocated pointers would otherwise grow it without bound
  cache.emplace(key, map);
  return map;
}

}  // namespace b200
