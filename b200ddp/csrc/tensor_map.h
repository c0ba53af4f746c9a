// The one encoder of TMA tensor maps.  The kernel files keep the geometry (which boxes, which pitches) and call this.
#pragma once
#include <cuda.h>
#include <cstdint>

namespace b200 {

// Tiled tensor map of rank <= 4 over `ptr`: dims / box innermost first, strides in bytes for dims 1..rank-1; no interleave,
// L2 promotion 256B, no out-of-bounds fill, element strides 1.  Cached: encoding costs a few microseconds on the host and
// the same (pointer, shape) recurs every step.
CUtensorMap encode_tensor_map(const void* ptr, CUtensorMapDataType dtype, CUtensorMapSwizzle swizzle, int rank,
                              const uint64_t* dims, const uint64_t* strides, const uint32_t* box);

}  // namespace b200
