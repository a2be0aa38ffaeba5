// Host-side helpers shared by the launchers: error reporting, TMA descriptor
// encoding through the driver entry point (no -lcuda link dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bv_b200.h"  // BV_OK / BV_ERR_* codes

namespace bv {

void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);
int num_sms();

// Encode a tiled tensor map with 128-byte swizzle (or none).  dims/strides are
// innermost-first; strides[i] is the byte stride of dim i+1.
int make_tmap(CUtensorMap* out, CUtensorMapDataType dt, int rank, const void* ptr,
              const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
              bool swizzle128);

inline int make_tmap_2d(CUtensorMap* out, CUtensorMapDataType dt, const void* ptr, uint64_t inner,
                        uint64_t outer, uint64_t row_stride_bytes, uint32_t box_inner,
                        uint32_t box_outer) {
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {row_stride_bytes};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap(out, dt, 2, ptr, dims, strides, box, true);
}

}  // namespace bv
