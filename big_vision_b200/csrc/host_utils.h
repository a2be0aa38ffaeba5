// Host-side helpers shared by the launchers: error reporting, grid sizes, the fixed-order
// finishing pass, TMA descriptor encoding through the driver entry point (no -lcuda link
// dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bv_b200.h"  // BV_OK / BV_ERR_* codes

namespace bv {

void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);
int num_sms();

// Blocks of a grid-stride launch: ceil(work / threads), at most cap_blocks, at least 1.  For a kernel
// that writes one partial per block this is also the number of partials, so it fixes the summation order.
inline unsigned grid_for(int64_t work, int threads, int64_t cap_blocks) {
  int64_t b = (work + threads - 1) / threads;
  if (b > cap_blocks) b = cap_blocks;
  if (b < 1) b = 1;
  return static_cast<unsigned>(b);
}

// The finishing pass of the deterministic reductions (DESIGN.md, "Run-to-run determinism"), one launch:
// for each row k < K of part [K, count], thread t of 256 sums entries t, t + 256, ... in index order, a
// shared-memory tree adds the 256 sums, and then out[k] = sum / div, or out[k] += sum when accumulate.
// A null out[k] is skipped.  K <= kFinishMaxRows.
constexpr int kFinishMaxRows = 5;
int finish_row_sums(const float* part, int K, int64_t count, float* const* out, float div, bool accumulate,
                    cudaStream_t s);

// Encode a tiled tensor map with 128-byte swizzle (or none).  dims/strides are
// innermost-first; strides[i] is the byte stride of dim i+1.
int make_tmap(CUtensorMap* out, CUtensorMapDataType dt, int rank, const void* ptr,
              const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
              bool swizzle128);

// Encode an im2col-mode map of a bf16 NHWC tensor [n, h, w, c] with 128-byte swizzle: a load yields
// `pixels` rows of 64 channels (128 B).  The base positions a load may start from span
// [lower, dim - 1 + upper] in w and h, stepped by `stride`.
int make_tmap_im2col_nhwc(CUtensorMap* out, const void* ptr, int64_t n, int h, int w, int c, int lower_w,
                          int lower_h, int upper_w, int upper_h, int stride, int pixels);

inline int make_tmap_2d(CUtensorMap* out, CUtensorMapDataType dt, const void* ptr, uint64_t inner,
                        uint64_t outer, uint64_t row_stride_bytes, uint32_t box_inner,
                        uint32_t box_outer) {
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {row_stride_bytes};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap(out, dt, 2, ptr, dims, strides, box, true);
}

}  // namespace bv
