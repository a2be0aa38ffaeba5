#include "host_utils.h"

#include <stdarg.h>
#include <stdio.h>
#include <string.h>

namespace bv {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return BV_OK;
  set_error("%s: %s", what, cudaGetErrorString(e));
  return BV_ERR_CUDA;
}

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

namespace {
struct FinishOuts { float* p[kFinishMaxRows]; };

__global__ void __launch_bounds__(256)
finish_row_sums_kernel(const float* __restrict__ part, int64_t count, FinishOuts out, float div, int accumulate) {
  __shared__ float sh[256];
  static_assert(kFinishMaxRows == 5, "one case per row");
  float* o;
  switch (blockIdx.x) {         // out.p[blockIdx.x] would copy out to the stack
    case 0: o = out.p[0]; break;
    case 1: o = out.p[1]; break;
    case 2: o = out.p[2]; break;
    case 3: o = out.p[3]; break;
    default: o = out.p[4]; break;
  }
  if (o == nullptr) return;     // uniform across the block
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < count; i += 256) acc += part[blockIdx.x * count + i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (static_cast<int>(threadIdx.x) < w) sh[threadIdx.x] += sh[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *o = accumulate ? *o + sh[0] : sh[0] / div;
}
}  // namespace

int finish_row_sums(const float* part, int K, int64_t count, float* const* out, float div, bool accumulate,
                    cudaStream_t s) {
  if (K < 1 || K > kFinishMaxRows) {
    set_error("finish_row_sums: %d rows, need 1 to %d", K, kFinishMaxRows);
    return BV_ERR_INVALID;
  }
  FinishOuts o = {};
  for (int k = 0; k < K; ++k) o.p[k] = out[k];
  finish_row_sums_kernel<<<K, 256, 0, s>>>(part, count, o, div, accumulate ? 1 : 0);
  return check_cuda(cudaGetLastError(), "finish_row_sums_kernel launch");
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

int make_tmap(CUtensorMap* out, CUtensorMapDataType dt, int rank, const void* ptr,
              const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
              bool swizzle128) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return BV_ERR_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) {
    set_error("TMA base pointer %p not 16-byte aligned", ptr);
    return BV_ERR_INVALID;
  }
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i + 1 < rank) {
      gs[i] = strides_bytes[i];
      if (gs[i] % 16 != 0) {
        set_error("TMA stride %llu (dim %d) not a multiple of 16 bytes",
                  (unsigned long long)gs[i], i + 1);
        return BV_ERR_INVALID;
      }
    }
  }
  CUresult r = enc(out, dt, (cuuint32_t)rank, const_cast<void*>(ptr), gd, gs, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d; rank %d dims %llu,%llu box %u,%u)",
              (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              box[0], rank > 1 ? box[1] : 0);
    return BV_ERR_CUDA;
  }
  return BV_OK;
}

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_tmap_im2col_nhwc(CUtensorMap* out, const void* ptr, int64_t n, int h, int w, int c, int lower_w,
                          int lower_h, int upper_w, int upper_h, int stride, int pixels) {
  static EncodeIm2colFn enc = nullptr;
  if (!enc) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
      set_error("cuTensorMapEncodeIm2col entry point unavailable (no CUDA driver?)");
      return BV_ERR_CUDA;
    }
    enc = reinterpret_cast<EncodeIm2colFn>(p);
  }
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) {
    set_error("TMA base pointer %p not 16-byte aligned", ptr);
    return BV_ERR_INVALID;
  }
  const cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  const cuuint64_t strides[3] = {(cuuint64_t)c * 2, (cuuint64_t)w * c * 2, (cuuint64_t)h * w * c * 2};
  const int lower[2] = {lower_w, lower_h}, upper[2] = {upper_w, upper_h};
  const cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, lower, upper, 64,
                   (cuuint32_t)pixels, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeIm2col failed (CUresult %d; n %lld h %d w %d c %d corners %d,%d / %d,%d stride %d)",
              (int)r, (long long)n, h, w, c, lower_w, lower_h, upper_w, upper_h, stride);
    return BV_ERR_CUDA;
  }
  return BV_OK;
}

}  // namespace bv

extern "C" {

const char* bv_last_error_string(void) { return bv::g_err; }
int bv_version(void) { return 101; }

int bv_device_supported(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  return major == 9 ? 1 : 0;
}

}  // extern "C"
