// FlexiViT resampling (include/bv_b200_flexi.h; reference models/proj/flexi/vit.py): a small fp32 matrix
// M [R, K] applied to every column of a [K, J] matrix, forward (M x, written as bf16) and backward
// (M^T dy, accumulated into fp32).  The shapes a FlexiViT-B step uses are at most R = 2304 (patch 48),
// K = 1024 (base patch 32) and J = 3 * 768, so the whole operation is a few MFLOP over a few MB.
//
// Shape of the kernel: a CTA owns kRows output rows and kThreads * 4 consecutive columns.  Each thread
// keeps kRows x 4 fp32 accumulators in registers and walks the reduction index in ascending order: per
// step one 16-byte load of the input row (coalesced across the CTA) and kRows broadcast reads of M's
// column from shared memory, where M's tile is staged kChunk reduction indices at a time.  No atomics:
// each output element is owned by one thread, so the result is the same bit for bit on every run.
#include "../../include/bv_b200_flexi.h"

#include "common.cuh"
#include "host_utils.h"

namespace bv {
namespace {

constexpr int kThreads = 128;        // 512 columns per CTA
constexpr int kRows = 8;             // output rows per CTA
constexpr int kChunk = 64;           // reduction indices of M staged in shared memory at a time

// out[o, j] = sum_{t ascending} c(o, t) * in[t, j] for o < O, j < J, with c(o, t) = M[o, t] (M is [O, T],
// the forward) or M[t, o] (TRANS: M is [T, O], the backward).  The forward stores bf16, the backward adds
// the sum to the fp32 output.
template <bool TRANS>
__global__ void __launch_bounds__(kThreads)
resample_kernel(const float* __restrict__ M, const float* __restrict__ in, void* out, int O, int T, int64_t J) {
  __shared__ __align__(16) float sm[kChunk][kRows];
  const int o0 = blockIdx.y * kRows;
  const int64_t j = (static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x) * 4;
  const bool active = j < J;
  float4 acc[kRows];
#pragma unroll
  for (int r = 0; r < kRows; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);

  for (int t0 = 0; t0 < T; t0 += kChunk) {
    const int tc = min(kChunk, T - t0);
    __syncthreads();                       // the previous chunk has been consumed
    for (int i = threadIdx.x; i < kChunk * kRows; i += kThreads) {
      const int t = TRANS ? i / kRows : i % kChunk;
      const int r = TRANS ? i % kRows : i / kChunk;
      const int o = o0 + r;
      float v = 0.f;
      if (t < tc && o < O) v = TRANS ? M[static_cast<int64_t>(t0 + t) * O + o] : M[static_cast<int64_t>(o) * T + t0 + t];
      sm[t][r] = v;
    }
    __syncthreads();
    if (active) {
      const float* src = in + static_cast<int64_t>(t0) * J + j;
#pragma unroll 4
      for (int t = 0; t < tc; ++t) {
        const float4 v = *reinterpret_cast<const float4*>(src + static_cast<int64_t>(t) * J);
        const float4 c0 = *reinterpret_cast<const float4*>(&sm[t][0]);
        const float4 c1 = *reinterpret_cast<const float4*>(&sm[t][4]);
        const float c[kRows] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
        for (int r = 0; r < kRows; ++r) {
          acc[r].x = fmaf(c[r], v.x, acc[r].x);
          acc[r].y = fmaf(c[r], v.y, acc[r].y);
          acc[r].z = fmaf(c[r], v.z, acc[r].z);
          acc[r].w = fmaf(c[r], v.w, acc[r].w);
        }
      }
    }
  }
  if (!active) return;
#pragma unroll
  for (int r = 0; r < kRows; ++r) {
    const int o = o0 + r;
    if (o >= O) break;
    const int64_t off = static_cast<int64_t>(o) * J + j;
    if (TRANS) {
      float4* dst = reinterpret_cast<float4*>(static_cast<float*>(out) + off);
      const float4 d = *dst;
      *dst = make_float4(d.x + acc[r].x, d.y + acc[r].y, d.z + acc[r].z, d.w + acc[r].w);
    } else {
      uint2 q;
      q.x = pack_bf16(acc[r].x, acc[r].y);
      q.y = pack_bf16(acc[r].z, acc[r].w);
      *reinterpret_cast<uint2*>(static_cast<bf16*>(out) + off) = q;
    }
  }
}

inline bool misaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

// Shared argument checks of both entry points; O output rows of the launch.
int check_args(const char* name, const float* M, const void* in, const void* out, int32_t R, int32_t K, int64_t J,
               uintptr_t out_align) {
  if (!M || !in || !out) {
    set_error("%s: null buffer", name);
    return BV_ERR_INVALID;
  }
  if (R < 1 || K < 1 || J < 4 || J % 4) {
    set_error("%s: need R >= 1, K >= 1 and J a positive multiple of 4, got R=%d K=%d J=%lld", name, R, K,
              static_cast<long long>(J));
    return BV_ERR_INVALID;
  }
  if ((J / 4 + kThreads - 1) / kThreads > 0x7fffffff) {
    set_error("%s: J=%lld is too large", name, static_cast<long long>(J));
    return BV_ERR_INVALID;
  }
  if (misaligned(in, 16) || misaligned(out, out_align)) {
    set_error("%s: the fp32 inputs and outputs must be 16-byte aligned, the bf16 output 8-byte aligned", name);
    return BV_ERR_INVALID;
  }
  return BV_OK;
}

inline dim3 grid_of(int O, int64_t J) {
  return dim3(static_cast<unsigned>((J / 4 + kThreads - 1) / kThreads), static_cast<unsigned>((O + kRows - 1) / kRows));
}

}  // namespace
}  // namespace bv

extern "C" {

int bv_resample_fwd(const float* M, const float* x, void* y_bf16, int32_t R, int32_t K, int64_t J, void* stream) {
  using namespace bv;
  const int rc = check_args("bv_resample_fwd", M, x, y_bf16, R, K, J, 8);
  if (rc) return rc;
  resample_kernel<false><<<grid_of(R, J), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(M, x, y_bf16, R, K, J);
  return check_cuda(cudaGetLastError(), "resample_kernel<fwd> launch");
}

int bv_resample_bwd(const float* M, const float* dy, float* dx, int32_t R, int32_t K, int64_t J, void* stream) {
  using namespace bv;
  const int rc = check_args("bv_resample_bwd", M, dy, dx, R, K, J, 16);
  if (rc) return rc;
  resample_kernel<true><<<grid_of(K, J), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(M, dy, dx, K, R, J);
  return check_cuda(cudaGetLastError(), "resample_kernel<bwd> launch");
}

}  // extern "C"
