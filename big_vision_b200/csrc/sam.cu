// GSAM / SAM vector algebra over the flat parameter and gradient buffers (include/bv_b200_sam.h;
// reference trainers/proj/gsam/gsam.py:28-122).  A GSAM step is two forward+backward passes joined
// by global-vector operations: the norm of the clean gradient, the perturbed weights, the dot
// products of the two gradients and their combination.  All of it is HBM-bound streaming; the norms
// and dot products stay on the device and each kernel reads them from there.
//   perturb  reads w, g (8 B) and writes w_sam, its bf16 shadow (6 B) per parameter;
//   dots     reads a, b (8 B; 4 B for the norm of one buffer);
//   combine  reads g_c, g_r (8 B) and writes g (4 B).
#include "../../include/bv_b200_sam.h"

#include "common.cuh"
#include "host_utils.h"

namespace bv {
namespace {

constexpr int kThreads = 256;
constexpr int kDotsBlocks = BV_SAM_WS_FLOATS / 2;   // grid cap of bv_sam_dots: one partial pair per block

__device__ __forceinline__ float perturb_one(float w, float g, float rho, float den, bool adaptive) {
  const float num = adaptive ? (fabsf(w) * rho) * g : rho * g;
  return w + __fdiv_rn(num, den);
}

__global__ void __launch_bounds__(kThreads)
sam_perturb_kernel(const float* __restrict__ w, const float* __restrict__ g, const float* __restrict__ g_sumsq,
                   float rho, float eps, int adaptive, float* w_out, bf16* __restrict__ w16, int64_t n) {
  // gsam.py:24-25 (dual_vector's norm) and :78-83: rho * g / (||g|| + eps)
  const float den = __fadd_rn(__fsqrt_rn(g_sumsq[0]), eps);
  const bool ad = adaptive != 0;
  const int64_t n4 = n / 4;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 wv = reinterpret_cast<const float4*>(w)[i];
    const float4 gv = reinterpret_cast<const float4*>(g)[i];
    const float4 o = make_float4(perturb_one(wv.x, gv.x, rho, den, ad), perturb_one(wv.y, gv.y, rho, den, ad),
                                 perturb_one(wv.z, gv.z, rho, den, ad), perturb_one(wv.w, gv.w, rho, den, ad));
    reinterpret_cast<float4*>(w_out)[i] = o;
    uint2 q;
    q.x = pack_bf16(o.x, o.y); q.y = pack_bf16(o.z, o.w);
    reinterpret_cast<uint2*>(w16)[i] = q;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = n4 * 4 + threadIdx.x;
    const float o = perturb_one(w[i], g[i], rho, den, ad);
    w_out[i] = o;
    w16[i] = __float2bfloat16_rn(o);
  }
}

template <bool SAME>
__global__ void __launch_bounds__(kThreads)
sam_dots_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ part, int64_t n) {
  __shared__ float sh[64];
  float ab = 0.f, bb = 0.f;
  const int64_t n4 = n / 4;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 bv = reinterpret_cast<const float4*>(b)[i];
    bb += bv.x * bv.x + bv.y * bv.y + bv.z * bv.z + bv.w * bv.w;
    if (!SAME) {
      const float4 av = reinterpret_cast<const float4*>(a)[i];
      ab += av.x * bv.x + av.y * bv.y + av.z * bv.z + av.w * bv.w;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = n4 * 4 + threadIdx.x;
    bb += b[i] * b[i];
    if (!SAME) ab += a[i] * b[i];
  }
  float sums[2] = {ab, bb};
  block_sum(sums, sh);
  if (threadIdx.x == 0) {
    part[blockIdx.x] = SAME ? sums[1] : sums[0];
    part[gridDim.x + blockIdx.x] = sums[1];
  }
}

// gsam.py:92-105 (minimize_fp) with (x, y) = (g_r, g_c) and sign -1; gsam.py:106-119 with
// (x, y) = (g_c, g_r) and sign +1.  Either way: out = x + sign * alpha * (y - c * (x_or_y / nrm)).
template <bool MIN_FP>
__device__ __forceinline__ float combine_one(float gc, float gr, float nrm, float c, float alpha) {
  if (MIN_FP) return gr - alpha * (gc - c * __fdiv_rn(gr, nrm));
  return gc + alpha * (gr - c * __fdiv_rn(gc, nrm));
}

template <bool MIN_FP>
__global__ void __launch_bounds__(kThreads)
gsam_combine_kernel(float* __restrict__ gc, const float* __restrict__ gr, const float* __restrict__ dot,
                    const float* __restrict__ norm_sq, float alpha, int64_t n) {
  const float nrm = __fsqrt_rn(norm_sq[0]);            // dual_vector's norm (gsam.py:24-25), no eps
  const float c = __fdiv_rn(dot[0], nrm);              // the projection norm of gsam.py:98-99 / :112-113
  const int64_t n4 = n / 4;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 cv = reinterpret_cast<const float4*>(gc)[i];
    const float4 rv = reinterpret_cast<const float4*>(gr)[i];
    reinterpret_cast<float4*>(gc)[i] =
        make_float4(combine_one<MIN_FP>(cv.x, rv.x, nrm, c, alpha), combine_one<MIN_FP>(cv.y, rv.y, nrm, c, alpha),
                    combine_one<MIN_FP>(cv.z, rv.z, nrm, c, alpha), combine_one<MIN_FP>(cv.w, rv.w, nrm, c, alpha));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = n4 * 4 + threadIdx.x;
    gc[i] = combine_one<MIN_FP>(gc[i], gr[i], nrm, c, alpha);
  }
}

inline bool misaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

inline unsigned stream_blocks(int64_t n) { return grid_for(n / 4, kThreads, num_sms() * 8); }

}  // namespace
}  // namespace bv

extern "C" {

int bv_sam_perturb(const float* w, const float* g, const float* g_sumsq, float rho, float eps, int32_t adaptive,
                   float* w_out, void* w_bf16, int64_t n, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n < 0 || (n > 0 && (!w || !g || !g_sumsq || !w_out || !w_bf16))) {
    set_error("bv_sam_perturb: null buffer or n < 0");
    return BV_ERR_INVALID;
  }
  if (n == 0) return BV_OK;
  if (misaligned(w, 16) || misaligned(g, 16) || misaligned(w_out, 16) || misaligned(w_bf16, 8)) {
    set_error("bv_sam_perturb: fp32 buffers must be 16-byte and the bf16 output 8-byte aligned");
    return BV_ERR_INVALID;
  }
  sam_perturb_kernel<<<stream_blocks(n), kThreads, 0, s>>>(w, g, g_sumsq, rho, eps, adaptive, w_out,
                                                            reinterpret_cast<bf16*>(w_bf16), n);
  return check_cuda(cudaGetLastError(), "sam_perturb_kernel launch");
}

int bv_sam_dots(const float* a, const float* b, float* out, float* ws, int64_t n, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n < 0 || !a || !b || !out || !ws) {
    set_error("bv_sam_dots: null buffer or n < 0");
    return BV_ERR_INVALID;
  }
  if (misaligned(a, 16) || misaligned(b, 16)) {
    set_error("bv_sam_dots: a and b must be 16-byte aligned");
    return BV_ERR_INVALID;
  }
  const unsigned blocks = grid_for(n / 4, kThreads, kDotsBlocks);
  if (a == b) sam_dots_kernel<true><<<blocks, kThreads, 0, s>>>(a, b, ws, n);
  else sam_dots_kernel<false><<<blocks, kThreads, 0, s>>>(a, b, ws, n);
  int rc = check_cuda(cudaGetLastError(), "sam_dots_kernel launch");
  if (rc) return rc;
  float* const outs[2] = {out, out + 1};
  return finish_row_sums(ws, 2, blocks, outs, 1.f, false, s);
}

int bv_gsam_combine(float* gc, const float* gr, const float* dot, const float* norm_sq, float alpha,
                    int32_t minimize_fp, int64_t n, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n < 0 || (n > 0 && (!gc || !gr || !dot || !norm_sq))) {
    set_error("bv_gsam_combine: null buffer or n < 0");
    return BV_ERR_INVALID;
  }
  if (n == 0) return BV_OK;
  if (misaligned(gc, 16) || misaligned(gr, 16)) {
    set_error("bv_gsam_combine: g_clean and g_robust must be 16-byte aligned");
    return BV_ERR_INVALID;
  }
  if (minimize_fp) gsam_combine_kernel<true><<<stream_blocks(n), kThreads, 0, s>>>(gc, gr, dot, norm_sq, alpha, n);
  else gsam_combine_kernel<false><<<stream_blocks(n), kThreads, 0, s>>>(gc, gr, dot, norm_sq, alpha, n);
  return check_cuda(cudaGetLastError(), "gsam_combine_kernel launch");
}

}  // extern "C"
