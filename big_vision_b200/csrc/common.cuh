// Shared device helpers for the sm_90a kernels: mbarrier, TMA and wgmma wrappers, warp
// reductions and small math.  Nothing here allocates or syncs.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "wgmma.cuh"

namespace bv {

typedef __nv_bfloat16 bf16;

// ----------------------------------------------------------------------------
// dtype codes shared with the C ABI (include/bv_b200.h)
// ----------------------------------------------------------------------------
enum : int { DT_F32 = 0, DT_BF16 = 1 };

// ----------------------------------------------------------------------------
// small utilities
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// Pins a value in a register: kernel parameters live in the constant bank, and ptxas prefers to
// RE-LOAD them (LDC / LDCU, ~40 cycles on the dependency chain) at every use inside unrolled
// loops instead of keeping a hoisted copy -- an empty inline asm does not stop it (nothing reaches
// ptxas).  Routing the value through a warp shuffle from the thread's own lane does: the result
// is opaque, costs one SHFL per kernel, and must be called with the full warp converged.
__device__ __forceinline__ uint32_t pin_reg(uint32_t v) {
  return __shfl_sync(0xffffffffu, v, static_cast<int>(threadIdx.x & 31));
}
__device__ __forceinline__ int pin_reg(int v) { return static_cast<int>(pin_reg(static_cast<uint32_t>(v))); }
__device__ __forceinline__ float pin_reg(float v) { return __uint_as_float(pin_reg(__float_as_uint(v))); }
template <typename T>
__device__ __forceinline__ T* pin_reg(T* v) {
  const unsigned long long u = reinterpret_cast<unsigned long long>(v);
  const uint32_t lo = pin_reg(static_cast<uint32_t>(u)), hi = pin_reg(static_cast<uint32_t>(u >> 32));
  return reinterpret_cast<T*>((static_cast<unsigned long long>(hi) << 32) | lo);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// CTA sums of N values per thread in the one fixed order of the deterministic reductions (DESIGN.md,
// "Run-to-run determinism"): a butterfly within each warp, then a butterfly over the warp totals, the
// lanes past the last warp adding 0.  Every thread gets the same sums.  blockDim.x is a multiple of 32
// (at most 1024); sh holds 32 * N values and may be reused after the call.
template <int N, typename T>
__device__ __forceinline__ void block_sum(T (&v)[N], T* sh) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) v[k] = warp_sum(v[k]);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k) sh[32 * k + warp] = v[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < N; ++k) v[k] = warp_sum(lane < nw ? sh[32 * k + lane] : T(0));
  __syncthreads();
}
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* sh) {
  T a[1] = {v};
  block_sum(a, sh);
  return a[0];
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// streaming 16-byte read-only load that does not allocate in L1
__device__ __forceinline__ uint4 ld_nc_na(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ float round_bf16(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

// tanh-approximate GELU, the Flax `nn.gelu` default (approximate=True):
//   0.5 x (1 + tanh( sqrt(2/pi) (x + 0.044715 x^3) ))
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  // exact-ish tanh via exp to stay within 1e-6 of the fp32 oracle
  float t = 1.0f - 2.0f / (1.0f + __expf(2.0f * u));
  return 0.5f * x * (1.0f + t);
}
__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float x2 = x * x;
  float u = k0 * (x + k1 * x * x2);
  float t = 1.0f - 2.0f / (1.0f + __expf(2.0f * u));
  float du = k0 * (1.0f + 3.0f * k1 * x2);
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * du;
}

// MUFU-based variants for the GEMM epilogues (bf16 outputs): tanh.approx.f32 has ~2^-11
// relative error.  That is inside the 2^-9 of the bf16 rounding for t = tanh(u) itself, but not
// for the results: 1 + t cancels as t -> -1, so the bound that holds is an ABSOLUTE error of
// |x|/2 * 2^-11 on gelu and (1/2 + |x| du) * 2^-11 on gelu' (du = d u / d x), plus one bf16
// rounding.  For x < -2 that is many bf16 ulps of the (small) result: measured on an H100 over
// every bf16 input, up to ~255 bf16 ulps, and 100 % relative error on x in [-8, -2] where the
// result rounds to 0.  The error is confined to values that are small next to the tensor's scale.
// (tests/test_kernel_edges_gpu.py sweeps every bf16 input against these bounds.)
__device__ __forceinline__ float gelu_tanh_fast(float x) {
  const float k0 = 0.7978845608028654f, k01 = 0.7978845608028654f * 0.044715f;
  const float t = tanh_fast(x * fmaf(k01, x * x, k0));
  const float h = 0.5f * x;
  return fmaf(h, t, h);
}
__device__ __forceinline__ float gelu_tanh_grad_fast(float x) {
  const float k0 = 0.7978845608028654f, k01 = 0.7978845608028654f * 0.044715f;
  const float x2 = x * x;
  const float t = tanh_fast(x * fmaf(k01, x2, k0));
  const float du = fmaf(3.0f * k01, x2, k0);
  return fmaf(0.5f * x * fmaf(-t, t, 1.0f), du, fmaf(0.5f, t, 0.5f));
}

// ----------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// BV_MBAR_SUSPEND_NS (build-time experiment, `python -m big_vision_b200.build --variant`): pass an
// explicit suspend-time hint so that a waiting warp is parked by the hardware for up to that long
// instead of returning to the polling loop after the (shorter, implementation-defined) default.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
#ifdef BV_MBAR_SUSPEND_NS
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity), "r"(static_cast<uint32_t>(BV_MBAR_SUSPEND_NS))
        : "memory");
#else
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
#endif
  } while (!ok);
}
// non-blocking: has the phase with this parity completed?
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// one lane of a fully converged warp (the same lane every time for a full mask)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor)
// ----------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col mode on an NHWC map (c, w, h, n): the map's pixelsPerColumn pixels from base (w, h, n), each shifted
// by the filter offset (ow, oh), channelsPerPixel channels from c
__device__ __forceinline__ void tma_load_im2col_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c, int w,
                                                   int h, int n, uint16_t ow, uint16_t oh) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"(ow), "h"(oh)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, uint32_t src, int c0, int c1,
                                             int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, uint32_t src, int c0,
                                                  int c1) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* m, uint32_t src, int c0,
                                                  int c1, int c2) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.bulk_group [%0, {%2, %3, %4}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------
// Philox4x64-10 (Salmon et al., SC'11), the generator of numpy's np.random.Philox: the counter-based
// stream of Jet's dequantization noise and of the dropout masks.  ctr is replaced by the block's output.
// ----------------------------------------------------------------------------
constexpr uint64_t kPhiloxM0 = 0xD2E7470EE14C6C93ull, kPhiloxM1 = 0xCA5A826395121157ull;
constexpr uint64_t kPhiloxW0 = 0x9E3779B97F4A7C15ull, kPhiloxW1 = 0xBB67AE8584CAA73Bull;

__device__ __forceinline__ void philox4x64_10(uint64_t ctr[4], uint64_t k0, uint64_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k0 += kPhiloxW0;
      k1 += kPhiloxW1;
    }
    const uint64_t hi0 = __umul64hi(kPhiloxM0, ctr[0]), lo0 = kPhiloxM0 * ctr[0];
    const uint64_t hi1 = __umul64hi(kPhiloxM1, ctr[2]), lo1 = kPhiloxM1 * ctr[2];
    const uint64_t c1 = ctr[1], c3 = ctr[3];
    ctr[0] = hi1 ^ c1 ^ k0;
    ctr[1] = lo1;
    ctr[2] = hi0 ^ c3 ^ k1;
    ctr[3] = lo0;
  }
}

}  // namespace bv
