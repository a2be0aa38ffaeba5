// Jet normalizing flow (include/bv_b200_jet.h; reference models/proj/jet/jet.py, trainers/proj/jet/train.py):
// the element-wise flow around the coupling DNNs.  Every kernel here is a gather / scatter over the fp32 flow
// state and reads or writes each element once, so they are bound by memory bandwidth; the DNN between them
// is the library's GEMM / attention / LayerNorm path.
//
// Determinism: the per-image sums (the coupling log-determinant, the negative log-likelihood) are computed by
// one CTA per image.  Each thread sums a fixed strided subset of the image in ascending order, the warp
// reduces with a fixed butterfly and thread 0 adds the warp totals in warp order: no atomics, so every
// output is the same bit for bit on every run.
#include "../../include/bv_b200_jet.h"

#include <cuda_bf16.h>

#include "common.cuh"
#include "host_utils.h"

namespace bv {
namespace {

constexpr int kThreads = 256;        // element-wise kernels
constexpr int kRedThreads = 512;     // one CTA per image for the reductions

// ---- Philox4x64-10 (Salmon et al., SC'11), the generator of numpy's np.random.Philox -----------------------
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

// Thread i owns Philox block (offset / 8 + i): the 8 uniforms of global elements [8 b, 8 b + 8), of which it
// writes those that fall in this batch.  Block b runs at counter (b + 1, counter, 0, 0): numpy increments the
// first counter word before each block.
__global__ void __launch_bounds__(kThreads)
dequantize_patchify_kernel(const float* __restrict__ image, float* __restrict__ z, int64_t N, int H, int W, int C,
                           int ps, uint64_t seed, uint64_t counter, int64_t offset, float noise_scale) {
  const int64_t blk = offset / 8 + static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  const int64_t g0 = blk * 8;
  if (g0 >= offset + N) return;
  uint64_t ctr[4] = {static_cast<uint64_t>(blk) + 1, counter, 0, 0};
  if (noise_scale != 0.f) philox4x64_10(ctr, seed, 0);
  const int gw = W / ps, Dt = ps * ps * C;
  const int64_t per_image = static_cast<int64_t>(H) * W * C;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t e = g0 + i - offset;
    if (e < 0 || e >= N) continue;
    float v = image[e];
    if (noise_scale != 0.f) {
      const uint64_t word = ctr[i >> 1];
      const uint32_t u32 = (i & 1) ? static_cast<uint32_t>(word >> 32) : static_cast<uint32_t>(word);
      const float u = static_cast<float>(u32 >> 8) * 5.9604644775390625e-08f;    // 2^-24, exact
      v = __fadd_rn(v, __fmul_rn(u, noise_scale));
    }
    const int64_t b = e / per_image;
    int r = static_cast<int>(e - b * per_image);
    const int ch = r % C;
    r /= C;
    const int x = r % W, y = r / W;
    const int t = (y / ps) * gw + x / ps, k = ((y % ps) * ps + x % ps) * C + ch;
    z[(b * (H / ps) * gw + t) * Dt + k] = v;
  }
}

__global__ void __launch_bounds__(kThreads)
unpatchify_kernel(const float* __restrict__ z, float* __restrict__ image, int64_t N, int H, int W, int C, int ps) {
  const int64_t e = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  if (e >= N) return;
  const int gw = W / ps, Dt = ps * ps * C;
  const int64_t per_image = static_cast<int64_t>(H) * W * C;
  const int64_t b = e / per_image;
  int r = static_cast<int>(e - b * per_image);
  const int ch = r % C;
  r /= C;
  const int x = r % W, y = r / W;
  const int t = (y / ps) * gw + x / ps, k = ((y % ps) * ps + x % ps) * C + ch;
  image[e] = z[(b * (H / ps) * gw + t) * Dt + k];
}

__global__ void __launch_bounds__(kThreads)
split_kernel(const float* __restrict__ x, const int* __restrict__ idx, bf16* __restrict__ x1, int64_t n, int half) {
  const int64_t e = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  if (e >= n * half) return;
  const int64_t b = e / half;
  const int j = static_cast<int>(e - b * half);
  x1[e] = __float2bfloat16_rn(x[b * 2 * half + idx[j]]);
}

__device__ __forceinline__ float sigmoid_stable(float r) {
  if (r >= 0.f) return 1.f / (1.f + expf(-r));
  const float e = expf(r);
  return e / (1.f + e);
}

// log(sigmoid(r)) = min(r, 0) - log1p(exp(-|r|)): finite for every finite r.
__device__ __forceinline__ float log_sigmoid_stable(float r) { return fminf(r, 0.f) - log1pf(expf(-fabsf(r))); }

// Sum of v over the CTA in a fixed order; the result is valid in thread 0.
__device__ __forceinline__ float block_sum(float v, float* warp_tot) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) warp_tot[w] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0)
    for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) s += warp_tot[i];
  return s;
}

// One CTA per image b.
__global__ void __launch_bounds__(kRedThreads)
coupling_fwd_kernel(const float* x, const int* __restrict__ idx, const float* __restrict__ br, float* y,
                    float* __restrict__ logdet, int T, int c, float scale_factor, float log_scale, int inverse) {
  __shared__ float warp_tot[kRedThreads / 32];
  const int half = T * c;
  const int64_t b = blockIdx.x;
  const float* xb = x + b * 2 * half;
  float* yb = y + b * 2 * half;
  const float* brb = br + b * 2 * half;
  float acc = 0.f;
  for (int j = threadIdx.x; j < half; j += kRedThreads) {
    const int row = j / c, col = j - row * c;
    const float bias = brb[row * 2 * c + col], raw = brb[row * 2 * c + c + col];
    const float s = __fmul_rn(sigmoid_stable(raw), scale_factor);
    const int p2 = idx[half + j];
    const float x2 = xb[p2];
    yb[p2] = inverse ? __fsub_rn(__fdiv_rn(x2, s), bias) : __fmul_rn(__fadd_rn(x2, bias), s);
    if (y != x) {
      const int p1 = idx[j];
      yb[p1] = xb[p1];
    }
    acc += log_sigmoid_stable(raw) + log_scale;
  }
  const float tot = block_sum(acc, warp_tot);
  if (threadIdx.x == 0) logdet[b] += inverse ? -tot : tot;
}

__global__ void __launch_bounds__(kThreads)
coupling_bwd_kernel(const float* dy, const float* __restrict__ x, const int* __restrict__ idx,
                    const float* __restrict__ br, float dlogdet, float* dx, bf16* __restrict__ dbr, int64_t n, int T,
                    int c, float scale_factor) {
  const int half = T * c;
  const int64_t e = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  if (e >= n * half) return;
  const int64_t b = e / half;
  const int j = static_cast<int>(e - b * half);
  const int row = j / c, col = j - row * c;
  const int64_t rb = (b * T + row) * 2 * c;
  const float bias = br[rb + col], raw = br[rb + c + col];
  const float sig = sigmoid_stable(raw), one_m = sigmoid_stable(-raw);
  const float s = sig * scale_factor;
  const int64_t p2 = b * 2 * half + idx[half + j];
  const float dy2 = dy[p2], x2 = x[p2];
  const float ds = dy2 * s;
  dx[p2] = ds;
  dbr[rb + col] = __float2bfloat16_rn(ds);
  dbr[rb + c + col] = __float2bfloat16_rn(ds * (x2 + bias) * one_m + dlogdet * one_m);
}

__global__ void __launch_bounds__(kThreads)
merge_grad_kernel(const float* dy, const float* __restrict__ dx1, const int* __restrict__ idx, float* dx, int64_t n,
                  int half) {
  const int64_t e = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  if (e >= n * half) return;
  const int64_t b = e / half;
  const int64_t p1 = b * 2 * half + idx[e - b * half];
  dx[p1] = dy[p1] + dx1[e];
}

// One CTA per image: rows[., b] and dz of image b.
__global__ void __launch_bounds__(kRedThreads)
bits_rows_kernel(const float* __restrict__ z, const float* __restrict__ logdet, float* __restrict__ rows,
                 float* __restrict__ dz, float grad_scale, int64_t n, int64_t D) {
  __shared__ float warp_tot[kRedThreads / 32];
  const int64_t b = blockIdx.x;
  const float* zb = z + b * D;
  float acc = 0.f;
  for (int64_t k = threadIdx.x; k < D; k += kRedThreads) {
    const float v = zb[k];
    acc = fmaf(v, v, acc);
    if (dz) dz[b * D + k] = grad_scale * v;
  }
  const float sumsq = block_sum(acc, warp_tot);
  if (threadIdx.x == 0) {
    const double cst = 0.5 * log(2.0 * 3.14159265358979323846) + log(127.5);
    const double norm = static_cast<double>(D) * 0.69314718055994530942;
    const double nll = 0.5 * static_cast<double>(sumsq) + static_cast<double>(D) * cst;
    const double ld = static_cast<double>(logdet[b]);
    rows[b] = static_cast<float>((nll - ld) / norm);
    rows[n + b] = static_cast<float>(nll / norm);
    rows[2 * n + b] = static_cast<float>(ld / norm);
  }
}

// One CTA: the batch means of the three rows, each summed over b in a fixed order.
__global__ void __launch_bounds__(kRedThreads) bits_means_kernel(const float* __restrict__ rows, float* means,
                                                                 int64_t n) {
  __shared__ float warp_tot[kRedThreads / 32];
  for (int k = 0; k < 3; ++k) {
    float acc = 0.f;
    for (int64_t b = threadIdx.x; b < n; b += kRedThreads) acc += rows[k * n + b];
    const float tot = block_sum(acc, warp_tot);
    if (threadIdx.x == 0) means[k] = tot / static_cast<float>(n);
    __syncthreads();     // warp_tot is reused by the next row
  }
}

inline unsigned blocks_of(int64_t n) { return static_cast<unsigned>((n + kThreads - 1) / kThreads); }

int bad(const char* fmt, const char* name) {
  set_error(fmt, name);
  return BV_ERR_INVALID;
}

int check_layout(const char* name, const void* a, const void* b, int64_t n, int H, int W, int C, int ps) {
  if (!a || !b) return bad("%s: null buffer", name);
  if (n < 1 || H < 1 || W < 1 || C < 1 || ps < 1 || H % ps || W % ps)
    return bad("%s: need n, H, W, C, ps >= 1 with H and W multiples of ps", name);
  if (n * H * W * C / kThreads + 1 > 0x7fffffffLL) return bad("%s: batch too large", name);
  return BV_OK;
}

int check_flow(const char* name, const void* a, const void* b, const void* c_, int64_t n, int T, int c) {
  if (!a || !b || !c_) return bad("%s: null buffer", name);
  if (n < 1 || T < 1 || c < 1) return bad("%s: need n, T, c >= 1", name);
  if (static_cast<int64_t>(T) * 2 * c > 0x7fffffffLL) return bad("%s: D = 2 T c exceeds int32", name);
  if (n > 0x7fffffffLL || n * T * c / kThreads + 1 > 0x7fffffffLL) return bad("%s: batch too large", name);
  return BV_OK;
}

}  // namespace
}  // namespace bv

extern "C" {

int bv_jet_dequantize_patchify(const float* image, float* z, int64_t n, int32_t H, int32_t W, int32_t C,
                               int32_t ps, uint64_t seed, uint64_t counter, int64_t offset, float noise_scale,
                               void* stream) {
  using namespace bv;
  int rc = check_layout("bv_jet_dequantize_patchify", image, z, n, H, W, C, ps);
  if (rc) return rc;
  if (offset < 0) return bad("%s: offset must be >= 0", "bv_jet_dequantize_patchify");
  const int64_t N = n * H * W * C;
  const int64_t nblk = (offset + N + 7) / 8 - offset / 8;
  dequantize_patchify_kernel<<<blocks_of(nblk), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      image, z, N, H, W, C, ps, seed, counter, offset, noise_scale);
  return check_cuda(cudaGetLastError(), "dequantize_patchify_kernel launch");
}

int bv_jet_unpatchify(const float* z, float* image, int64_t n, int32_t H, int32_t W, int32_t C, int32_t ps,
                      void* stream) {
  using namespace bv;
  int rc = check_layout("bv_jet_unpatchify", z, image, n, H, W, C, ps);
  if (rc) return rc;
  const int64_t N = n * H * W * C;
  unpatchify_kernel<<<blocks_of(N), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(z, image, N, H, W, C, ps);
  return check_cuda(cudaGetLastError(), "unpatchify_kernel launch");
}

int bv_jet_split(const float* x, const int32_t* idx, void* x1_bf16, int64_t n, int32_t T, int32_t c, void* stream) {
  using namespace bv;
  int rc = check_flow("bv_jet_split", x, idx, x1_bf16, n, T, c);
  if (rc) return rc;
  const int half = T * c;
  split_kernel<<<blocks_of(n * half), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      x, idx, static_cast<bf16*>(x1_bf16), n, half);
  return check_cuda(cudaGetLastError(), "split_kernel launch");
}

int bv_jet_coupling_fwd(const float* x, const int32_t* idx, const float* br, float* y, float* logdet, int64_t n,
                        int32_t T, int32_t c, float scale_factor, int32_t inverse, void* stream) {
  using namespace bv;
  int rc = check_flow("bv_jet_coupling_fwd", x, idx, br, n, T, c);
  if (rc) return rc;
  if (!y || !logdet) return bad("%s: null buffer", "bv_jet_coupling_fwd");
  if (!(scale_factor > 0.f)) return bad("%s: scale_factor must be > 0", "bv_jet_coupling_fwd");
  if (inverse != 0 && inverse != 1) return bad("%s: inverse must be 0 or 1", "bv_jet_coupling_fwd");
  coupling_fwd_kernel<<<static_cast<unsigned>(n), kRedThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      x, idx, br, y, logdet, T, c, scale_factor, logf(scale_factor), inverse);
  return check_cuda(cudaGetLastError(), "coupling_fwd_kernel launch");
}

int bv_jet_coupling_bwd(const float* dy, const float* x, const int32_t* idx, const float* br, float dlogdet,
                        float* dx, void* dbr_bf16, int64_t n, int32_t T, int32_t c, float scale_factor,
                        void* stream) {
  using namespace bv;
  int rc = check_flow("bv_jet_coupling_bwd", x, idx, br, n, T, c);
  if (rc) return rc;
  if (!dy || !dx || !dbr_bf16) return bad("%s: null buffer", "bv_jet_coupling_bwd");
  if (!(scale_factor > 0.f)) return bad("%s: scale_factor must be > 0", "bv_jet_coupling_bwd");
  coupling_bwd_kernel<<<blocks_of(n * T * c), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      dy, x, idx, br, dlogdet, dx, static_cast<bf16*>(dbr_bf16), n, T, c, scale_factor);
  return check_cuda(cudaGetLastError(), "coupling_bwd_kernel launch");
}

int bv_jet_merge_grad(const float* dy, const float* dx1, const int32_t* idx, float* dx, int64_t n, int32_t T,
                      int32_t c, void* stream) {
  using namespace bv;
  int rc = check_flow("bv_jet_merge_grad", dy, dx1, idx, n, T, c);
  if (rc) return rc;
  if (!dx) return bad("%s: null buffer", "bv_jet_merge_grad");
  const int half = T * c;
  merge_grad_kernel<<<blocks_of(n * half), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(dy, dx1, idx, dx, n,
                                                                                              half);
  return check_cuda(cudaGetLastError(), "merge_grad_kernel launch");
}

int bv_jet_bits(const float* z, const float* logdet, float* rows, float* means, float* dz, float grad_scale,
                int64_t n, int64_t D, void* stream) {
  using namespace bv;
  if (!z || !logdet || !rows || !means) return bad("%s: null buffer", "bv_jet_bits");
  if (n < 1 || n > 0x7fffffffLL || D < 1) return bad("%s: need 1 <= n < 2^31 and D >= 1", "bv_jet_bits");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  bits_rows_kernel<<<static_cast<unsigned>(n), kRedThreads, 0, s>>>(z, logdet, rows, dz, grad_scale, n, D);
  int rc = check_cuda(cudaGetLastError(), "bits_rows_kernel launch");
  if (rc) return rc;
  bits_means_kernel<<<1, kRedThreads, 0, s>>>(rows, means, n);
  return check_cuda(cudaGetLastError(), "bits_means_kernel launch");
}

}  // extern "C"
