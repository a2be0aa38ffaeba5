// LayerNorm forward / backward (K3).  Reference: flax.linen.LayerNorm as called at
// models/vit.py:92,103,160,181 and models/mlp_mixer.py:48,53,79 -- eps = 1e-6,
// statistics in fp32 with the "fast variance" form var = max(E[x^2] - E[x]^2, 0).
//
// HBM-bound: one warp per row, 16-byte vector loads, the row stays in registers
// between the statistics pass and the normalise pass (one read + one write of
// [rows, d]).  The backward also folds in the residual-branch gradient and the
// column sums that are the bias gradients of the GEMMs upstream of the residual
// stream, so those need no extra pass over HBM.
#include "common.cuh"
#include "host_utils.h"

namespace bv {
namespace {

__device__ __forceinline__ void load8(const void* base, int dtype, int64_t elem_off, float (&v)[8]) {
  if (dtype == DT_BF16) {
    const uint4 q = *reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(base) + elem_off);
    v[0] = bf16_lo(q.x); v[1] = bf16_hi(q.x); v[2] = bf16_lo(q.y); v[3] = bf16_hi(q.y);
    v[4] = bf16_lo(q.z); v[5] = bf16_hi(q.z); v[6] = bf16_lo(q.w); v[7] = bf16_hi(q.w);
  } else {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem_off);
    const float4 a = p[0], b = p[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
}
__device__ __forceinline__ void store8(void* base, int dtype, int64_t elem_off, const float (&v)[8]) {
  if (dtype == DT_BF16) {
    uint4 q;
    q.x = pack_bf16(v[0], v[1]); q.y = pack_bf16(v[2], v[3]);
    q.z = pack_bf16(v[4], v[5]); q.w = pack_bf16(v[6], v[7]);
    *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(base) + elem_off) = q;
  } else {
    float4* p = reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + elem_off);
    p[0] = make_float4(v[0], v[1], v[2], v[3]);
    p[1] = make_float4(v[4], v[5], v[6], v[7]);
  }
}
__device__ __forceinline__ void load8f(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

constexpr int LN_THREADS = 256;
constexpr int LN_WARPS = LN_THREADS / 32;

template <int NCH>
__global__ void __launch_bounds__(LN_THREADS)
ln_fwd_kernel(const void* __restrict__ x, int x_dt, const float* __restrict__ scale,
              const float* __restrict__ bias, void* __restrict__ y, int y_dt,
              float* __restrict__ mean_out, float* __restrict__ rstd_out, int64_t rows, int d,
              float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * LN_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nchunks = d >> 3;
  float v[NCH][8];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      load8(x, x_dt, row * d + c * 8, v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s1 += v[i][j]; s2 += v[i][j] * v[i][j]; }
    }
  }
  s1 = warp_sum(s1);
  s2 = warp_sum(s2);
  const float inv_d = 1.0f / static_cast<float>(d);
  const float mean = s1 * inv_d;
  const float var = fmaxf(s2 * inv_d - mean * mean, 0.f);
  const float rstd = rsqrtf(var + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      float g[8], b[8], o[8];
      load8f(scale + c * 8, g);
      load8f(bias + c * 8, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * g[j] + b[j];
      store8(y, y_dt, row * d + c * 8, o);
    }
  }
}

// bf16 -> bf16 streaming forward: persistent warps walk the rows with a grid stride, keep scale and
// bias in registers (re-reading them per row costs 4x the L1 traffic of the row itself) and keep
// the load of the next row in flight while the current one is reduced and written.
template <int NCH>
__global__ void __launch_bounds__(LN_THREADS, NCH <= 3 ? 2 : 1)
ln_fwd_stream_kernel(const bf16* __restrict__ x, const float* __restrict__ scale,
                     const float* __restrict__ bias, bf16* __restrict__ y,
                     float* __restrict__ mean_out, float* __restrict__ rstd_out, int64_t rows, int d,
                     float eps) {
  const int lane = threadIdx.x & 31;
  const int nchunks = d >> 3;
  float g[NCH][8], b[NCH][8];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
#pragma unroll
    for (int j = 0; j < 8; ++j) { g[i][j] = 0.f; b[i][j] = 0.f; }
    if (c < nchunks) { load8f(scale + c * 8, g[i]); load8f(bias + c * 8, b[i]); }
  }
  const int64_t stride = static_cast<int64_t>(gridDim.x) * LN_WARPS;
  const int64_t row0 = static_cast<int64_t>(blockIdx.x) * LN_WARPS + (threadIdx.x >> 5);
  const float inv_d = 1.0f / static_cast<float>(d);
  uint4 buf[2][NCH];
  auto fetch = [&](int64_t row, uint4 (&q)[NCH]) {
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      q[i] = make_uint4(0u, 0u, 0u, 0u);
      if (row < rows && c < nchunks) q[i] = ld_nc_na(reinterpret_cast<const uint4*>(x + row * d + c * 8));
    }
  };
  auto process = [&](int64_t row, uint4 (&q)[NCH]) {
    float v[NCH][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      v[i][0] = bf16_lo(q[i].x); v[i][1] = bf16_hi(q[i].x); v[i][2] = bf16_lo(q[i].y); v[i][3] = bf16_hi(q[i].y);
      v[i][4] = bf16_lo(q[i].z); v[i][5] = bf16_hi(q[i].z); v[i][6] = bf16_lo(q[i].w); v[i][7] = bf16_hi(q[i].w);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s1 += v[i][j]; s2 += v[i][j] * v[i][j]; }   // padded chunks are zero
    }
    fetch(row + 2 * stride, q);        // this buffer is free again: refill it two rows ahead
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    const float mean = s1 * inv_d;
    const float var = fmaxf(s2 * inv_d - mean * mean, 0.f);
    const float rstd = rsqrtf(var + eps);
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nchunks) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * g[i][j] + b[i][j];
        store8(y, DT_BF16, row * d + c * 8, o);
      }
    }
  };
  fetch(row0, buf[0]);
  fetch(row0 + stride, buf[1]);
  for (int64_t row = row0; row < rows; row += 2 * stride) {
    process(row, buf[0]);
    if (row + stride < rows) process(row + stride, buf[1]);
  }
}

// dx = dres + rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * scale
// dscale += sum_rows dy * xhat ; dbias += sum_rows dy ; dx_colsum += sum_rows dx
template <int NCH>
__global__ void __launch_bounds__(LN_THREADS)
ln_bwd_kernel(const void* __restrict__ dy, int dy_dt, const void* __restrict__ x, int x_dt,
              const float* __restrict__ scale, const float* __restrict__ mean_in,
              const float* __restrict__ rstd_in, const void* __restrict__ dres,
              void* __restrict__ dx, int dx_dt, float* __restrict__ dscale,
              float* __restrict__ dbias, float* __restrict__ dx_colsum, int64_t rows, int d) {
  extern __shared__ float red[];   // [3][d]
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nchunks = d >> 3;
  const bool want_cs = dx_colsum != nullptr;
  for (int i = threadIdx.x; i < 3 * d; i += LN_THREADS) red[i] = 0.f;
  __syncthreads();

  float acc_g[NCH][8], acc_b[NCH][8], acc_c[NCH][8];
  float g[NCH][8];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc_g[i][j] = 0.f; acc_b[i][j] = 0.f; acc_c[i][j] = 0.f; g[i][j] = 0.f; }
    if (c < nchunks) load8f(scale + c * 8, g[i]);
  }
  const float inv_d = 1.0f / static_cast<float>(d);
  const int64_t warp_stride = static_cast<int64_t>(gridDim.x) * LN_WARPS;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * LN_WARPS + warp; row < rows;
       row += warp_stride) {
    const float mean = mean_in[row], rstd = rstd_in[row];
    float xh[NCH][8], gy[NCH][8];
    float c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nchunks) {
        float xv[8], dv[8];
        load8(x, x_dt, row * d + c * 8, xv);
        load8(dy, dy_dt, row * d + c * 8, dv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[i][j] = (xv[j] - mean) * rstd;
          gy[i][j] = dv[j] * g[i][j];
          c1 += gy[i][j];
          c2 += gy[i][j] * xh[i][j];
          acc_g[i][j] += dv[j] * xh[i][j];
          acc_b[i][j] += dv[j];
        }
      }
    }
    c1 = warp_sum(c1) * inv_d;
    c2 = warp_sum(c2) * inv_d;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nchunks) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (gy[i][j] - c1 - xh[i][j] * c2);
        if (dres != nullptr) {
          float r[8];
          load8(dres, dx_dt, row * d + c * 8, r);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r[j];
        }
        if (dx_dt == DT_BF16) {
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = round_bf16(o[j]);
        }
        store8(dx, dx_dt, row * d + c * 8, o);
        if (want_cs) {
#pragma unroll
          for (int j = 0; j < 8; ++j) acc_c[i][j] += o[j];
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        atomicAdd(&red[c * 8 + j], acc_g[i][j]);
        atomicAdd(&red[d + c * 8 + j], acc_b[i][j]);
        if (want_cs) atomicAdd(&red[2 * d + c * 8 + j], acc_c[i][j]);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < d; i += LN_THREADS) {
    if (dscale) atomicAdd(dscale + i, red[i]);
    if (dbias) atomicAdd(dbias + i, red[d + i]);
    if (want_cs) atomicAdd(dx_colsum + i, red[2 * d + i]);
  }
}

// ---------------------------------------------------------------------------
// bf16 fast path of the backward: same math, but every warp streams its rows through a private
// shared-memory ring filled by cp.async (16 B per lane per request), DEPTH rows ahead of the
// arithmetic.  Memory-level parallelism then no longer depends on registers: 8 warps x
// (DEPTH-1) rows x 4.5 KB are in flight per SM, enough to cover HBM latency.
// ---------------------------------------------------------------------------
constexpr int LNP_DEPTH = 3;
// 12 warps up to d = 768 (the kernel is issue-bound, more warps = more IPC); 8 warps for d <= 1024 so
// that the per-warp rings (DEPTH x 3 arrays x 2 KB) still fit in shared memory
template <int NCH> struct LnpCfg { static constexpr int WARPS = NCH <= 3 ? 12 : 8; static constexpr int THREADS = WARPS * 32; };

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void lds8(uint32_t addr, float (&v)[8]) {
  uint4 q;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
               : "=r"(q.x), "=r"(q.y), "=r"(q.z), "=r"(q.w) : "r"(addr));
  v[0] = bf16_lo(q.x); v[1] = bf16_hi(q.x); v[2] = bf16_lo(q.y); v[3] = bf16_hi(q.y);
  v[4] = bf16_lo(q.z); v[5] = bf16_hi(q.z); v[6] = bf16_lo(q.w); v[7] = bf16_hi(q.w);
}

template <int NCH, bool HAS_RES>
__global__ void __launch_bounds__(LnpCfg<NCH>::THREADS, 1)
ln_bwd_pipe_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                   const float* __restrict__ scale, const float* __restrict__ mean_in,
                   const float* __restrict__ rstd_in, const bf16* __restrict__ dres,
                   bf16* __restrict__ dx, float* __restrict__ dscale, float* __restrict__ dbias,
                   float* __restrict__ dx_colsum, int64_t rows, int d) {
  extern __shared__ __align__(16) uint8_t smem_ln[];
  constexpr int NARR = HAS_RES ? 3 : 2;
  constexpr int LNP_THREADS = LnpCfg<NCH>::THREADS, LNP_WARPS = LnpCfg<NCH>::WARPS;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nchunks = d >> 3;
  const bool want_cs = dx_colsum != nullptr;
  float* red = reinterpret_cast<float*>(smem_ln);                       // [3][d]
  const int row_bytes = d * 2;
  const uint32_t ring = smem_u32(smem_ln) + 3 * d * 4 + warp * (LNP_DEPTH * NARR * row_bytes);
  for (int i = threadIdx.x; i < 3 * d; i += LNP_THREADS) red[i] = 0.f;
  __syncthreads();

  float acc_g[NCH][8], acc_b[NCH][8], acc_c[NCH][8];
  float g[NCH][8];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc_g[i][j] = 0.f; acc_b[i][j] = 0.f; acc_c[i][j] = 0.f; g[i][j] = 0.f; }
    if (c < nchunks) load8f(scale + c * 8, g[i]);
  }
  const float inv_d = 1.0f / static_cast<float>(d);
  const int64_t warp_stride = static_cast<int64_t>(gridDim.x) * LNP_WARPS;
  const int64_t row0 = static_cast<int64_t>(blockIdx.x) * LNP_WARPS + warp;

  auto issue = [&](int64_t row, int slot) {
    if (row < rows) {
      const uint32_t sbase = ring + slot * (NARR * row_bytes);
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        const int c = lane + 32 * i;
        if (c < nchunks) {
          const int64_t off = row * d + c * 8;
          cp_async16(sbase + c * 16, x + off);
          cp_async16(sbase + row_bytes + c * 16, dy + off);
          if (HAS_RES) cp_async16(sbase + 2 * row_bytes + c * 16, dres + off);
        }
      }
    }
    cp_async_commit();
  };

#pragma unroll
  for (int k = 0; k < LNP_DEPTH - 1; ++k) issue(row0 + k * warp_stride, k);

  int slot = 0;
  for (int64_t row = row0; row < rows; row += warp_stride) {
    issue(row + (LNP_DEPTH - 1) * warp_stride, (slot + LNP_DEPTH - 1) % LNP_DEPTH);
    cp_async_wait<LNP_DEPTH - 1>();
    __syncwarp();
    const float mean = mean_in[row], rstd = rstd_in[row];
    const float nmr = -mean * rstd;
    const uint32_t sbase = ring + slot * (NARR * row_bytes);
    float c1 = 0.f, c2 = 0.f;
    // xhat and g = dy * scale stay in registers between the two passes (the kernel is bound by
    // instruction issue, not by HBM: re-reading and re-converting them costs a fifth of its time)
    float xh[NCH][8], gy[NCH][8];
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
#pragma unroll
      for (int j = 0; j < 8; ++j) { xh[i][j] = 0.f; gy[i][j] = 0.f; }
      if (c < nchunks) {
        float xv[8], dv[8];
        lds8(sbase + c * 16, xv);
        lds8(sbase + row_bytes + c * 16, dv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[i][j] = fmaf(xv[j], rstd, nmr);
          gy[i][j] = dv[j] * g[i][j];
          c1 += gy[i][j];
          c2 = fmaf(gy[i][j], xh[i][j], c2);
          acc_g[i][j] = fmaf(dv[j], xh[i][j], acc_g[i][j]);
          acc_b[i][j] += dv[j];
        }
      }
    }
    c1 = warp_sum(c1) * inv_d;
    c2 = warp_sum(c2) * inv_d;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nchunks) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (gy[i][j] - c1 - xh[i][j] * c2);
        if (HAS_RES) {
          float r[8];
          lds8(sbase + 2 * row_bytes + c * 16, r);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r[j];
        }
        store8(dx, DT_BF16, row * d + c * 8, o);
        if (want_cs) {
          // column sums of dx (upstream bias gradient) from the fp32 values, before the bf16 rounding
#pragma unroll
          for (int j = 0; j < 8; ++j) acc_c[i][j] += o[j];
        }
      }
    }
    __syncwarp();   // all lanes done with this slot before it is refilled next iteration
    slot = (slot + 1) % LNP_DEPTH;
  }
  cp_async_wait<0>();
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        atomicAdd(&red[c * 8 + j], acc_g[i][j]);
        atomicAdd(&red[d + c * 8 + j], acc_b[i][j]);
        if (want_cs) atomicAdd(&red[2 * d + c * 8 + j], acc_c[i][j]);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < d; i += LNP_THREADS) {
    if (dscale) atomicAdd(dscale + i, red[i]);
    if (dbias) atomicAdd(dbias + i, red[d + i]);
    if (want_cs) atomicAdd(dx_colsum + i, red[2 * d + i]);
  }
}

template <int NCH>
int launch_ln_bwd_pipe(const void* dy, const void* x, const float* scale, const float* mean,
                       const float* rstd, const void* dres, void* dx, float* dscale, float* dbias,
                       float* dx_colsum, int64_t rows, int d, cudaStream_t s) {
  const int narr = dres ? 3 : 2;
  constexpr int LNP_THREADS = LnpCfg<NCH>::THREADS, LNP_WARPS = LnpCfg<NCH>::WARPS;
  const size_t smem = 3 * static_cast<size_t>(d) * 4 +
                      static_cast<size_t>(LNP_WARPS) * LNP_DEPTH * narr * d * 2;
  int64_t blocks = (rows + LNP_WARPS - 1) / LNP_WARPS;
  const int64_t cap = num_sms();
  if (blocks > cap) blocks = cap;
  cudaError_t e;
  if (dres) {
    auto k = ln_bwd_pipe_kernel<NCH, true>;
    e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(ln_bwd_pipe)");
    k<<<(unsigned)blocks, LNP_THREADS, smem, s>>>(
        reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x), scale, mean, rstd,
        reinterpret_cast<const bf16*>(dres), reinterpret_cast<bf16*>(dx), dscale, dbias, dx_colsum, rows, d);
  } else {
    auto k = ln_bwd_pipe_kernel<NCH, false>;
    e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(ln_bwd_pipe)");
    k<<<(unsigned)blocks, LNP_THREADS, smem, s>>>(
        reinterpret_cast<const bf16*>(dy), reinterpret_cast<const bf16*>(x), scale, mean, rstd,
        nullptr, reinterpret_cast<bf16*>(dx), dscale, dbias, dx_colsum, rows, d);
  }
  return check_cuda(cudaGetLastError(), "ln_bwd_pipe_kernel launch");
}

int check_ln(int64_t rows, int d, const char* who) {
  if (rows < 0 || d <= 0 || d % 8 != 0 || d > 2048) {
    set_error("%s: need rows >= 0 and d %% 8 == 0, d <= 2048 (got rows=%lld d=%d)", who,
              (long long)rows, d);
    return BV_ERR_INVALID;
  }
  return BV_OK;
}

}  // namespace
}  // namespace bv

extern "C" {

int bv_layernorm_fwd(const void* x, int x_dt, const float* scale, const float* bias, void* y,
                     int y_dt, float* mean, float* rstd, int64_t rows, int32_t d, float eps,
                     void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc = check_ln(rows, d, "bv_layernorm_fwd");
  if (rc) return rc;
  if (rows == 0) return BV_OK;
  const int nch = (d / 8 + 31) / 32;
  if (x_dt == DT_BF16 && y_dt == DT_BF16 && rows >= 4096 && nch <= 4) {
    // streaming fast path: two persistent blocks per SM (one for d > 768: twice the registers per row)
    const unsigned pgrid = static_cast<unsigned>((nch <= 3 ? 2 : 1) * num_sms());
    const bf16* xb = reinterpret_cast<const bf16*>(x);
    bf16* yb = reinterpret_cast<bf16*>(y);
    switch (nch) {
      case 1: ln_fwd_stream_kernel<1><<<pgrid, LN_THREADS, 0, s>>>(xb, scale, bias, yb, mean, rstd, rows, d, eps); break;
      case 2: ln_fwd_stream_kernel<2><<<pgrid, LN_THREADS, 0, s>>>(xb, scale, bias, yb, mean, rstd, rows, d, eps); break;
      case 4: ln_fwd_stream_kernel<4><<<pgrid, LN_THREADS, 0, s>>>(xb, scale, bias, yb, mean, rstd, rows, d, eps); break;
      default: ln_fwd_stream_kernel<3><<<pgrid, LN_THREADS, 0, s>>>(xb, scale, bias, yb, mean, rstd, rows, d, eps); break;
    }
    return check_cuda(cudaGetLastError(), "ln_fwd_stream_kernel launch");
  }
  const unsigned grid = static_cast<unsigned>((rows + LN_WARPS - 1) / LN_WARPS);
#define LN_FWD_CASE(N)                                                                        \
  case N:                                                                                     \
    ln_fwd_kernel<N><<<grid, LN_THREADS, 0, s>>>(x, x_dt, scale, bias, y, y_dt, mean, rstd,   \
                                                 rows, d, eps);                               \
    break;
  switch (nch) {
    LN_FWD_CASE(1) LN_FWD_CASE(2) LN_FWD_CASE(3) LN_FWD_CASE(4)
    LN_FWD_CASE(5) LN_FWD_CASE(6) LN_FWD_CASE(7) LN_FWD_CASE(8)
    default: set_error("bv_layernorm_fwd: d too large"); return BV_ERR_INVALID;
  }
#undef LN_FWD_CASE
  return check_cuda(cudaGetLastError(), "ln_fwd_kernel launch");
}

int bv_layernorm_bwd(const void* dy, int dy_dt, const void* x, int x_dt, const float* scale,
                     const float* mean, const float* rstd, const void* dres, void* dx,
                     int dx_dt, float* dscale, float* dbias, float* dx_colsum, int64_t rows,
                     int32_t d, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc = check_ln(rows, d, "bv_layernorm_bwd");
  if (rc) return rc;
  if (rows == 0) return BV_OK;
  const int nch = (d / 8 + 31) / 32;
  {
    // streaming bf16 fast path (cp.async ring); the generic kernel below covers fp32 operands,
    // small problems and widths whose ring does not fit in shared memory
    const size_t ring = 3 * static_cast<size_t>(d) * 4 +
                        static_cast<size_t>(nch <= 3 ? 12 : 8) * LNP_DEPTH * (dres ? 3 : 2) * d * 2;
    if (dy_dt == DT_BF16 && x_dt == DT_BF16 && dx_dt == DT_BF16 && rows >= 4096 && nch <= 4 &&
        ring <= 220 * 1024) {
      switch (nch) {
        case 4: return launch_ln_bwd_pipe<4>(dy, x, scale, mean, rstd, dres, dx, dscale, dbias, dx_colsum, rows, d, s);
        case 1: return launch_ln_bwd_pipe<1>(dy, x, scale, mean, rstd, dres, dx, dscale, dbias, dx_colsum, rows, d, s);
        case 2: return launch_ln_bwd_pipe<2>(dy, x, scale, mean, rstd, dres, dx, dscale, dbias, dx_colsum, rows, d, s);
        default: return launch_ln_bwd_pipe<3>(dy, x, scale, mean, rstd, dres, dx, dscale, dbias, dx_colsum, rows, d, s);
      }
    }
  }
  int64_t blocks = (rows + LN_WARPS - 1) / LN_WARPS;
  const int64_t cap = static_cast<int64_t>(num_sms()) * 2;   // 2 resident blocks/SM (register-bound)
  if (blocks > cap) blocks = cap;
  const size_t smem = 3 * static_cast<size_t>(d) * sizeof(float);
#define LN_BWD_CASE(N)                                                                         \
  case N:                                                                                      \
    ln_bwd_kernel<N><<<(unsigned)blocks, LN_THREADS, smem, s>>>(                               \
        dy, dy_dt, x, x_dt, scale, mean, rstd, dres, dx, dx_dt, dscale, dbias, dx_colsum, rows, d); \
    break;
  switch (nch) {
    LN_BWD_CASE(1) LN_BWD_CASE(2) LN_BWD_CASE(3) LN_BWD_CASE(4)
    LN_BWD_CASE(5) LN_BWD_CASE(6) LN_BWD_CASE(7) LN_BWD_CASE(8)
    default:
      set_error("bv_layernorm_bwd: d=%d > 2048 not supported", d);
      return BV_ERR_UNSUPPORTED;
  }
#undef LN_BWD_CASE
  return check_cuda(cudaGetLastError(), "ln_bwd_kernel launch");
}

}  // extern "C"
