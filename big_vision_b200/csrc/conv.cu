// Convolutions and the element-wise kernels of the BiT ResNet-v2 (include/bv_conv.h).
//
// The three convolution entry points describe each call as an implicit GEMM (conv_gemm.h) that gemm.cu's
// persistent kernel runs with the activation read through TMA in im2col mode:
//   forward         rows = output pixels, k = (tap, cin), B = the HWIO kernel read MN-major;
//   data gradient   rows = input pixels of one (row, column) parity class, k = (tap, cout) over the taps that
//                   reach that class, A = dy, B = the same kernel read K-major (its [cin, cout] slice of the
//                   tap as rows = cin); at stride 1 there is one class, the flipped-kernel convolution;
//   kernel gradient rows = (tap, cin), k = output pixels, split over pixels with fp32 atomics.
// GroupNorm, weight standardisation, the max pool and the root block's patch extraction are bandwidth-
// bound kernels with fixed-order block sums.
#include "../../include/bv_conv.h"

#include <cuda_bf16.h>
#include <math.h>

#include "common.cuh"
#include "conv_gemm.h"
#include "host_utils.h"

namespace bv {
namespace {

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
int out_size(int h, int k, int stride) { return (h + 2 * (k / 2) - k) / stride + 1; }

int check_conv(const char* fn, const bv_conv_args* a) {
  if (!a) {
    set_error("%s: null args", fn);
    return BV_ERR_INVALID;
  }
  if (a->k != 1 && a->k != 3 && a->k != 7) {
    set_error("%s: k = %d; supported are 1, 3 and 7", fn, a->k);
    return BV_ERR_INVALID;
  }
  if (a->stride != 1 && a->stride != 2) {
    set_error("%s: stride %d; supported are 1 and 2", fn, a->stride);
    return BV_ERR_INVALID;
  }
  if (a->cin < 64 || a->cout < 64 || a->cin % 64 || a->cout % 64) {
    set_error("%s: cin %d and cout %d must be positive multiples of 64", fn, a->cin, a->cout);
    return BV_ERR_INVALID;
  }
  if (a->n < 1 || a->h < 1 || a->w < 1 || a->h > 32767 || a->w > 32767) {
    set_error("%s: need n >= 1 and 1 <= h, w <= 32767", fn);
    return BV_ERR_INVALID;
  }
  const int ho = out_size(a->h, a->k, a->stride), wo = out_size(a->w, a->k, a->stride);
  const long long big = a->n * (long long)a->h * a->w, small = a->n * (long long)ho * wo;
  if (big > 0x7fffffffLL || small * a->cout > (1LL << 40) || big * a->cin > (1LL << 40)) {
    set_error("%s: tensor too large", fn);
    return BV_ERR_INVALID;
  }
  return BV_OK;
}

int need(const char* fn, const void* p, const char* what) {
  if (!p) {
    set_error("%s: null %s", fn, what);
    return BV_ERR_INVALID;
  }
  if (!aligned16(p)) {
    set_error("%s: %s must be 16-byte aligned", fn, what);
    return BV_ERR_INVALID;
  }
  return BV_OK;
}

// the forward's implicit GEMM over x (also the kernel gradient's, with wgrad set and b = dy)
ConvGemm forward_gemm(const bv_conv_args& a) {
  ConvGemm g = {};
  const int p = a.k / 2;
  g.x = a.x; g.n = a.n; g.h = a.h; g.w = a.w; g.c = a.cin;
  g.gh = out_size(a.h, a.k, a.stride); g.gw = out_size(a.w, a.k, a.stride);
  g.lw = g.lh = -p; g.stride = a.stride;
  g.ntaps = a.k * a.k;
  for (int kh = 0; kh < a.k; ++kh)
    for (int kw = 0; kw < a.k; ++kw) g.taps[kh * a.k + kw] = {kw, kh, (kh * a.k + kw) * a.cin};
  return g;
}

// One parity class (ph, pw) of the data gradient: input rows hi = s * hp + ph get contributions from the filter
// rows kh with (ph + p - kh) divisible by s, from dy row hp + (ph + p - kh) / s.  Returns the class's grid
// (gh, gw) and fills its taps (none when no filter row or column reaches it: k = 1 at stride 2).
ConvGemm dgrad_gemm(const bv_conv_args& a, int ph, int pw) {
  ConvGemm g = {};
  const int p = a.k / 2, s = a.stride;
  g.x = a.dy; g.n = a.n; g.c = a.cout;
  g.h = out_size(a.h, a.k, s); g.w = out_size(a.w, a.k, s);
  g.gh = (a.h - ph + s - 1) / s; g.gw = (a.w - pw + s - 1) / s;
  g.stride = 1;
  int dminh = 1 << 20, dminw = 1 << 20;
  for (int kh = 0; kh < a.k; ++kh)
    if ((ph + p - kh) % s == 0 && (ph + p - kh) / s < dminh) dminh = (ph + p - kh) / s;
  for (int kw = 0; kw < a.k; ++kw)
    if ((pw + p - kw) % s == 0 && (pw + p - kw) / s < dminw) dminw = (pw + p - kw) / s;
  g.lh = dminh; g.lw = dminw;
  g.ntaps = 0;
  for (int kh = 0; kh < a.k; ++kh) {
    if ((ph + p - kh + 2 * s) % s) continue;
    for (int kw = 0; kw < a.k; ++kw) {
      if ((pw + p - kw + 2 * s) % s) continue;
      g.taps[g.ntaps++] = {(pw + p - kw) / s - dminw, (ph + p - kh) / s - dminh, (kh * a.k + kw) * a.cin};
    }
  }
  g.b = a.kernel; g.b_rows = (int64_t)a.k * a.k * a.cin; g.b_cols = a.cout; g.b_mn = 0;
  g.N = a.cin;
  return g;
}

// dx[img, hi, wi, :] = the parity class's output (or 0 for a class no tap reaches) (+ resid), 8 channels
// per thread
struct ScatterParams {
  int64_t n;
  int h, w, c;
  int64_t off[4];      // element offset of each class's [n, gh, gw, c] block in the workspace
  int gh[2], gw[2];
  int has[4];
};

__global__ void __launch_bounds__(256)
dgrad_scatter_kernel(const bf16* __restrict__ ws, const bf16* __restrict__ resid, bf16* __restrict__ dx,
                     ScatterParams sp) {
  const int64_t total = sp.n * sp.h * sp.w * (sp.c / 8);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % (sp.c / 8));
    const int64_t pix = i / (sp.c / 8);
    const int wi = (int)(pix % sp.w);
    const int64_t t = pix / sp.w;
    const int hi = (int)(t % sp.h);
    const int64_t img = t / sp.h;
    const int ph = hi & 1, pw = wi & 1, q = 2 * ph + pw;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    // selects instead of indexing, which would copy the parameter arrays to the stack
    const int has = q == 0 ? sp.has[0] : q == 1 ? sp.has[1] : q == 2 ? sp.has[2] : sp.has[3];
    const int64_t off = q == 0 ? sp.off[0] : q == 1 ? sp.off[1] : q == 2 ? sp.off[2] : sp.off[3];
    const int gh = ph ? sp.gh[1] : sp.gh[0], gw = pw ? sp.gw[1] : sp.gw[0];
    if (has) {
      const int64_t src = off + ((img * gh + (hi >> 1)) * gw + (wi >> 1)) * sp.c + 8 * c8;
      const uint4 u = *reinterpret_cast<const uint4*>(ws + src);
      const uint32_t* uw = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) { v[2 * j] = bf16_lo(uw[j]); v[2 * j + 1] = bf16_hi(uw[j]); }
    }
    if (resid) {
      const uint4 u = *reinterpret_cast<const uint4*>(resid + pix * sp.c + 8 * c8);
      const uint32_t* uw = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) { v[2 * j] += bf16_lo(uw[j]); v[2 * j + 1] += bf16_hi(uw[j]); }
    }
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) ow[j] = pack_bf16(v[2 * j], v[2 * j + 1]);
    *reinterpret_cast<uint4*>(dx + pix * sp.c + 8 * c8) = o;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Weight standardisation: block = 32 columns x 8 row lanes; each column's sums are fixed-order (row lane
// r sums rows r, r + 8, ... in order; the 8 lane sums are added in order).
constexpr int WS_ROWS = 8;

__device__ __forceinline__ float col_sum(float v, float (*sh)[33]) {
  sh[threadIdx.y][threadIdx.x] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int r = 0; r < WS_ROWS; ++r) s += sh[r][threadIdx.x];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(256)
weight_std_fwd_kernel(const float* __restrict__ w, int64_t rows, int cout, bf16* __restrict__ ws,
                      float* __restrict__ mean_out, float* __restrict__ rstd_out) {
  __shared__ float sh[WS_ROWS][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const bool in = col < cout;
  float s = 0.f;
  if (in)
    for (int64_t r = threadIdx.y; r < rows; r += WS_ROWS) s += w[r * cout + col];
  const float mean = col_sum(s, sh) / (float)rows;
  float q = 0.f;
  if (in)
    for (int64_t r = threadIdx.y; r < rows; r += WS_ROWS) {
      const float d = w[r * cout + col] - mean;
      q += d * d;
    }
  const float var = col_sum(q, sh) / (float)rows;
  const float rstd = 1.f / sqrtf(var + 1e-10f);
  if (!in) return;
  for (int64_t r = threadIdx.y; r < rows; r += WS_ROWS) ws[r * cout + col] = __float2bfloat16_rn((w[r * cout + col] - mean) * rstd);
  if (threadIdx.y == 0) {
    mean_out[col] = mean;
    rstd_out[col] = rstd;
  }
}

__global__ void __launch_bounds__(256)
weight_std_bwd_kernel(const float* __restrict__ w, const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                      const float* __restrict__ g, int64_t rows, int cout, float* __restrict__ dw) {
  __shared__ float sh[WS_ROWS][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const bool in = col < cout;
  const float mean = in ? mean_in[col] : 0.f, rstd = in ? rstd_in[col] : 0.f;
  float sg = 0.f, sgx = 0.f;
  if (in)
    for (int64_t r = threadIdx.y; r < rows; r += WS_ROWS) {
      const float gv = g[r * cout + col];
      sg += gv;
      sgx += gv * (w[r * cout + col] - mean) * rstd;
    }
  const float mg = col_sum(sg, sh) / (float)rows;
  const float mgx = col_sum(sgx, sh) / (float)rows;
  if (!in) return;
  for (int64_t r = threadIdx.y; r < rows; r += WS_ROWS) {
    const float xh = (w[r * cout + col] - mean) * rstd;
    dw[r * cout + col] = rstd * (g[r * cout + col] - mg - xh * mgx);
  }
}

// ---------------------------------------------------------------------------------------------------------
// GroupNorm: one block per (group, image).  Element e of the group is pixel e / cg, channel e % cg; a thread
// t < step = (256 / cg) * cg visits e = t, t + step, ..., so its channel is fixed (t % cg).
constexpr int GN_THREADS = 256;
constexpr int GN_GROUPS = 32;

__global__ void __launch_bounds__(GN_THREADS)
groupnorm_fwd_kernel(const bf16* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ bias,
                     bf16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int64_t hw,
                     int c, int relu) {
  __shared__ float sh[32];
  const int grp = blockIdx.x, cg = c / GN_GROUPS, step = (GN_THREADS / cg) * cg;
  const int64_t img = blockIdx.y, count = hw * cg;
  const bf16* xb = x + img * hw * c + grp * cg;
  bf16* yb = y + img * hw * c + grp * cg;
  const int t = threadIdx.x, ch = t % cg;
  const bool act = t < step;
  float s = 0.f;
  if (act)
    for (int64_t e = t; e < count; e += step) s += __bfloat162float(xb[(e / cg) * c + ch]);
  const float mean = block_sum(s, sh) / (float)count;
  float q = 0.f;
  if (act)
    for (int64_t e = t; e < count; e += step) {
      const float d = __bfloat162float(xb[(e / cg) * c + ch]) - mean;
      q += d * d;
    }
  const float var = block_sum(q, sh) / (float)count;
  const float rstd = 1.f / sqrtf(var + 1e-5f);
  if (act) {
    const float g = scale[grp * cg + ch], b = bias[grp * cg + ch];
    for (int64_t e = t; e < count; e += step) {
      const int64_t o = (e / cg) * c + ch;
      float z = (__bfloat162float(xb[o]) - mean) * rstd * g + b;
      if (relu) z = fmaxf(z, 0.f);
      yb[o] = __float2bfloat16_rn(z);
    }
  }
  if (t == 0) {
    mean_out[img * GN_GROUPS + grp] = mean;
    rstd_out[img * GN_GROUPS + grp] = rstd;
  }
}

__global__ void __launch_bounds__(GN_THREADS)
groupnorm_bwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy, const float* __restrict__ scale,
                     const float* __restrict__ bias, const float* __restrict__ mean_in,
                     const float* __restrict__ rstd_in, const bf16* __restrict__ dx_add, bf16* __restrict__ dx,
                     float* __restrict__ dscale, float* __restrict__ dbias, int64_t hw, int c, int relu) {
  __shared__ float sh[64];
  __shared__ float shc[2][GN_THREADS];
  const int grp = blockIdx.x, cg = c / GN_GROUPS, step = (GN_THREADS / cg) * cg;
  const int64_t img = blockIdx.y, count = hw * cg, base = img * hw * c + grp * cg;
  const int t = threadIdx.x, ch = t % cg;
  const bool act = t < step;
  const float mean = mean_in[img * GN_GROUPS + grp], rstd = rstd_in[img * GN_GROUPS + grp];
  const float g = act ? scale[grp * cg + ch] : 0.f, b = act ? bias[grp * cg + ch] : 0.f;
  // pass 1: sum(dz * g), sum(dz * g * x_hat) over the group; per-channel sum(dz * x_hat), sum(dz)
  float v[2] = {0.f, 0.f};
  float ds = 0.f, db = 0.f;
  if (act)
    for (int64_t e = t; e < count; e += step) {
      const int64_t o = base + (e / cg) * c + ch;
      const float xh = (__bfloat162float(x[o]) - mean) * rstd;
      float dz = __bfloat162float(dy[o]);
      if (relu && !(xh * g + b > 0.f)) dz = 0.f;
      v[0] += dz * g;
      v[1] += dz * g * xh;
      ds += dz * xh;
      db += dz;
    }
  block_sum(v, sh);
  shc[0][t] = ds;
  shc[1][t] = db;
  __syncthreads();
  if (t < cg) {
    float a0 = 0.f, a1 = 0.f;
    for (int j = t; j < step; j += cg) { a0 += shc[0][j]; a1 += shc[1][j]; }
    atomicAdd(dscale + grp * cg + t, a0);
    atomicAdd(dbias + grp * cg + t, a1);
  }
  const float m1 = v[0] / (float)count, m2 = v[1] / (float)count;
  if (!act) return;
  for (int64_t e = t; e < count; e += step) {
    const int64_t o = base + (e / cg) * c + ch;
    const float xh = (__bfloat162float(x[o]) - mean) * rstd;
    float dz = __bfloat162float(dy[o]);
    if (relu && !(xh * g + b > 0.f)) dz = 0.f;
    float r = rstd * (dz * g - m1 - xh * m2);
    if (dx_add) r += __bfloat162float(dx_add[o]);
    dx[o] = __float2bfloat16_rn(r);
  }
}

// ---------------------------------------------------------------------------------------------------------
// Max pool 3 x 3 / 2, padding 1 with -inf: padded positions never win, since every window holds a real one.
__device__ __forceinline__ void window_argmax(const bf16* xb, int h, int w, int c, int ho, int wo, int ch,
                                              float& best, int& bh, int& bw) {
  best = -INFINITY;
  bh = bw = -1;
  for (int i = 0; i < 3; ++i) {
    const int hh = 2 * ho - 1 + i;
    if (hh < 0 || hh >= h) continue;
    for (int j = 0; j < 3; ++j) {
      const int ww = 2 * wo - 1 + j;
      if (ww < 0 || ww >= w) continue;
      const float v = __bfloat162float(xb[((int64_t)hh * w + ww) * c + ch]);
      if (bh < 0 || v > best) { best = v; bh = hh; bw = ww; }
    }
  }
}

__global__ void __launch_bounds__(256)
maxpool_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int64_t n, int h, int w, int c, int ho, int wo) {
  const int64_t total = n * ho * wo * c;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % c);
    const int64_t pix = i / c;
    const int ow = (int)(pix % wo);
    const int64_t t = pix / wo;
    const int oh = (int)(t % ho);
    const int64_t img = t / ho;
    float best;
    int bh, bw;
    window_argmax(x + img * h * w * c, h, w, c, oh, ow, ch, best, bh, bw);
    y[i] = __float2bfloat16_rn(best);
  }
}

__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy, bf16* __restrict__ dx, int64_t n, int h,
                   int w, int c, int ho, int wo) {
  const int64_t total = n * h * w * c;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % c);
    const int64_t pix = i / c;
    const int wi = (int)(pix % w);
    const int64_t t = pix / w;
    const int hi = (int)(t % h);
    const int64_t img = t / h;
    const bf16* xb = x + img * h * w * c;
    // windows (oh, ow) with 2 oh - 1 <= hi <= 2 oh + 1, in row-major order
    float acc = 0.f;
    for (int oh = (hi) / 2; oh >= 0 && oh <= (hi + 1) / 2 && oh < ho; ++oh) {
      if (2 * oh - 1 > hi || 2 * oh + 1 < hi) continue;
      for (int ow = wi / 2; ow <= (wi + 1) / 2 && ow < wo; ++ow) {
        if (2 * ow - 1 > wi || 2 * ow + 1 < wi) continue;
        float best;
        int bh, bw;
        window_argmax(xb, h, w, c, oh, ow, ch, best, bh, bw);
        if (bh == hi && bw == wi) acc += __bfloat162float(dy[((img * ho + oh) * wo + ow) * c + ch]);
      }
    }
    dx[i] = __float2bfloat16_rn(acc);
  }
}

// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
stem_im2col_kernel(const float* __restrict__ img, bf16* __restrict__ cols, int64_t n, int h, int w, int ho, int wo) {
  const int64_t total = n * ho * wo * BV_STEM_K_PAD;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int col = (int)(i % BV_STEM_K_PAD);
    const int64_t pix = i / BV_STEM_K_PAD;
    float v = 0.f;
    if (col < BV_STEM_K) {
      const int ow = (int)(pix % wo);
      const int64_t t = pix / wo;
      const int oh = (int)(t % ho);
      const int64_t b = t / ho;
      const int kh = col / 21, kw = (col / 3) % 7, ch = col % 3;
      const int hh = 2 * oh - 3 + kh, ww = 2 * ow - 3 + kw;
      if (hh >= 0 && hh < h && ww >= 0 && ww < w) v = img[((b * h + hh) * w + ww) * 3 + ch];
    }
    cols[i] = __float2bfloat16_rn(v);
  }
}

unsigned grid_of(int64_t work) { return grid_for(work, 256, 16LL * num_sms()); }

}  // namespace
}  // namespace bv

extern "C" {

int bv_conv_fwd(const bv_conv_args* args, void* stream) {
  using namespace bv;
  const char* fn = "bv_conv_fwd";
  int rc = check_conv(fn, args);
  if (!rc) rc = need(fn, args->x, "x");
  if (!rc) rc = need(fn, args->kernel, "kernel");
  if (!rc) rc = need(fn, args->y, "y");
  if (!rc && args->resid) rc = need(fn, args->resid, "resid");
  if (rc) return rc;
  ConvGemm g = forward_gemm(*args);
  g.b = args->kernel; g.b_rows = (int64_t)args->k * args->k * args->cin; g.b_cols = args->cout; g.b_mn = 1;
  g.N = args->cout; g.out = args->y; g.resid = args->resid;
  return conv_gemm(g, static_cast<cudaStream_t>(stream));
}

int bv_conv_dgrad(const bv_conv_args* args, void* stream) {
  using namespace bv;
  const char* fn = "bv_conv_dgrad";
  int rc = check_conv(fn, args);
  if (!rc) rc = need(fn, args->dy, "dy");
  if (!rc) rc = need(fn, args->kernel, "kernel");
  if (!rc) rc = need(fn, args->dx, "dx");
  if (!rc && args->resid) rc = need(fn, args->resid, "resid");
  if (!rc && args->stride == 2) rc = need(fn, args->workspace, "workspace");
  if (rc) return rc;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bv_conv_args& a = *args;
  if (a.stride == 1) {
    ConvGemm g = dgrad_gemm(a, 0, 0);
    g.out = a.dx; g.resid = a.resid;
    return conv_gemm(g, s);
  }
  ScatterParams sp = {};
  sp.n = a.n; sp.h = a.h; sp.w = a.w; sp.c = a.cin;
  int64_t off = 0;
  for (int ph = 0; ph < 2; ++ph) {
    for (int pw = 0; pw < 2; ++pw) {
      ConvGemm g = dgrad_gemm(a, ph, pw);
      const int q = 2 * ph + pw;
      sp.gh[ph] = g.gh; sp.gw[pw] = g.gw;
      sp.off[q] = off;
      sp.has[q] = g.ntaps > 0 && g.gh > 0 && g.gw > 0;
      if (!sp.has[q]) continue;
      g.out = static_cast<bf16*>(a.workspace) + off;
      off += a.n * g.gh * g.gw * a.cin;
      rc = conv_gemm(g, s);
      if (rc) return rc;
    }
  }
  dgrad_scatter_kernel<<<grid_of(a.n * a.h * a.w * (a.cin / 8)), 256, 0, s>>>(
      static_cast<const bf16*>(a.workspace), static_cast<const bf16*>(a.resid), static_cast<bf16*>(a.dx), sp);
  return check_cuda(cudaGetLastError(), "dgrad_scatter_kernel launch");
}

int bv_conv_wgrad(const bv_conv_args* args, void* stream) {
  using namespace bv;
  const char* fn = "bv_conv_wgrad";
  int rc = check_conv(fn, args);
  if (!rc) rc = need(fn, args->x, "x");
  if (!rc) rc = need(fn, args->dy, "dy");
  if (!rc) rc = need(fn, args->dkernel, "dkernel");
  if (rc) return rc;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bv_conv_args& a = *args;
  if (!a.accumulate) {
    rc = check_cuda(cudaMemsetAsync(a.dkernel, 0, sizeof(float) * a.k * a.k * a.cin * a.cout, s), "bv_conv_wgrad memset");
    if (rc) return rc;
  }
  ConvGemm g = forward_gemm(a);
  g.wgrad = 1;
  g.b = a.dy; g.b_rows = a.n * (int64_t)g.gh * g.gw; g.b_cols = a.cout;
  g.N = a.cout; g.out = a.dkernel;
  return conv_gemm(g, s);
}

int bv_weight_std_fwd(const float* w, int64_t rows, int32_t cout, void* w_std, float* mean, float* rstd,
                      void* stream) {
  using namespace bv;
  if (!w || !w_std || !mean || !rstd) { set_error("bv_weight_std_fwd: null pointer"); return BV_ERR_INVALID; }
  if (rows < 1 || cout < 1) { set_error("bv_weight_std_fwd: need rows, cout >= 1"); return BV_ERR_INVALID; }
  weight_std_fwd_kernel<<<(cout + 31) / 32, dim3(32, WS_ROWS), 0, static_cast<cudaStream_t>(stream)>>>(
      w, rows, cout, static_cast<bf16*>(w_std), mean, rstd);
  return check_cuda(cudaGetLastError(), "weight_std_fwd_kernel launch");
}

int bv_weight_std_bwd(const float* w, const float* mean, const float* rstd, const float* g, int64_t rows,
                      int32_t cout, float* dw, void* stream) {
  using namespace bv;
  if (!w || !mean || !rstd || !g || !dw) { set_error("bv_weight_std_bwd: null pointer"); return BV_ERR_INVALID; }
  if (rows < 1 || cout < 1) { set_error("bv_weight_std_bwd: need rows, cout >= 1"); return BV_ERR_INVALID; }
  weight_std_bwd_kernel<<<(cout + 31) / 32, dim3(32, WS_ROWS), 0, static_cast<cudaStream_t>(stream)>>>(
      w, mean, rstd, g, rows, cout, dw);
  return check_cuda(cudaGetLastError(), "weight_std_bwd_kernel launch");
}

static int check_gn(const char* fn, int64_t n, int64_t hw, int32_t c) {
  if (n < 1 || n > 65535 || hw < 1 || c < bv::GN_GROUPS || c % bv::GN_GROUPS || c > 8192) {
    bv::set_error("%s: need 1 <= n <= 65535, hw >= 1 and c a multiple of 32 up to 8192", fn);
    return BV_ERR_INVALID;
  }
  return BV_OK;
}

int bv_groupnorm_fwd(const void* x, const float* scale, const float* bias, void* y, float* mean, float* rstd,
                     int64_t n, int64_t hw, int32_t c, int32_t relu, void* stream) {
  using namespace bv;
  if (!x || !scale || !bias || !y || !mean || !rstd) { set_error("bv_groupnorm_fwd: null pointer"); return BV_ERR_INVALID; }
  const int rc = check_gn("bv_groupnorm_fwd", n, hw, c);
  if (rc) return rc;
  groupnorm_fwd_kernel<<<dim3(GN_GROUPS, (unsigned)n), GN_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const bf16*>(x), scale, bias, static_cast<bf16*>(y), mean, rstd, hw, c, relu ? 1 : 0);
  return check_cuda(cudaGetLastError(), "groupnorm_fwd_kernel launch");
}

int bv_groupnorm_bwd(const void* x, const void* dy, const float* scale, const float* bias, const float* mean,
                     const float* rstd, const void* dx_add, void* dx, float* dscale, float* dbias, int64_t n,
                     int64_t hw, int32_t c, int32_t relu, void* stream) {
  using namespace bv;
  if (!x || !dy || !scale || !bias || !mean || !rstd || !dx || !dscale || !dbias) {
    set_error("bv_groupnorm_bwd: null pointer");
    return BV_ERR_INVALID;
  }
  const int rc = check_gn("bv_groupnorm_bwd", n, hw, c);
  if (rc) return rc;
  groupnorm_bwd_kernel<<<dim3(GN_GROUPS, (unsigned)n), GN_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const bf16*>(x), static_cast<const bf16*>(dy), scale, bias, mean, rstd,
      static_cast<const bf16*>(dx_add), static_cast<bf16*>(dx), dscale, dbias, hw, c, relu ? 1 : 0);
  return check_cuda(cudaGetLastError(), "groupnorm_bwd_kernel launch");
}

static int check_pool(const char* fn, int64_t n, int32_t h, int32_t w, int32_t c) {
  if (n < 1 || h < 1 || w < 1 || c < 1) {
    bv::set_error("%s: need n, h, w, c >= 1", fn);
    return BV_ERR_INVALID;
  }
  return BV_OK;
}

int bv_maxpool_fwd(const void* x, void* y, int64_t n, int32_t h, int32_t w, int32_t c, void* stream) {
  using namespace bv;
  if (!x || !y) { set_error("bv_maxpool_fwd: null pointer"); return BV_ERR_INVALID; }
  const int rc = check_pool("bv_maxpool_fwd", n, h, w, c);
  if (rc) return rc;
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  maxpool_fwd_kernel<<<grid_of(n * ho * wo * c), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const bf16*>(x), static_cast<bf16*>(y), n, h, w, c, ho, wo);
  return check_cuda(cudaGetLastError(), "maxpool_fwd_kernel launch");
}

int bv_maxpool_bwd(const void* x, const void* dy, void* dx, int64_t n, int32_t h, int32_t w, int32_t c,
                   void* stream) {
  using namespace bv;
  if (!x || !dy || !dx) { set_error("bv_maxpool_bwd: null pointer"); return BV_ERR_INVALID; }
  const int rc = check_pool("bv_maxpool_bwd", n, h, w, c);
  if (rc) return rc;
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  maxpool_bwd_kernel<<<grid_of(n * h * w * c), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const bf16*>(x), static_cast<const bf16*>(dy), static_cast<bf16*>(dx), n, h, w, c, ho, wo);
  return check_cuda(cudaGetLastError(), "maxpool_bwd_kernel launch");
}

int bv_stem_im2col(const float* image, void* cols, int64_t n, int32_t h, int32_t w, void* stream) {
  using namespace bv;
  if (!image || !cols) { set_error("bv_stem_im2col: null pointer"); return BV_ERR_INVALID; }
  if (n < 1 || h < 1 || w < 1) { set_error("bv_stem_im2col: need n, h, w >= 1"); return BV_ERR_INVALID; }
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  stem_im2col_kernel<<<grid_of(n * ho * wo * BV_STEM_K_PAD), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      image, static_cast<bf16*>(cols), n, h, w, ho, wo);
  return check_cuda(cudaGetLastError(), "stem_im2col_kernel launch");
}

}  // extern "C"
