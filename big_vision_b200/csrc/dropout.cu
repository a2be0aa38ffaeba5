// Dropout (include/bv_dropout.h): y = dropout(x) and out = resid + dropout(y) on bf16 matrices.
// Thread i owns one Philox block, the 16 consecutive global elements [16 b, 16 b + 16) of which it writes
// those in this matrix.  With cols and every stride a multiple of 8 each half of the block is 8 elements of
// one row, loaded and stored as one 16-byte vector; otherwise each element is located on its own.  Both
// kernels read and write each element once, so they are bound by memory bandwidth.
#include "../../include/bv_dropout.h"

#include <cuda_bf16.h>
#include <math.h>

#include "common.cuh"
#include "host_utils.h"

namespace bv {
namespace {

constexpr int kThreads = 256;

struct DropParams {
  uint64_t seed, step, site;
  int64_t row0, rows, cols, first_blk, start, end;   // global element range [start, end)
  uint32_t T;                                         // drop when the 16-bit lane < T
  float keep;                                         // 1 - rate in fp32
};

__device__ __forceinline__ float drop_one(float v, const uint64_t (&w)[4], int lane, uint32_t T, float keep) {
  const uint32_t bits = static_cast<uint32_t>(w[lane >> 2] >> (16 * (lane & 3))) & 0xffffu;
  return bits < T ? 0.f : __fdiv_rn(v, keep);
}

// kAdd: out = bf16(resid + drop(y)); otherwise out = bf16(drop(y)) (resid unused).
template <bool kAdd, bool kVec>
__global__ void __launch_bounds__(kThreads)
dropout_kernel(const bf16* resid, int64_t ldr, const bf16* y, int64_t ldy, bf16* out, int64_t ldo, DropParams p) {
  const int64_t blk = p.first_blk + static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  const int64_t e0 = blk * 16;
  if (e0 >= p.end) return;
  uint64_t w[4] = {static_cast<uint64_t>(blk) + 1, p.step, p.site, 0};
  philox4x64_10(w, p.seed, 0);
  if (kVec) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t e = e0 + 8 * h;
      if (e < p.start || e >= p.end) continue;
      const int64_t g = e / p.cols, c = e - g * p.cols, r = g - p.row0;
      uint4 yv = *reinterpret_cast<const uint4*>(y + r * ldy + c);
      uint4 rv;
      if (kAdd) rv = *reinterpret_cast<const uint4*>(resid + r * ldr + c);
      const bf16* ye = reinterpret_cast<const bf16*>(&yv);
      const bf16* re = reinterpret_cast<const bf16*>(&rv);
      uint4 ov;
      bf16* oe = reinterpret_cast<bf16*>(&ov);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float v = drop_one(__bfloat162float(ye[j]), w, 8 * h + j, p.T, p.keep);
        if (kAdd) v = __fadd_rn(__bfloat162float(re[j]), v);
        oe[j] = __float2bfloat16_rn(v);
      }
      *reinterpret_cast<uint4*>(out + r * ldo + c) = ov;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int64_t e = e0 + j;
      if (e < p.start || e >= p.end) continue;
      const int64_t g = e / p.cols, c = e - g * p.cols, r = g - p.row0;
      float v = drop_one(__bfloat162float(y[r * ldy + c]), w, j, p.T, p.keep);
      if (kAdd) v = __fadd_rn(__bfloat162float(resid[r * ldr + c]), v);
      out[r * ldo + c] = __float2bfloat16_rn(v);
    }
  }
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

// Checks the arguments shared by both entry points and launches; resid == nullptr for bv_dropout.
int launch(const char* fn, const void* resid, int64_t ldr, const void* y, int64_t ldy, void* out, int64_t ldo,
           int64_t rows, int64_t cols, const bv_dropout_key* key, void* stream) {
  const bool add = resid != nullptr;
  if (!key || !y || !out) {
    set_error("%s: null key or matrix", fn);
    return BV_ERR_INVALID;
  }
  if (!(key->rate >= 0.f && key->rate < 1.f)) {
    set_error("%s: rate %g outside [0, 1)", fn, static_cast<double>(key->rate));
    return BV_ERR_INVALID;
  }
  if (key->site == 0) {
    set_error("%s: site 0 is Jet's noise stream; dropout sites start at 1", fn);
    return BV_ERR_INVALID;
  }
  if (rows < 0 || cols < 1 || key->row0 < 0 || ldy < cols || ldo < cols || (add && ldr < cols)) {
    set_error("%s: need rows >= 0, cols >= 1, row0 >= 0 and every stride >= cols", fn);
    return BV_ERR_INVALID;
  }
  if (!aligned(y, 2) || !aligned(out, 2) || (add && !aligned(resid, 2))) {
    set_error("%s: bf16 matrices must be 2-byte aligned", fn);
    return BV_ERR_INVALID;
  }
  if ((out == y && ldo != ldy) || (add && out == resid && ldo != ldr)) {
    set_error("%s: an output aliasing an input must have its stride", fn);
    return BV_ERR_INVALID;
  }
  if (rows == 0) return BV_OK;
  DropParams p;
  p.seed = key->seed;
  p.step = key->step;
  p.site = key->site;
  p.row0 = key->row0;
  p.rows = rows;
  p.cols = cols;
  p.start = key->row0 * cols;
  p.end = (key->row0 + rows) * cols;
  p.first_blk = p.start / 16;
  p.T = static_cast<uint32_t>(nearbyint(static_cast<double>(key->rate) * 65536.0));
  p.keep = 1.f - key->rate;
  const int64_t nblk = (p.end - 1) / 16 - p.first_blk + 1;
  const bool vec = cols % 8 == 0 && ldy % 8 == 0 && ldo % 8 == 0 && aligned(y, 16) && aligned(out, 16) &&
                   (!add || (ldr % 8 == 0 && aligned(resid, 16)));
  const dim3 grid(static_cast<unsigned>((nblk + kThreads - 1) / kThreads));
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bf16* r = static_cast<const bf16*>(resid);
  const bf16* yb = static_cast<const bf16*>(y);
  bf16* o = static_cast<bf16*>(out);
  if (add && vec) dropout_kernel<true, true><<<grid, kThreads, 0, s>>>(r, ldr, yb, ldy, o, ldo, p);
  else if (add) dropout_kernel<true, false><<<grid, kThreads, 0, s>>>(r, ldr, yb, ldy, o, ldo, p);
  else if (vec) dropout_kernel<false, true><<<grid, kThreads, 0, s>>>(r, ldr, yb, ldy, o, ldo, p);
  else dropout_kernel<false, false><<<grid, kThreads, 0, s>>>(r, ldr, yb, ldy, o, ldo, p);
  return check_cuda(cudaGetLastError(), fn);
}

}  // namespace
}  // namespace bv

extern "C" {

int bv_dropout(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int64_t cols,
               const bv_dropout_key* key, void* stream) {
  return bv::launch("bv_dropout", nullptr, 0, x, ldx, y, ldy, rows, cols, key, stream);
}

int bv_dropout_add(const void* resid, int64_t ldr, const void* y, int64_t ldy, void* out, int64_t ldo,
                   int64_t rows, int64_t cols, const bv_dropout_key* key, void* stream) {
  if (!resid) {
    bv::set_error("bv_dropout_add: null resid");
    return BV_ERR_INVALID;
  }
  return bv::launch("bv_dropout_add", resid, ldr, y, ldy, out, ldo, rows, cols, key, stream);
}

}  // extern "C"
