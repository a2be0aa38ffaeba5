// The convolution modes of the persistent wgmma GEMM (gemm.cu), called by the convolution entry points
// (conv.cu).  One call is one implicit GEMM whose A operand is read from an NHWC bf16 tensor by TMA in
// im2col mode.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bv {

constexpr int kConvMaxTaps = 49;   // a 7 x 7 filter

struct ConvTap {
  int ow, oh;   // shift of the base position, >= 0
  int brow;     // forward / data gradient: first row of the tap's kernel slice in the 2-D view of b
};

struct ConvGemm {
  // the NHWC input A is read from: [n, h, w, c], c a multiple of 64
  const void* x;
  int64_t n;
  int h, w, c;
  // output grid (gh, gw) whose pixel (img, y, x) starts from input base (lw + stride x, lh + stride y); the base
  // positions span [lw, lw + stride (gw - 1)] x [lh, lh + stride (gh - 1)]
  int gh, gw, lw, lh, stride;
  int ntaps;
  ConvTap taps[kConvMaxTaps];
  // wgrad = 0: out[img, y, x, :] (bf16, N columns) = sum over taps and channels of the shifted input times the
  //   tap's slice of b, a row-major bf16 matrix read MN-major (b_mn = 1, the slice is c rows from
  //   brow) or K-major (b_mn = 0, the slice is N rows from brow whose first c columns are read); plus resid
  //   (bf16, out's layout) when not NULL.
  // wgrad = 1: out (fp32 [ntaps * c, N], row tap * c + channel) += the shifted input^T times b = dy
  //   (bf16 [n * gh * gw, N]), split over pixels; the caller zeroes out first to overwrite.
  int wgrad;
  const void* b;
  int64_t b_rows, b_cols;   // b is row-major [b_rows, b_cols] (wgrad: [n * gh * gw, N])
  int b_mn;
  int N;
  void* out;
  const void* resid;
};

int conv_gemm(const ConvGemm& g, cudaStream_t stream);

}  // namespace bv
