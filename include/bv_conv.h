/* bv_conv.h -- C ABI of the convolution kernels in libbv_b200.so: the BiT ResNet-v2 of the reference's
 * models/bit_paper.py (weight-standardised convolutions, GroupNorm + ReLU, the root block's max pool).
 *
 * Exported from the same library as bv_b200.h and following its conventions:
 *  - every pointer is a DEVICE pointer; the caller owns all buffers;
 *  - functions only ENQUEUE work on `stream` (a cudaStream_t passed as void*); they never allocate
 *    device memory and never synchronise;
 *  - return 0 on success, a negative BV_ERR_* code otherwise (bv_last_error_string() describes it);
 *    invalid arguments are refused with BV_ERR_INVALID before anything is launched.
 *
 * Layouts: activations are NHWC bf16, kernels HWIO [k, k, cin, cout] (the reference's layout); the fp32
 * parameters stay with the caller and the convolutions read a bf16 copy of the standardised kernel.
 */
#ifndef BV_CONV_H_
#define BV_CONV_H_

#include <stdint.h>

#include "bv_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------
 * Convolution (flax nn.Conv with explicit symmetric padding k / 2, no bias): k x k filters, k in {1, 3, 7},
 * stride 1 or 2, cin and cout multiples of 64, 1 <= h, w <= 32767.  The output is ho x wo with
 * ho = (h + 2 (k / 2) - k) / stride + 1 (likewise wo).  Every call is an implicit GEMM on the tensor cores
 * (bf16 operands, fp32 accumulation) that reads the activation through TMA in im2col mode; the zero padding
 * is TMA's out-of-bounds fill.
 *
 *   bv_conv_fwd:   y = conv(x, kernel) (+ resid)                            bf16, rounded once (twice with resid:
 *                  the sum is rounded to bf16, then resid is added and the total rounded)
 *   bv_conv_dgrad: dx = the input gradient of conv for output gradient dy (+ resid), rounded likewise.  At
 *                  stride 2 it runs as up to four sub-convolutions, one per (row, column) parity of dx,
 *                  whose outputs go to `workspace` (bf16, n * h * w * cin elements) before one pass moves
 *                  them into dx; at stride 1 workspace is unused.
 *   bv_conv_wgrad: dkernel (+)= the kernel gradient, fp32 HWIO, summed over pixels in splits whose partial
 *                  sums are added with fp32 atomics (so the bits may vary from run to run); accumulate = 0
 *                  overwrites dkernel.
 *
 * Refused with BV_ERR_INVALID before any launch: a NULL args pointer or NULL tensor that the call reads or
 * writes, a tensor base that is not 16-byte aligned, an unsupported k, stride, channel count or size, and a
 * NULL workspace for the stride-2 data gradient.
 * --------------------------------------------------------------------------------- */
typedef struct bv_conv_args {
  const void* x;       /* bf16 [n, h, w, cin]: the input (forward, kernel gradient) */
  const void* kernel;  /* bf16 [k, k, cin, cout]: the standardised kernel (forward, data gradient) */
  const void* dy;      /* bf16 [n, ho, wo, cout]: the output gradient (data and kernel gradient) */
  void* y;             /* bf16 [n, ho, wo, cout]: forward output */
  void* dx;            /* bf16 [n, h, w, cin]: data-gradient output */
  float* dkernel;      /* fp32 [k, k, cin, cout]: kernel-gradient output */
  const void* resid;   /* NULL, or bf16 in the layout of y (forward) or dx (data gradient), added to it */
  void* workspace;     /* bf16, n * h * w * cin elements: the stride-2 data gradient */
  int64_t n;
  int32_t h, w, cin, cout, k, stride;
  int32_t accumulate;  /* kernel gradient: 1 adds into dkernel, 0 overwrites it */
} bv_conv_args;
int bv_conv_fwd(const bv_conv_args* args, void* stream);
int bv_conv_dgrad(const bv_conv_args* args, void* stream);
int bv_conv_wgrad(const bv_conv_args* args, void* stream);

/* ---------------------------------------------------------------------------------
 * Weight standardisation (bit_paper.StdConv, standardize(kernel, axis=[0, 1, 2], eps=1e-10)) of a kernel
 * viewed as the fp32 matrix [rows = k * k * cin, cout]: per output channel (column) the mean and the variance
 * (the mean of squared deviations, two passes), rstd = 1 / sqrt(var + 1e-10).
 *   fwd: w_std = bf16((w - mean) * rstd); mean and rstd (fp32 [cout]) are saved for the backward.
 *   bwd: dw = rstd * (g - mean(g) - w_hat * mean(g * w_hat)) with w_hat = (w - mean) * rstd and g the fp32
 *        gradient of the standardised kernel; dw is overwritten.
 * rows >= 1, cout >= 1, non-NULL pointers; fixed-order sums, so the bits repeat.
 * --------------------------------------------------------------------------------- */
int bv_weight_std_fwd(const float* w, int64_t rows, int32_t cout, void* w_std, float* mean, float* rstd,
                      void* stream);
int bv_weight_std_bwd(const float* w, const float* mean, const float* rstd, const float* g, int64_t rows,
                      int32_t cout, float* dw, void* stream);

/* ---------------------------------------------------------------------------------
 * GroupNorm with 32 groups and eps 1e-5 (bit_paper.GroupNorm), optionally followed by ReLU, on bf16
 * [n, hw, c] (NHWC with the pixels flattened), c a multiple of 32 and at most 8192.  Statistics per (image,
 * group) over hw * c / 32 values in fp32, two passes as the reference (mean, then the mean of squared
 * deviations); mean and rstd are saved as fp32 [n, 32].
 *   fwd: y = bf16(relu?((x - mean) * rstd * scale + bias)).
 *   bwd: dz = dy, times (z > 0) with relu, where z is the pre-ReLU value recomputed in fp32;
 *        dx = bf16(rstd * (dz*scale - mean(dz*scale) - x_hat * mean(dz*scale * x_hat)) (+ dx_add));
 *        dscale += sum(dz * x_hat), dbias += sum(dz) over images and pixels (fp32 atomics, one per block
 *        and channel, as LayerNorm's parameter gradients).
 * --------------------------------------------------------------------------------- */
int bv_groupnorm_fwd(const void* x, const float* scale, const float* bias, void* y, float* mean, float* rstd,
                     int64_t n, int64_t hw, int32_t c, int32_t relu, void* stream);
int bv_groupnorm_bwd(const void* x, const void* dy, const float* scale, const float* bias, const float* mean,
                     const float* rstd, const void* dx_add, void* dx, float* dscale, float* dbias, int64_t n,
                     int64_t hw, int32_t c, int32_t relu, void* stream);

/* ---------------------------------------------------------------------------------
 * Max pool 3 x 3, stride 2, padding (1, 1) with -inf (flax nn.max_pool in bit_paper.RootBlock) on bf16
 * NHWC [n, h, w, c]: ho = (h - 1) / 2 + 1, likewise wo.  The backward routes each output gradient to the
 * first maximal element of its window in row-major window order, written as a gather over the (at most 4)
 * windows of each input element, so its bits repeat; dx is overwritten.
 * --------------------------------------------------------------------------------- */
int bv_maxpool_fwd(const void* x, void* y, int64_t n, int32_t h, int32_t w, int32_t c, void* stream);
int bv_maxpool_bwd(const void* x, const void* dy, void* dx, int64_t n, int32_t h, int32_t w, int32_t c,
                   void* stream);

/* ---------------------------------------------------------------------------------
 * The root convolution's operand: the 7 x 7 / 2 patches (padding 3) of an fp32 NHWC image with 3 channels,
 * as bf16 [n * ho * wo, BV_STEM_K_PAD] with column (kh * 7 + kw) * 3 + channel (the row order of the HWIO
 * kernel [7, 7, 3, cout]) and zeros in columns 147 .. 151.  ho = (h - 1) / 2 + 1.  The root convolution is then
 * bv_gemm with K = 147.
 * --------------------------------------------------------------------------------- */
#define BV_STEM_K 147
#define BV_STEM_K_PAD 152
int bv_stem_im2col(const float* image, void* cols, int64_t n, int32_t h, int32_t w, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BV_CONV_H_ */
