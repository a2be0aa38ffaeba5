/* bv_b200_flexi.h -- C ABI of the FlexiViT resampling kernels in libbv_b200.so (models/proj/flexi/vit.py of
 * the reference).  A FlexiViT step draws a sequence length, resizes the patch-embedding kernel and the
 * position embedding from their stored base shapes to it, and runs the encoder at that token count.  Both
 * resizes are linear maps fixed by the two shapes: a small fp32 matrix M [R, K] (R outputs, K inputs) applied
 * to every column of a [K, J] matrix.  The forward writes the bf16 GEMM operand; the backward applies M^T and
 * accumulates into the fp32 gradient of the stored parameter.
 * Exported from the same library as bv_b200.h and following its conventions:
 *  - every pointer is a DEVICE pointer; the caller owns all buffers;
 *  - functions only ENQUEUE work on `stream` (a cudaStream_t passed as void*); they never allocate
 *    device memory and never synchronise;
 *  - return 0 on success, a negative BV_ERR_* code otherwise (bv_last_error_string() describes it);
 *    invalid arguments are refused before anything is launched;
 *  - matrices are row-major and dense: M [R, K], x / dy [K, J] / [R, J] with row stride J.  J % 4 == 0;
 *    x, dy and dx are 16-byte aligned, y_bf16 8-byte aligned (BV_ERR_INVALID otherwise).  R, K >= 1.
 *  - no atomics: every output element is summed by one thread in ascending index order, so results are
 *    identical bit for bit from run to run.
 */
#ifndef BV_B200_FLEXI_H_
#define BV_B200_FLEXI_H_

#include <stdint.h>

#include "bv_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* y[r, j] = bf16( sum_{k ascending} M[r, k] * x[k, j] ),  r < R, j < J.  fp32 products and sums (fused
 * multiply-adds), one round-to-nearest-even to bf16 at the end.  y has R rows of J elements. */
int bv_resample_fwd(const float* M, const float* x, void* y_bf16, int32_t R, int32_t K, int64_t J, void* stream);

/* dx[k, j] += sum_{r ascending} M[r, k] * dy[r, j],  k < K, j < J.  fp32 fused multiply-adds; the sum is
 * formed first and then added to dx. */
int bv_resample_bwd(const float* M, const float* dy, float* dx, int32_t R, int32_t K, int64_t J, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BV_B200_FLEXI_H_ */
