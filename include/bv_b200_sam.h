/* bv_b200_sam.h -- C ABI of the sharpness-aware minimisation kernels in libbv_b200.so: the flat-buffer
 * vector algebra of GSAM / SAM (trainers/proj/gsam/gsam.py:28-122 of the reference), exported from the
 * same library as bv_b200.h and following its conventions:
 *  - every pointer is a DEVICE pointer; the caller owns all buffers (inputs, outputs, workspace);
 *  - functions only ENQUEUE work on `stream` (a cudaStream_t passed as void*); they never allocate
 *    device memory and never synchronise.  The scalars a kernel needs (norms, dot products) are read
 *    from device memory, so a GSAM step runs without a device-to-host copy;
 *  - return 0 on success, a negative BV_ERR_* code otherwise (bv_last_error_string() describes it);
 *  - fp32 buffers are 16-byte aligned, the bf16 output 8-byte aligned (BV_ERR_INVALID otherwise).  Any
 *    n >= 0: 16-byte vectors, and a scalar tail for n % 4 != 0.
 */
#ifndef BV_B200_SAM_H_
#define BV_B200_SAM_H_

#include <stdint.h>

#include "bv_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Floats of workspace bv_sam_dots needs (per-block partials of its two sums). */
#define BV_SAM_WS_FLOATS 2048

/* The perturbed weights of gsam.py:77-83, with the bf16 shadow the GEMMs read, in one pass:
 *   s = (rho * g[i]) / (sqrt(g_sumsq[0]) + eps)             adaptive == 0
 *   s = ((|w[i]| * rho) * g[i]) / (sqrt(g_sumsq[0]) + eps)  adaptive != 0
 *   w_out[i] = w[i] + s;  w_bf16[i] = round-to-nearest-even bf16 of w_out[i].
 * Each operation is one IEEE fp32 rounding in the order written.  w_out may equal w. */
int bv_sam_perturb(const float* w, const float* g, const float* g_sumsq, float rho, float eps, int32_t adaptive,
                   float* w_out, void* w_bf16, int64_t n, void* stream);

/* out[0] = sum_i a[i]*b[i], out[1] = sum_i b[i]*b[i] in one read of both buffers (one read when a == b).
 * Written, not accumulated.  Per-block partials in ws (BV_SAM_WS_FLOATS floats) and a fixed-order
 * finishing pass: the grid depends on n alone, so the two sums are identical bit for bit from run to
 * run and from device to device. */
int bv_sam_dots(const float* a, const float* b, float* out, float* ws, int64_t n, void* stream);

/* The GSAM gradient of gsam.py:92-119, in place over g_clean (g_c on entry, the combined g on exit):
 *   minimize_fp != 0:  nr = sqrt(norm_sq[0]) = ||g_r||, c = dot[0] / nr, g = g_r - alpha * (g_c - c * (g_r / nr))
 *   minimize_fp == 0:  nc = sqrt(norm_sq[0]) = ||g_c||, c = dot[0] / nc, g = g_c + alpha * (g_r - c * (g_c / nc))
 * with dot[0] = g_c . g_r.  No eps, like the reference: a zero norm gives NaN. */
int bv_gsam_combine(float* g_clean, const float* g_robust, const float* dot, const float* norm_sq, float alpha,
                    int32_t minimize_fp, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BV_B200_SAM_H_ */
