/* bv_b200_jet.h -- C ABI of the Jet normalizing-flow kernels in libbv_b200.so (models/proj/jet/jet.py and
 * trainers/proj/jet/train.py of the reference).  Jet maps an image to a Gaussian through `depth` affine
 * couplings.  Each coupling permutes the image's D values (a fixed 0/1 permutation matrix, over the values of
 * a token or over the tokens), splits them into halves x1 and x2, runs a ViT on x1 and maps x2 affinely with
 * the ViT's output.  The ViT is the library's GEMM / attention / LayerNorm path; these kernels are the flow
 * around it: dequantization noise and the patch layout, the permuted split and merge, the affine map with its
 * log-determinant and its gradient, and the bits-per-dim loss.
 *
 * Exported from the same library as bv_b200.h and following its conventions:
 *  - every pointer is a DEVICE pointer; the caller owns all buffers;
 *  - functions only ENQUEUE work on `stream` (a cudaStream_t passed as void*); they never allocate
 *    device memory and never synchronise;
 *  - return 0 on success, a negative BV_ERR_* code otherwise (bv_last_error_string() describes it);
 *    invalid arguments are refused with BV_ERR_INVALID before anything is launched.
 *
 * The flow state is fp32 [n, D] per batch, D = T * 2c: T tokens of 2c = ps*ps*C values each, in the order
 * `b (h hp) (w wp) c -> b (h w) (hp wp c)`.  A coupling is described by its index table idx[0:D] (int32,
 * shared by all images): x1[j] = x[idx[j]] and x2[j] = x[idx[D/2 + j]] for j < D/2, and x1 / x2 are read
 * as [T, c] row-major matrices.  idx must be a permutation of 0..D-1 (not checked on the device).  The
 * DNN's output `br` is fp32 [n * T, 2c]: columns 0..c-1 the bias, c..2c-1 the raw scale of each x2 value.
 * s = sigmoid(raw) * scale_factor.  Every reduction is summed in a fixed order without atomics, so each
 * output is identical bit for bit from run to run.
 */
#ifndef BV_B200_JET_H_
#define BV_B200_JET_H_

#include <stdint.h>

#include "bv_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* z[b, t, k] = image[b, y, x, ch] + fp32(u * noise_scale) with t = (y / ps) * (W / ps) + x / ps and
 * k = ((y % ps) * ps + x % ps) * C + ch, image fp32 NHWC [n, H, W, C].  The product and the sum are two
 * separately rounded fp32 operations; noise_scale = 0 adds nothing (a plain patchify).
 * u is element (offset + e) of the global stream, e the element's NHWC index in this batch:
 * np.random.Generator(np.random.Philox(key=seed, counter=[0, counter, 0, 0])).random(N, dtype=np.float32),
 * i.e. Philox4x64-10 under key (seed, 0) at counters (1 + i, counter, 0, 0) for block i = 0, 1, ..., each
 * 64-bit output word giving its low then its high 32 bits u32, and u = (u32 >> 8) * 2^-24.  A data-parallel
 * rank r passes offset = r * n * H * W * C, so the noise of a global batch does not depend on how many
 * ranks share it.  H and W multiples of ps; offset >= 0. */
int bv_jet_dequantize_patchify(const float* image, float* z, int64_t n, int32_t H, int32_t W, int32_t C,
                               int32_t ps, uint64_t seed, uint64_t counter, int64_t offset, float noise_scale,
                               void* stream);

/* The inverse layout change: image[b, y, x, ch] = z[b, t, k] (indices as above). */
int bv_jet_unpatchify(const float* z, float* image, int64_t n, int32_t H, int32_t W, int32_t C, int32_t ps,
                      void* stream);

/* x1_bf16[b * D/2 + j] = bf16(x[b * D + idx[j]]) for j < D/2 (round to nearest even): the [n * T, c] operand
 * of the DNN's first GEMM. */
int bv_jet_split(const float* x, const int32_t* idx, void* x1_bf16, int64_t n, int32_t T, int32_t c,
                 void* stream);

/* One coupling, forward (inverse = 0) or inverse (inverse = 1).  For j < D/2, with x2 = x[idx[D/2 + j]]
 * and (bias, raw) the entries of br for x2's row j / c and column j % c:
 *   forward: y[idx[D/2 + j]] = (x2 + bias) * s;   inverse: y[idx[D/2 + j]] = x2 / s - bias;
 * y[idx[j]] = x[idx[j]].  logdet[b] += (inverse ? -1 : 1) * sum_j (log_sigmoid(raw) + log(scale_factor)),
 * with log_sigmoid in its stable form (finite for any finite raw).  y may alias x. */
int bv_jet_coupling_fwd(const float* x, const int32_t* idx, const float* br, float* y, float* logdet, int64_t n,
                        int32_t T, int32_t c, float scale_factor, int32_t inverse, void* stream);

/* Backward of the forward coupling.  dy is the gradient of its output, x its saved input and dlogdet the
 * gradient of the loss with respect to every image's logdet.  For j < D/2, with dy2 = dy[idx[D/2 + j]] and
 * sigma = sigmoid(raw):
 *   dx[idx[D/2 + j]] = dy2 * s;
 *   dbr_bf16[row, col] = bf16(dy2 * s)                                        (the bias gradient)
 *   dbr_bf16[row, c + col] = bf16(dy2 * (x2 + bias) * s * (1 - sigma) + dlogdet * (1 - sigma)).
 * dx at positions idx[0:D/2] is not written (bv_jet_merge_grad writes it).  dx may alias dy. */
int bv_jet_coupling_bwd(const float* dy, const float* x, const int32_t* idx, const float* br, float dlogdet,
                        float* dx, void* dbr_bf16, int64_t n, int32_t T, int32_t c, float scale_factor,
                        void* stream);

/* dx[b * D + idx[j]] = dy[b * D + idx[j]] + dx1[b * D/2 + j] for j < D/2: the gradient of x1, which passes
 * through the coupling and feeds the DNN (dx1 fp32 [n * T, c]).  dx may alias dy. */
int bv_jet_merge_grad(const float* dy, const float* dx1, const int32_t* idx, float* dx, int64_t n, int32_t T,
                      int32_t c, void* stream);

/* Bits per dimension of z fp32 [n, D] under a standard normal, for pixels quantized to 1/127.5:
 *   nll[b] = sum_k (z[b, k]^2 / 2 + log(2 pi) / 2 + log(127.5)),   bits[b] = nll[b] - logdet[b];
 * rows fp32 [3, n] = (bits, nll, logdet) / (D ln 2) per example and means fp32 [3] their batch means.
 * dz (may be NULL) = grad_scale * z: with grad_scale = 1 / (n D ln 2) the gradient of the mean of bits / (D ln 2)
 * with respect to z (the gradient with respect to logdet is the constant -grad_scale). */
int bv_jet_bits(const float* z, const float* logdet, float* rows, float* means, float* dz, float grad_scale,
                int64_t n, int64_t D, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BV_B200_JET_H_ */
