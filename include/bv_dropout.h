/* bv_dropout.h -- C ABI of the dropout kernels in libbv_b200.so (flax nn.Dropout in models/vit.py and
 * models/proj/image_text/text_transformer.py of the reference).
 *
 * Exported from the same library as bv_b200.h and following its conventions:
 *  - every pointer is a DEVICE pointer; the caller owns all buffers;
 *  - functions only ENQUEUE work on `stream` (a cudaStream_t passed as void*); they never allocate
 *    device memory and never synchronise;
 *  - return 0 on success, a negative BV_ERR_* code otherwise (bv_last_error_string() describes it);
 *    invalid arguments are refused with BV_ERR_INVALID before anything is launched.
 */
#ifndef BV_DROPOUT_H_
#define BV_DROPOUT_H_

#include <stdint.h>

#include "bv_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------
 * Dropout (flax nn.Dropout at models/vit.py:76,100,109,228): a kept element becomes x / (1 - rate), a
 * dropped one 0.  The mask is a pure function of the key and the element's global index, so a backward or a
 * recompute regenerates it instead of storing it.
 *
 * The mask stream: Philox4x64-10 under key (seed, 0).  Block b = 0, 1, ... is the output at counter
 * (b + 1, step, site, 0), four 64-bit words w0..w3 (numpy:
 * np.random.Philox(key=seed, counter=[0, step, site, 0]).random_raw(4 * nblocks)).  Element e uses the 16-bit
 * lane e % 16 of block e / 16, i.e. bits [16 (e % 4), 16 (e % 4) + 16) of word (e % 16) / 4, and is dropped
 * when that lane is below T = round(rate * 65536) (rate as the float below, the product in double, rounded
 * to nearest even).  The realized drop probability T / 65536 is within 2^-17 of rate.
 * The element of row r, column c of a [rows, cols] matrix is e = (row0 + r) * cols + c: a data-parallel rank
 * whose rows start at global row row0 draws the masks of those rows of the global batch.
 * site = 0 is Jet's dequantization noise (bv_b200_jet.h) and is refused here, so the two never share a
 * counter.
 *
 * Rounding: a kept value is the fp32 quotient fp32(x) / (1 - rate) (the divisor 1 - rate computed in fp32),
 * rounded once to bf16; bv_dropout_add rounds fp32(resid) + that fp32 quotient once to bf16.
 *
 * Matrices are bf16 with row strides (elements) >= cols and 2-byte aligned bases; 16-byte vectors are used
 * when cols and every stride are multiples of 8 and every base is 16-byte aligned.  The output may alias an
 * input of the same stride.  Refused with BV_ERR_INVALID before any launch: a NULL key or matrix, rate
 * outside [0, 1), site 0, rows < 0, cols < 1, row0 < 0, a stride < cols, a misaligned base, or an alias
 * with another stride.
 * --------------------------------------------------------------------------------- */
typedef struct bv_dropout_key {
  uint64_t seed;   /* Philox key word 0 (word 1 is 0) */
  uint64_t step;   /* counter word 1: the optimizer step */
  uint64_t site;   /* counter word 2, >= 1: which dropout of the model */
  int64_t row0;    /* global row of the matrix's row 0 */
  float rate;      /* drop probability, in [0, 1) */
} bv_dropout_key;
/* y = dropout(x): x, y bf16 [rows, cols] with row strides ldx, ldy. */
int bv_dropout(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int64_t cols,
               const bv_dropout_key* key, void* stream);
/* out = resid + dropout(y): the residual add after a dropped branch (models/vit.py:100,109). */
int bv_dropout_add(const void* resid, int64_t ldr, const void* y, int64_t ldy, void* out, int64_t ldo,
                   int64_t rows, int64_t cols, const bv_dropout_key* key, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BV_DROPOUT_H_ */
