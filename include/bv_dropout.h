/* bv_dropout.h -- C ABI of the dropout kernels in libbv_b200.so (flax nn.Dropout in models/vit.py and
 * models/proj/image_text/text_transformer.py of the reference), and the attention-probability dropout flag of
 * the attention entry points of bv_b200.h (BERT, models/proj/flaxformer/bert.py).
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

/* ---------------------------------------------------------------------------------
 * Attention-probability dropout (BERT's attention_probs_dropout_prob; flaxformer's BertEncoder with
 * enable_dropout, models/proj/flaxformer/bert.py:55): the key-masked attention of bv_b200.h drops each
 * softmax probability P[b, h, q, k] with probability `rate` and scales the kept ones by 1 / (1 - rate).
 * Built for key-masked attention at head dim 64 only: pass head_dim = 64 | BV_ATTN_KEY_MASK | BV_ATTN_DROPOUT to
 * bv_attention_fwd_hd / bv_attention_bwd_hd, with args pointing to a bv_attn_dropout_args /
 * bv_attn_dropout_bwd_args.  The backward must be given the forward's key.  The flag without
 * BV_ATTN_KEY_MASK, at any other head dim, with a NULL args pointer, site 0, row0 < 0 or a rate outside [0, 1)
 * is refused with BV_ERR_INVALID before any launch.
 *
 * The mask is never stored: the forward, dQ and dK/dV kernels each regenerate it.  Its stream is the
 * generator of bv_dropout, Philox4x64-10 under key (seed, 0).  Probability (b, h, q, k) belongs to the global
 * row r = row0 + (b * H + h) * Nq + q (a data-parallel rank whose batch starts at global sample sample0
 * passes row0 = sample0 * H * Nq) and uses the 16-bit lane k % 16 of the block at counter
 * (k / 16 + 1, step, site, r + 1), i.e. numpy's
 * np.random.Philox(key=seed, counter=[0, step, site, r + 1]).random_raw(4 * ceil(Nk / 16)), lanes as above.  It
 * is dropped when that lane is below T = round(rate * 65536), as in bv_dropout.  Counter word 3 is >= 1
 * here and 0 in every bv_dropout counter, so the two streams never meet, even at the same site.
 *
 * Maths, with Z the keep mask and kappa = 1 - rate in fp32: lse and the row sums l are those of the
 * undropped softmax, and O = ((P o Z) V) / (l * kappa).  The backward's delta = rowsum(dO o O) is unchanged;
 * dS = P o (Z o dP / kappa - delta) with dP = dO V^T, and dV = (Z o P / kappa)^T dO.  Masked keys and keys
 * past Nk keep P = 0 whatever their mask bits.  At rate 0 the results are the bits of the call without the
 * flag.
 * --------------------------------------------------------------------------------- */
#define BV_ATTN_DROPOUT 131072   /* head_dim flag: args carries a dropout key (with BV_ATTN_KEY_MASK) */
typedef struct bv_attn_dropout_args {
  bv_attn_masked_args masked;
  bv_dropout_key drop;
} bv_attn_dropout_args;
typedef struct bv_attn_dropout_bwd_args {
  bv_attn_masked_bwd_args masked;   /* masked.attn.fwd and the mask: the forward call's */
  bv_dropout_key drop;              /* the forward call's key */
} bv_attn_dropout_bwd_args;

#ifdef __cplusplus
}
#endif
#endif /* BV_DROPOUT_H_ */
