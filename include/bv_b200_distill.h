/* bv_b200_distill.h -- C ABI of the distillation kernels in libbv_b200.so: the distance between a
 * student's and a teacher's outputs (evaluators/proj/distill/distance.py:35-67 of the reference) and the
 * fused loss / gradient / measurements of one distillation step (trainers/proj/distill/distill.py:217-248).
 * Exported from the same library as bv_b200.h and following its conventions:
 *  - every pointer is a DEVICE pointer; the caller owns all buffers (inputs, outputs, workspace);
 *  - functions only ENQUEUE work on `stream` (a cudaStream_t passed as void*); they never allocate
 *    device memory and never synchronise;
 *  - return 0 on success, a negative BV_ERR_* code otherwise (bv_last_error_string() describes it);
 *    invalid arguments are refused before anything is launched;
 *  - matrices are fp32, row-major, each with its own row stride in elements (>= the column count), so
 *    the [n, C] view of a head stored [n, Cp] is passed as it is.  Rows are read with 16-byte loads when
 *    every base pointer is 16-byte aligned and every stride a multiple of 4, with 4-byte loads otherwise.
 *    Logits are finite.
 */
#ifndef BV_B200_DISTILL_H_
#define BV_B200_DISTILL_H_

#include <stdint.h>

#include "bv_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* `kind` of dist() (distance.py:35-67). */
#define BV_DIST_EUCLIDEAN 0            /* sqrt(sum (s - u)^2 + epsilon) */
#define BV_DIST_L2 1                   /* sum (s - u)^2 */
#define BV_DIST_HARD 2                 /* softmax_xent(s, smoothed one-hot of argmax u, kl=True) */
#define BV_DIST_KL 3                   /* t^2 * softmax_xent(s / t, softmax(u / t), kl=True) */
#define BV_DIST_LOGSOFTMAX_EUCLIDEAN 4 /* sqrt(sum (log_softmax s - log_softmax u)^2 + epsilon) */
#define BV_DIST_AGREE 5                /* is argmax u among the k largest of s (int32 0 / 1) */

/* Scalars bv_distill_loss produces, and the rows of its [BV_DISTILL_OUTPUTS, n] workspace. */
#define BV_DISTILL_DISTANCE 0          /* the distance (distill_loss_<teacher>) */
#define BV_DISTILL_ENTROPY_STUDENT 1   /* -sum softmax(s) log_softmax(s), at temperature 1 */
#define BV_DISTILL_ENTROPY_TEACHER 2
#define BV_DISTILL_TASK_STUDENT 3      /* softmax_xent(s, labels); 0 without labels */
#define BV_DISTILL_TASK_TEACHER 4
#define BV_DISTILL_OUTPUTS 5

/* One teacher's term of the distillation loss, its gradient and the step's measurements.
 *   kind BV_DIST_KL:   d_i = t^2 * [ -sum_c p_c log_softmax(s_i / t)_c + sum_c p_c log(max(p_c, 1e-8)) ],
 *                      p = softmax(u_i / t)                       (utils.py:276-281 with kl=True)
 *   kind BV_DIST_HARD: the same cross-entropy at temperature 1 with p = (1 - ls) onehot(a) +
 *                      ls / (C - 1) (1 - onehot(a)), a the FIRST maximal index of u_i (jnp.argmax); `t` unused
 *   any other kind:    BV_ERR_UNSUPPORTED.
 * rows_ws[k * n + i] (k = BV_DISTILL_*) holds row i's value of output k, so rows_ws[0 .. n) are the per-row
 * distances; out[k] = (1/n) sum_i rows_ws[k * n + i], WRITTEN, summed in a fixed order: identical bit for
 * bit from run to run.  Without labels (NULL) the two task losses are 0.
 * dlogits (NULL: no gradient) [n, ld_dlogits] = d out[0] / d student: (t / n) (softmax(s / t) - p) for KL,
 * (1 / n) (softmax(s) - p) for HARD.  accumulate == 0: written, with zeros in columns C .. ld_dlogits - 1;
 * accumulate != 0: added to what is there (a second teacher), the padding columns left as they are. */
int bv_distill_loss(const float* student, int64_t ld_student, const float* teacher, int64_t ld_teacher,
                    const float* labels, int64_t ld_labels, int32_t kind, float t, float ls, int32_t accumulate,
                    float* dlogits, int64_t ld_dlogits, float* out, float* rows_ws, int64_t n, int32_t C,
                    void* stream);

/* out[i] = dist(student_i, teacher_i, kind) for every kind of dist(): float32 [n], int32 [n] for
 * BV_DIST_AGREE.  `epsilon` is used by the two euclidean kinds, `t` by KL, `ls` by HARD, `k` by AGREE.
 * AGREE is exact integer arithmetic: the student's rank of class a = argmax u_i is the number of classes
 * ordered before it, #{c : s_c > s_a or (s_c == s_a and c < a)} (lax.top_k puts the lower index first
 * among equal values), and out[i] = rank < k. */
int bv_distance(const float* student, int64_t ld_student, const float* teacher, int64_t ld_teacher, int32_t kind,
                float epsilon, float t, float ls, int32_t k, void* out, int64_t n, int32_t C, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BV_B200_DISTILL_H_ */
