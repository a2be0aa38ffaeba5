/* bv_b200.h -- C ABI of libbv_b200.so: the H100-native (sm_90a) kernels for the
 * big_vision ViT / MLP-Mixer / SigLIP training hot path.
 *
 * The reference (google-research/big_vision) has no operator/FFI ABI of its own: the
 * arithmetic below is issued through flax.linen / jax.nn call sites inside jitted
 * Python (SURVEY.md section 8b).  Each entry point therefore cites the reference call
 * site(s) whose computation it replaces; INTEGRATION.md shows the jax.ffi / ctypes
 * binding a maintainer would add on the reference side.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless stated otherwise; the caller owns all
 *    buffers (inputs, outputs, saved-for-backward, workspace);
 *  - functions only ENQUEUE work on `stream` (a cudaStream_t passed as void*); they
 *    never allocate device memory and never synchronise;
 *  - return 0 on success, a negative BV_ERR_* code otherwise; bv_last_error_string()
 *    (thread-local) describes the last failure;
 *  - dtype codes: BV_F32 = 0, BV_BF16 = 1.  Matrix operands of the tensor-core paths
 *    are bf16 with fp32 accumulation; statistics, losses, parameters and parameter
 *    gradients are fp32;
 *  - "ld*" are row strides in ELEMENTS.  TMA operands need 16-byte aligned bases and
 *    row strides that are multiples of 8 bf16 / 4 fp32 elements.
 */
#ifndef BV_B200_H_
#define BV_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BV_OK 0
#define BV_ERR_INVALID (-1)
#define BV_ERR_CUDA (-2)
#define BV_ERR_UNSUPPORTED (-3)

#define BV_F32 0
#define BV_BF16 1

/* GEMM epilogues */
#define BV_EPI_NONE 0        /* D = alpha*acc  (bias, if given, is ignored)          */
#define BV_EPI_BIAS 1        /* D = alpha*acc + bias[n]                              */
#define BV_EPI_BIAS_GELU 2   /* D2 = bf16(alpha*acc + bias); D = gelu_tanh(D2)       */
#define BV_EPI_BIAS_RESID 3  /* D = bf16(alpha*acc + bias) + aux[m (% aux_row_mod), n] */
#define BV_EPI_DGELU 4       /* D = alpha*acc * gelu_tanh'(aux[m, n])                */
#define BV_EPI_BIAS_GELU_ACT 5 /* D = gelu_tanh(bf16(alpha*acc + bias)); no D2: the
                                  forward-only BIAS_GELU (same bits as its D)          */

const char* bv_last_error_string(void);
int bv_version(void);
/* 1 if the library was compiled for sm_90a and a device of compute capability 9.x is
 * current; the product path refuses to run otherwise (no CPU / other-arch fallback). */
int bv_device_supported(void);

/* ---------------------------------------------------------------------------------
 * Dense contraction  D[M,N] = epilogue(alpha * sum_k A(m,k) B(n,k))   (wgmma + TMA)
 * Replaces flax nn.Dense / nn.DenseGeneral / nn.Conv(patch,stride=patch) forward and both
 * backward contractions: models/vit.py:72,77 (MlpBlock), :93-98 and :176-178
 * (q/k/v/out projections inside MultiHeadDotProductAttention), :212-214 (patch embed as
 * im2col GEMM), :261,272 (pre_logits, head); models/mlp_mixer.py:35-37,72,82;
 * models/proj/image_text/text_transformer.py:98; the logits product
 * trainers/proj/image_text/siglip.py:291.
 *   a_mn / b_mn : 0 = operand stored K-major  ([M or N rows, K contiguous]),
 *                 1 = operand stored MN-major ([K rows, M or N contiguous]).
 *     forward  Y = X W    : A=X (a_mn=0), B=W[K,N] (b_mn=1)
 *     dgrad    dX = dY W^T: A=dY (a_mn=0), B=W[K,N] read as [N'=K rows, K'=N] (b_mn=0)
 *     wgrad    dW = X^T dY: A=X (a_mn=1), B=dY (b_mn=1), out fp32, reduce_out=1
 *   reduce_out : 1 = accumulate into D with atomic adds (split-K / grad accumulation)
 *   splits     : 0 = auto (more than one split only with reduce_out, once K >= 2048), >1 only
 *                with reduce_out.  Under split-K each split's partial goes through the epilogue,
 *                is rounded to the output dtype and added into D on its own, in no fixed order;
 *                bias and the BIAS_RESID aux are added once (by the first split), DGELU's
 *                gelu'(aux) scales every partial.
 *   block_n    : output tile width, 0 = auto, else 128 or 256.  128 runs the two consumer
 *                warpgroups ping-pong on alternate tiles, 256 runs them together on each tile;
 *                the output bits are the same.  Auto: 256 for fp32 outputs with N > 128, else
 *                128.  bf16 reduce-adds (reduce_out with a bf16 output) are fixed at 128.
 *   bias (fp32 [N]) and aux (bf16) must be readable up to round_up(N, 8) columns.
 * --------------------------------------------------------------------------------- */
typedef struct bv_gemm_args {
  const void* A; const void* B; void* D; void* D2;
  const float* bias; const void* aux;
  float* colsum;   /* optional fp32 [N]: += column sums of the stored bf16 output (bias gradient) */
  int64_t M, N, K;
  int64_t lda, ldb, ldd, ldd2, ldaux;
  int32_t a_mn, b_mn;
  int32_t epilogue, out_dtype, reduce_out, splits, block_n, aux_row_mod;
  float alpha;
} bv_gemm_args;
int bv_gemm(const bv_gemm_args* args, void* stream);

/* ---------------------------------------------------------------------------------
 * LayerNorm (flax nn.LayerNorm, eps=1e-6, fast variance; models/vit.py:92,103,160,181,
 * models/mlp_mixer.py:48,53,79).  x,y: [rows,d], d % 8 == 0, d <= 2048.
 * bwd: dx = dres + LN'(dy); dscale/dbias/dx_colsum are ACCUMULATED (atomics); any of
 * dres, dscale, dbias, dx_colsum may be NULL.  dres has dtype dx_dtype.  dx_colsum receives the
 * column sums of dx (summed in fp32; the streaming bf16 path sums before the bf16 rounding of dx).
 * --------------------------------------------------------------------------------- */
int bv_layernorm_fwd(const void* x, int x_dtype, const float* scale, const float* bias, void* y,
                     int y_dtype, float* mean, float* rstd, int64_t rows, int32_t d, float eps,
                     void* stream);
int bv_layernorm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* scale,
                     const float* mean, const float* rstd, const void* dres, void* dx,
                     int dx_dtype, float* dscale, float* dbias, float* dx_colsum, int64_t rows,
                     int32_t d, void* stream);

/* ---------------------------------------------------------------------------------
 * Scaled-dot-product attention, optional key-padding mask, any Nq, Nk >= 1
 * (flax MultiHeadDotProductAttention core: models/vit.py:93-98, :176-178).  Keys stream through
 * on-chip memory in 64-key blocks (online combination of per-block softmax statistics), so every
 * sequence length takes the same path.
 * Head dim dh: 64, 72, 80, 96 or 104 (ViT Ti..L, So400m, H, g-opt / G-opt, G).  The entry points take
 * dh and refuse any other value with BV_ERR_UNSUPPORTED before touching the device.
 * q/k/v/o are bf16 strided views: element (b, t, h*dh + j) at
 * base + b*bs + t*ld + h*dh + j  (e.g. column slices of the fused QKV GEMM output).
 * lse [B,H,Nq] fp32 = log sum_j exp(scale * q_i.k_j) is saved for the backward.
 * Key-padding mask (dh = 64 only; the reference's BERT input_mask, models/proj/flaxformer/bert.py:54):
 * pass head_dim | BV_ATTN_KEY_MASK, and args then points to a bv_attn_masked_args (forward) or a
 * bv_attn_masked_bwd_args (backward), which append the mask to the unmasked arguments.  key_mask is
 * uint8, element (b, k) at key_mask[b*bsmask + k], nonzero = attend; masked keys get probability 0
 * wherever they sit.  A query with every key masked gets O = 0, lse = 0 and zero gradients.  The flag
 * at any other head dim, or with a NULL key_mask, is refused with BV_ERR_INVALID before any launch.
 * --------------------------------------------------------------------------------- */
typedef struct bv_attn_args {
  const void* q; const void* k; const void* v; void* o; float* lse;
  int64_t B; int32_t H, Nq, Nk;
  int64_t ldq, ldk, ldv, ldo;
  int64_t bsq, bsk, bsv, bso;
  float scale;
} bv_attn_args;
#define BV_ATTN_KEY_MASK 65536   /* head_dim flag: args carries a key mask (see above) */
int bv_attention_fwd_hd(const bv_attn_args* args, int32_t head_dim, void* stream);
typedef struct bv_attn_bwd_args {
  bv_attn_args fwd;            /* same q,k,v,o,lse as the forward call */
  const void* d_o; int64_t lddo, bsdo;
  void* dq; void* dk; void* dv;
  int64_t lddq, lddk, lddv, bsdq, bsdk, bsdv;
  /* optional fp32 [H*dh] each: += column sums over the valid rows of dq / dk / dv, i.e. the bias
   * gradients of the projections that produced q / k / v */
  float* dq_colsum; float* dk_colsum; float* dv_colsum;
  /* REQUIRED workspace: delta [B,H,Nq] fp32 = rowsum(O o dO).  dq, dk and dv are each summed in a
   * fixed order inside one kernel (reproducible bit for bit), with no other workspace. */
  float* delta;
} bv_attn_bwd_args;
int bv_attention_bwd_hd(const bv_attn_bwd_args* args, int32_t head_dim, void* stream);
typedef struct bv_attn_masked_args {
  bv_attn_args attn;
  const uint8_t* key_mask; int64_t bsmask;
} bv_attn_masked_args;
typedef struct bv_attn_masked_bwd_args {
  bv_attn_bwd_args attn;       /* attn.fwd: the forward call's arguments */
  const uint8_t* key_mask; int64_t bsmask;   /* the forward call's mask */
} bv_attn_masked_bwd_args;

/* ---------------------------------------------------------------------------------
 * Data movement / small reductions
 * --------------------------------------------------------------------------------- */
/* image [n,H,W,C] fp32 NHWC -> bf16 patches [n*(H/P)*(W/P), round_up(P*P*C,8)], column order
 * (ph,pw,c) = row-major HWIO conv kernel (models/vit.py:212-217). */
int bv_patchify(const float* image, void* patches, int64_t n, int32_t H, int32_t W, int32_t C,
                int32_t P, void* stream);
/* The same patch extraction from the DECODED uint8 image with the input pipeline's value_range op
 * fused in (pp/ops_general.py:32-64; configs/vit_i1k.py:96 `value_range(-1, 1)`):
 *   y = vmin + ((float(u8) - in_min) / (in_max - in_min)) * (vmax - vmin), optionally clipped;
 * fp32, each operation rounded separately (bit-identical to the TensorFlow op), then bf16.  Cuts the
 * host->device bytes of the image hand-off (input_pipeline.py:316-329) by 4. */
int bv_patchify_u8(const uint8_t* image, void* patches, int64_t n, int32_t H, int32_t W, int32_t C,
                   int32_t P, float vmin, float vmax, float in_min, float in_max, int32_t clip_values,
                   void* stream);
/* out[b,l,:] = table[ids[b,l],:] + pos[l,:] (text_transformer.py:63-70); pos may be NULL */
int bv_embed_fwd(const int32_t* ids, const float* table, const float* pos, void* out,
                 int out_dtype, int64_t n, int32_t L, int32_t d, int32_t vocab, void* stream);
/* backward of the embedding lookup + position embedding (text_transformer.py:63-70):
   dtable[ids] += dy (atomics), dpos[l] += sum_b dy; either may be NULL */
int bv_embed_bwd(const int32_t* ids, const void* dy, int dy_dtype, float* dtable, float* dpos,
                 int64_t n, int32_t L, int32_t d, int32_t vocab, void* stream);
/* out[c] += sum_r x[r,c] : the bias gradients of flax Dense / DenseGeneral (models/vit.py:72-77,95) and
   the batch sums behind the pos_embedding / cls gradients (models/vit.py:219-225) */
int bv_colsum(const void* x, int x_dtype, float* out, int64_t rows, int64_t cols, int64_t ld,
              void* stream);
/* dtype conversion fp32 <-> bf16: the `dtype_mm` casts of the reference's Dense layers (models/vit.py:61,72-78) */
int bv_cast(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n, void* stream);
/* z = x / (||x||_2 + eps) (two_towers.py:60-61,73-74) */
int bv_l2norm_fwd(const void* x, int x_dtype, float* z, float* norm, int64_t n, int32_t d,
                  float eps, void* stream);
int bv_l2norm_bwd(const float* dz, const float* z, const float* norm, void* dx, int dx_dtype,
                  int64_t n, int32_t d, float eps, void* stream);
/* mode 0: mean over tokens (gap); mode 1: take token `tok` (models/vit.py:245-253);
   mode 2: max over tokens ("max"/"gmp", text_transformer.py:89-90), backward = bv_pool_max_bwd */
int bv_pool_fwd(const void* x, int x_dtype, void* y, int y_dtype, int64_t n, int32_t N, int32_t d,
                int32_t mode, int32_t tok, void* stream);
int bv_pool_bwd(const void* dy, int dy_dtype, void* dx, int dx_dtype, int64_t n, int32_t N,
                int32_t d, int32_t mode, int32_t tok, void* stream);
/* gradient of the mode-2 pool: dy[n,d] goes to the positions of x[n,N,d] holding the column maximum,
   split evenly between ties (the jnp.max differentiation rule; text_transformer.py:89-90) */
int bv_pool_max_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, void* dx, int dx_dtype,
                    int64_t n, int32_t N, int32_t d, void* stream);
/* y[r,:] = x[0,:] (+ row[:]) for r < rows : broadcast one row (MAP probe, models/vit.py:174) */
int bv_broadcast_row(const void* x, int x_dtype, const float* row, void* y, int y_dtype,
                     int64_t rows, int32_t d, void* stream);
int bv_tanh_fwd(const void* x, void* y, int dtype, int64_t n, void* stream);
int bv_tanh_bwd(const void* dy, const void* y, void* dx, int dtype, int64_t n, void* stream);
int bv_gelu_fwd(const void* x, void* y, int dtype, int64_t n, void* stream);
/* utils.py:1146-1158 (get_mixup): out[i,:] = a * x[i,:] + (1-a) * x[(i-1) mod n,:], fp32, out != x;
 * products and sum rounded separately (bit-identical to the fp32 expression).  Any row_elems >= 1 and
 * 4-byte aligned buffers; 16-byte vectors when row_elems % 4 == 0 and both buffers are 16-byte aligned. */
int bv_mixup(const float* x, float* out, int64_t n, int64_t row_elems, float a, void* stream);
int bv_axpby(const void* x, const void* y, void* out, int dtype, float a, float b, int64_t n,
             void* stream);
/* cls token (models/vit.py:223-225): out[b,0,:] = cls, out[b,1+t,:] = x[b,t,:]  (bf16, cls fp32) */
int bv_concat_cls(const void* x, const float* cls, void* out, int64_t n, int32_t N0, int32_t d,
                  void* stream);
/* out[b,t,:] = x[b,1+t,:] : the patch rows of a [n,N0+1,d] tensor (backward of the concat of
   models/vit.py:223-225; also `encoded[:, 1:]` of models/vit.py:251) */
int bv_drop_cls(const void* x, void* out, int64_t n, int32_t N0, int32_t d, void* stream);
/* bf16 [n,N,d] -> [n,d,round_up(N,8)] (zero pad): Mixer token mixing, mlp_mixer.py:49-51 */
int bv_transpose_tokens(const void* x, void* y, int64_t n, int32_t N, int32_t d, void* stream);

/* out[b,t,:] = (res ? res[b,t,:] : 0) + y[b,:,t], y stored [n,d,round_up(N,8)]: the transpose back
 * fused with the residual add (mlp_mixer.py:51-52); res may be NULL */
int bv_untranspose_add(const void* y, const void* res, void* out, int64_t n, int32_t N, int32_t d,
                       void* stream);

/* Stochastic-depth residual gate (models/mlp_mixer.py:52,55 with the per-sample mask of :173-177,
 * mask = 1 - Bernoulli(drop_p), no 1/(1-p) rescale): out[b,t,:] = mask[b] != 0 ? a[b,t,:] :
 * (b ? b[b,t,:] : 0).  a, b, out bf16 [n,N,d]; mask fp32 [n]; b may be NULL (backward: mask * dout). */
int bv_row_select(const void* a, const void* b, const float* mask, void* out, int64_t n, int32_t N,
                  int32_t d, void* stream);

/* ---------------------------------------------------------------------------------
 * Losses
 * --------------------------------------------------------------------------------- */
/* SigLIP pairwise sigmoid loss on a slab of dot products dots[n,B] = zimg_local . ztxt_all^T
 * (trainers/proj/image_text/siglip.py:291-306; per-device form
 * _deprecated_contrastive.py:117-141).  row_offset = rank*n locates the positives.
 * Accumulates: loss += sum_ij -loglik_ij / global_B ; dt += dloss/dt' ; db += dloss/db.
 * Writes G[n,B] (bf16) = dloss/ddots.
 * partials_ws: BV_LOSS_WS_FLOATS floats of per-block partials, summed in a fixed order, so the scalars
 * are run-to-run deterministic like the reference.  NULL: BV_ERR_INVALID before any CUDA call. */
#define BV_LOSS_WS_FLOATS 8192
int bv_siglip_loss(const float* dots, int64_t n, int64_t B, int64_t ld, int64_t row_offset,
                   const float* t_param, const float* b_param, int64_t global_B, void* G,
                   int64_t ldg, float* loss, float* dt, float* db, float* partials_ws,
                   void* stream);
/* One direction of the softmax (CLIP) contrastive loss, `softmax_loss` of
 * trainers/proj/image_text/_deprecated_contrastive.py:80-101, on a slab dots[n,B] = z1_local . z2_all^T:
 *   x = dots * exp(t'); loss += weight/global_B * sum_i (logsumexp_j x_ij - x_i,pos(i)), pos(i) = row_offset+i;
 *   G[n,B] (bf16) = d loss / d dots; dt += d loss / d t'; ncorrect += #(argmax_j x_ij == pos(i)).
 * rows_ws: [3, n] floats (per-row partials, summed in a fixed order: deterministic).  The trainer
 * calls it once per direction (i2t, t2i) with weight 0.5. */
int bv_softmax_contrastive_loss(const float* dots, int64_t n, int64_t B, int64_t ld, int64_t row_offset,
                                const float* t_param, int64_t global_B, float weight, void* G, int64_t ldg,
                                float* loss, float* dt, float* ncorrect, float* rows_ws, void* stream);
/* utils.py:236-243 / 276-281 : mean over n rows; loss is accumulated; dlogits may be NULL.
 * row_loss_ws: [n] floats of per-row losses, summed in a fixed order (deterministic).  NULL with n > 0:
 * BV_ERR_INVALID before any CUDA call.
 * Row-strided logits [n, ld_logits], labels [n, ld_labels] and dlogits [n, ld_dlogits] (columns 0..C-1
 * used).  The dlogits columns C..ld_dlogits-1 are written as zeros, so a classifier head stored with
 * padded columns takes the gradient as its GEMM operand unchanged.  Any ld < C: BV_ERR_INVALID before
 * any CUDA call. */
int bv_sigmoid_xent_ld(const float* logits, int64_t ld_logits, const float* labels, int64_t ld_labels, float* loss,
                       float* dlogits, int64_t ld_dlogits, float* row_loss_ws, int64_t n, int32_t C, void* stream);
int bv_softmax_xent_ld(const float* logits, int64_t ld_logits, const float* labels, int64_t ld_labels, float* loss,
                       float* dlogits, int64_t ld_dlogits, float* row_loss_ws, int64_t n, int32_t C, void* stream);

/* ---------------------------------------------------------------------------------
 * Optimizer (optax.py:143-149 chain with scale_by_adam; siglip.py:312-321)
 *   g' = g * grad_mult * clip(gnorm)           m,v Adam moments (mu bf16 or fp32)
 *   p += -(lr_eff * mhat/(sqrt(vhat)+eps) + wd_eff * p)
 * lr_eff / wd_eff already include the schedule value for this step.  Also writes the
 * bf16 shadow copy (params_bf16, may be NULL) and accumulates |update|^2, |param|^2.
 * --------------------------------------------------------------------------------- */
typedef struct bv_adam_args {
  float* params; const float* grads; void* mu; float* nu; void* params_bf16;
  int64_t n; int32_t mu_dtype;
  float lr_eff, b1, b2, eps, wd_eff, grad_mult, clip_norm;
  const float* gnorm_sq;     /* device scalar: sum of squares of ALL grads (pre grad_mult) */
  int64_t step;              /* 1-based */
  float* upd_sq; float* param_sq;
} bv_adam_args;
int bv_adam_step(const bv_adam_args* args, void* stream);
/* out[0] += sum x^2 : optax.global_norm of the gradients / updates / params (optax.py:100-105
   `clip_by_global_norm`; trainers/proj/image_text/siglip.py:316-321 `l2_grads`, `l2_params`, `l2_updates`) */
int bv_sumsq(const float* x, float* out, int64_t n, void* stream);
/* The same chain with optax.scale(step_size) as the inner transform (plain SGD; what the reference's
 * optimizer known-answer tests drive, optax_test.py:103-299): p += -(lr_eff * g' + wd_eff * p) with
 * g' = g * grad_mult * clip(gnorm); lr_eff already holds schedule * lr * lr_mult * step_size. */
int bv_scale_step(float* params, const float* grads, void* params_bf16, int64_t n, float lr_eff,
                  float wd_eff, float grad_mult, float clip_norm, const float* gnorm_sq, float* upd_sq,
                  float* param_sq, void* stream);

/* BV-Adafactor (`big_vision.scale_by_adafactor`, optax.py:187-214: optax.scale_by_factored_rms with
 * decay min(beta2_cap, 1 - (t+1)^-0.8), min_dim_size_to_factor 32, eps 1e-30, then optax.ema(momentum,
 * debias=False, bf16 accumulator)) for ONE reference tensor given as the strided view [A, L, M, H] of the
 * flat buffers (element strides sA, sL, sM; H contiguous), inside the same outer chain as bv_adam_step:
 *   mode 0  unfactored: vfull [A*L*M*H] <- decay*vfull + (1-decay)(g'^2+eps);  u = g' * vfull^-1/2
 *   mode 1  factored, largest axis d0 = H, d1 = L;   mode 2  factored, d0 = L, d1 = H:
 *           red_h [A,L,M] <- ema(mean_H(g'^2+eps)), red_l [A,M,H] <- ema(mean_L(g'^2+eps)),
 *           nrm [A,M] = mean_{d1}(R0) (scratch), u = g' * (R0/nrm)^-1/2 * R1^-1/2   (R0 = stat reduced over d0)
 *   momentum (bf16 [A*L*M*H], may be NULL): m <- beta*m + (1-beta)*u, u = m (pre-rounding value)
 *   p += -(lr_eff * u + wd_eff * p);  g' = g * grad_mult * clip(gnorm) as in bv_adam_step.
 * `decay` is the step's second-moment decay, computed by the caller. */
typedef struct bv_adafactor_args {
  float* params; const float* grads; void* params_bf16;
  int64_t A, L, M, H, sA, sL, sM;
  int32_t mode;
  float* vfull; float* red_h; float* red_l; float* nrm; void* momentum;
  float decay, eps, beta, lr_eff, wd_eff, grad_mult, clip_norm;
  const float* gnorm_sq; float* upd_sq; float* param_sq;
} bv_adafactor_args;
int bv_adafactor_step(const bv_adafactor_args* args, void* stream);

/* ---------------------------------------------------------------------------------
 * Integer evaluation paths (bit-exact index arithmetic)
 * bv_top1 -- evaluators/classification.py:46-52 and the zero-shot argmax of
 *   evaluators/proj/image_text/discriminative_classifier.py:284-288:
 *   idx[r] = argmax_c logits[r,c] (first maximal index, NaN counts as maximal; fp32 or bf16 logits,
 *   row stride ld).  With labels [rows,C] fp32 (row stride ldl): top1_correct[r] = labels[r,idx[r]],
 *   m[r] = mask[r] * max_c labels[r,c] (mask NULL = ones), sums[0] += sum top1_correct*m (ncorrect),
 *   sums[1] += sum m (nseen).  idx, labels, mask, top1_correct, sums may each be NULL.
 * bv_retrieval_ranks -- evaluators/proj/image_text/image_text_retrieval.py:23-85 on the distance
 *   matrix dist [NI images, NT texts] fp32 (row stride ld) with corr[j] = image of text j:
 *   rank_t2i[j] = position of image corr[j] in the ascending order of column j;
 *   rank_i2t[i] = position of the first text of image i in the ascending order of row i
 *   (INT32_MAX if image i has no text / corr[j] is out of range).  Ties order by index (stable
 *   argsort).  Recall@k = mean(rank < k).  Either output may be NULL. */
int bv_top1(const void* logits, int logits_dtype, int64_t rows, int32_t C, int64_t ld, int32_t* idx,
            const float* labels, int64_t ldl, const float* mask, float* top1_correct, float* sums,
            void* stream);
int bv_retrieval_ranks(const float* dist, int64_t NI, int64_t NT, int64_t ld, const int32_t* corr,
                       int32_t* rank_t2i, int32_t* rank_i2t, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BV_B200_H_ */
