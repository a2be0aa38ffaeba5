// Internal launcher declarations (C++ side of the C ABI in include/bv_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bv {

enum : int { EPI_NONE = 0, EPI_BIAS = 1, EPI_BIAS_GELU = 2, EPI_BIAS_RESID = 3, EPI_DGELU = 4,
             EPI_BIAS_GELU_ACT = 5 };

struct GemmArgs {
  const void* A; const void* B; void* D; void* D2;
  const float* bias; const void* aux;
  float* colsum;                        // optional [N] fp32: += column sums of the stored bf16 output
  int64_t M, N, K;
  int64_t lda, ldb, ldd, ldd2, ldaux;   // element strides of the stored matrices
  int a_mn, b_mn;                       // 0 = K-major storage, 1 = MN-major storage
  int epi, out_dtype, reduce_out, splits, block_n, aux_row_mod;
  float alpha;
};
int launch_gemm(const GemmArgs& g, cudaStream_t stream);

// ---- LayerNorm (layernorm.cu)
int launch_layernorm_fwd(const void* x, int x_dtype, const float* scale, const float* bias,
                         void* y, int y_dtype, float* mean, float* rstd, int64_t rows, int d,
                         float eps, cudaStream_t s);
int launch_layernorm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype,
                         const float* scale, const float* mean, const float* rstd,
                         const void* dres, void* dx, int dx_dtype, float* dscale, float* dbias,
                         float* dres_colsum, int64_t rows, int d, cudaStream_t s);

// ---- attention (attention.cu)
struct AttnArgs {
  const void* q; const void* k; const void* v;   // bf16, [B, N, ld] views with head h at col h*head_dim
  void* o;                                       // bf16 [B, Nq, ldo]
  float* lse;                                    // [B, H, Nq] fp32 (log-sum-exp of scaled scores)
  int64_t B; int H; int Nq; int Nk;
  int64_t ldq, ldk, ldv, ldo;                    // row strides (elements)
  int64_t bsq, bsk, bsv, bso;                    // batch strides (elements)
  float scale;
};
// head_dim: 64, 72, 80, 96 or 104 (anything else: BV_ERR_UNSUPPORTED before any CUDA call)
int launch_attention_fwd(const AttnArgs& a, int head_dim, cudaStream_t s);
struct AttnBwdArgs {
  AttnArgs f;
  const void* d_o; int64_t lddo, bsdo;
  void* dq; void* dk; void* dv;                  // bf16, same geometry as q/k/v
  float* dq_colsum; float* dk_colsum; float* dv_colsum;   // optional [H*head_dim] fp32 bias gradients
  int64_t lddq, lddk, lddv, bsdq, bsdk, bsdv;
  float* delta;                                  // workspace [B, H, Nq] fp32
};
int launch_attention_bwd(const AttnBwdArgs& a, int head_dim, cudaStream_t s);

// ---- integer evaluation paths (eval.cu)
int launch_top1(const void* logits, int dtype, int64_t rows, int C, int64_t ld, int32_t* idx,
                const float* labels, int64_t ldl, const float* mask, float* top1_correct,
                float* sums, cudaStream_t s);
int launch_retrieval_ranks(const float* dist, int64_t NI, int64_t NT, int64_t ld, const int32_t* corr,
                           int32_t* rank_t2i, int32_t* rank_i2t, cudaStream_t s);

// ---- element-wise / reductions (elementwise.cu)
int launch_patchify(const float* img, void* out, int64_t n, int H, int W, int C, int P,
                    cudaStream_t s);
int launch_patchify_u8(const uint8_t* img, void* out, int64_t n, int H, int W, int C, int P, float vmin,
                       float vmax, float in_min, float in_max, int clip, cudaStream_t s);
int launch_untranspose_add(const void* y, const void* res, void* out, int64_t n, int N, int d,
                           cudaStream_t s);
int launch_concat_cls(const void* x, const float* cls, void* out, int64_t n, int N0, int d,
                      cudaStream_t s);
int launch_drop_cls(const void* x, void* out, int64_t n, int N0, int d, cudaStream_t s);
int launch_embed_fwd(const int32_t* ids, const float* table, const float* pos, void* out,
                     int out_dtype, int64_t n, int L, int d, int vocab, cudaStream_t s);
int launch_embed_bwd(const int32_t* ids, const void* dy, int dy_dtype, float* dtable, float* dpos,
                     int64_t n, int L, int d, int vocab, cudaStream_t s);
int launch_colsum(const void* x, int x_dtype, float* out, int64_t rows, int64_t cols, int64_t ld,
                  cudaStream_t s);
int launch_cast(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n,
                cudaStream_t s);
int launch_l2norm_fwd(const void* x, int x_dtype, float* z, float* norm, int64_t n, int d,
                      float eps, cudaStream_t s);
int launch_l2norm_bwd(const float* dz, const float* z, const float* norm, void* dx, int dx_dtype,
                      int64_t n, int d, float eps, cudaStream_t s);
int launch_pool(const void* x, int x_dtype, void* y, int y_dtype, int64_t n, int N, int d,
                int mode, int tok_offset, cudaStream_t s);
int launch_pool_bwd(const void* dy, int dy_dtype, void* dx, int dx_dtype, int64_t n, int N, int d,
                    int mode, int tok_offset, cudaStream_t s);
int launch_pool_max_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, void* dx,
                        int dx_dtype, int64_t n, int N, int d, cudaStream_t s);
int launch_add_rows(const void* x, int x_dtype, const float* row, void* y, int y_dtype,
                    int64_t rows, int d, cudaStream_t s);
int launch_tanh_fwd(const void* x, void* y, int dtype, int64_t n, cudaStream_t s);
int launch_tanh_bwd(const void* dy, const void* y, void* dx, int dtype, int64_t n, cudaStream_t s);
int launch_gelu_fwd(const void* x, void* y, int dtype, int64_t n, cudaStream_t s);
int launch_mixup(const float* x, float* out, int64_t n, int64_t row_elems, float a, cudaStream_t s);
int launch_axpby(const void* x, const void* y, void* out, int dtype, float a, float b, int64_t n,
                 cudaStream_t s);
int launch_transpose_tokens(const void* x, void* y, int64_t n, int N, int d, cudaStream_t s);
int launch_row_select(const void* a, const void* b, const float* mask, void* out, int64_t n, int N,
                      int d, cudaStream_t s);

// ---- losses (loss.cu)
int launch_siglip_loss_ew(const float* dots, int64_t n, int64_t B, int64_t ld, int64_t row_offset,
                          const float* t_param, const float* b_param, int64_t global_B, void* G,
                          int64_t ldg, float* loss, float* dt, float* db, float* partials,
                          cudaStream_t s);
int launch_softmax_contrastive(const float* dots, int64_t n, int64_t B, int64_t ld, int64_t row_offset,
                               const float* t_param, int64_t global_B, float weight, void* G, int64_t ldg,
                               float* loss, float* dt, float* ncorrect, float* rows_ws, cudaStream_t s);
// row strides ldx / ldy / ldd >= C (else BV_ERR_INVALID before any CUDA call); dlogits columns C..ldd-1 = 0
int launch_sigmoid_xent(const float* logits, int64_t ldx, const float* labels, int64_t ldy, float* loss,
                        float* dlogits, int64_t ldd, float* row_loss, int64_t n, int C, cudaStream_t s);
int launch_softmax_xent(const float* logits, int64_t ldx, const float* labels, int64_t ldy, float* loss,
                        float* dlogits, int64_t ldd, float* row_loss, int64_t n, int C, cudaStream_t s);

// ---- optimizer (optim.cu)
struct AdamArgs {
  float* params; const float* grads; void* mu; float* nu; void* params_bf16;
  const float* wd_mask;     // per-element decay multiplier (0/1) or null
  int64_t n; int mu_dtype;
  float lr, b1, b2, eps, wd, grad_scale_host;   // grad_scale = clip factor computed on device
  const float* gnorm_sq;    // [1] device: sum of squared grads (for clipping); may be null
  float clip_norm;          // <=0 : no clipping
  int64_t step;             // 1-based
  float* upd_sq;            // [1] device accumulator of |update|^2 (may be null)
  float* param_sq;          // [1] device accumulator of |param|^2 (may be null)
};
int launch_adam(const AdamArgs& a, cudaStream_t s);
int launch_sumsq(const float* x, float* out, int64_t n, cudaStream_t s);
struct AdafactorArgs {
  float* params; const float* grads; void* params_bf16;
  int64_t A, L, M, H, sA, sL, sM;       // the tensor as a strided view [A, L, M, H] (H contiguous)
  int mode;                              // 0 unfactored, 1 factored with d0 = H, 2 factored with d0 = L
  float* vfull; float* red_h; float* red_l; float* nrm; void* momentum;
  float decay, eps, beta, lr, wd, grad_mult, clip_norm;
  const float* gnorm_sq; float* upd_sq; float* param_sq;
};
int launch_adafactor(const AdafactorArgs& a, cudaStream_t s);
int launch_scale_step(float* params, const float* grads, void* params_bf16, int64_t n, float lr, float wd,
                      float grad_mult, float clip_norm, const float* gnorm_sq, float* upd_sq,
                      float* param_sq, cudaStream_t s);

// ---- GSAM / SAM vector algebra (sam.cu; C ABI in include/bv_b200_sam.h)
int launch_sam_perturb(const float* w, const float* g, const float* g_sumsq, float rho, float eps, int adaptive,
                       float* w_out, void* w_bf16, int64_t n, cudaStream_t s);
int launch_sam_dots(const float* a, const float* b, float* out, float* ws, int64_t n, cudaStream_t s);
int launch_gsam_combine(float* gc, const float* gr, const float* dot, const float* norm_sq, float alpha,
                        int minimize_fp, int64_t n, cudaStream_t s);

}  // namespace bv
