// extern "C" surface of libbv_b200.so (see include/bv_b200.h and include/bv_b200_sam.h).
#include "../../include/bv_b200.h"
#include "../../include/bv_b200_sam.h"

#include "host_utils.h"
#include "kernels.h"

using namespace bv;

static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }

extern "C" {

const char* bv_last_error_string(void) { return last_error(); }
int bv_version(void) { return 100; }

int bv_device_supported(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  return major == 9 ? 1 : 0;
}

int bv_gemm(const bv_gemm_args* a, void* stream) {
  if (!a) { set_error("bv_gemm: null args"); return BV_ERR_INVALID; }
  GemmArgs g;
  g.A = a->A; g.B = a->B; g.D = a->D; g.D2 = a->D2; g.bias = a->bias; g.aux = a->aux;
  g.colsum = a->colsum;
  g.M = a->M; g.N = a->N; g.K = a->K;
  g.lda = a->lda; g.ldb = a->ldb; g.ldd = a->ldd; g.ldd2 = a->ldd2; g.ldaux = a->ldaux;
  g.a_mn = a->a_mn; g.b_mn = a->b_mn; g.epi = a->epilogue; g.out_dtype = a->out_dtype;
  g.reduce_out = a->reduce_out; g.splits = a->splits; g.block_n = a->block_n;
  g.aux_row_mod = a->aux_row_mod; g.alpha = a->alpha;
  return launch_gemm(g, S(stream));
}

int bv_layernorm_fwd(const void* x, int x_dtype, const float* scale, const float* bias, void* y,
                     int y_dtype, float* mean, float* rstd, int64_t rows, int32_t d, float eps,
                     void* stream) {
  return launch_layernorm_fwd(x, x_dtype, scale, bias, y, y_dtype, mean, rstd, rows, d, eps, S(stream));
}
int bv_layernorm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* scale,
                     const float* mean, const float* rstd, const void* dres, void* dx,
                     int dx_dtype, float* dscale, float* dbias, float* dx_colsum, int64_t rows,
                     int32_t d, void* stream) {
  return launch_layernorm_bwd(dy, dy_dtype, x, x_dtype, scale, mean, rstd, dres, dx, dx_dtype,
                              dscale, dbias, dx_colsum, rows, d, S(stream));
}

static AttnArgs to_attn(const bv_attn_args& a) {
  AttnArgs r;
  r.q = a.q; r.k = a.k; r.v = a.v; r.o = a.o; r.lse = a.lse;
  r.B = a.B; r.H = a.H; r.Nq = a.Nq; r.Nk = a.Nk;
  r.ldq = a.ldq; r.ldk = a.ldk; r.ldv = a.ldv; r.ldo = a.ldo;
  r.bsq = a.bsq; r.bsk = a.bsk; r.bsv = a.bsv; r.bso = a.bso;
  r.scale = a.scale;
  return r;
}
int bv_attention_fwd(const bv_attn_args* a, void* stream) { return bv_attention_fwd_hd(a, 64, stream); }
int bv_attention_fwd_hd(const bv_attn_args* a, int32_t head_dim, void* stream) {
  if (!a) { set_error("bv_attention_fwd: null args"); return BV_ERR_INVALID; }
  return launch_attention_fwd(to_attn(*a), head_dim, S(stream));
}
int bv_attention_bwd(const bv_attn_bwd_args* a, void* stream) { return bv_attention_bwd_hd(a, 64, stream); }
int bv_attention_bwd_hd(const bv_attn_bwd_args* a, int32_t head_dim, void* stream) {
  if (!a) { set_error("bv_attention_bwd: null args"); return BV_ERR_INVALID; }
  AttnBwdArgs g;
  g.f = to_attn(a->fwd);
  g.d_o = a->d_o; g.lddo = a->lddo; g.bsdo = a->bsdo;
  g.dq = a->dq; g.dk = a->dk; g.dv = a->dv;
  g.lddq = a->lddq; g.lddk = a->lddk; g.lddv = a->lddv;
  g.bsdq = a->bsdq; g.bsdk = a->bsdk; g.bsdv = a->bsdv;
  g.dq_colsum = a->dq_colsum; g.dk_colsum = a->dk_colsum; g.dv_colsum = a->dv_colsum;
  g.delta = a->delta;                  // a->dq_accum is ignored (kept for the struct layout)
  return launch_attention_bwd(g, head_dim, S(stream));
}

int bv_patchify(const float* image, void* patches, int64_t n, int32_t H, int32_t W, int32_t C,
                int32_t P, void* stream) {
  return launch_patchify(image, patches, n, H, W, C, P, S(stream));
}
int bv_patchify_u8(const uint8_t* image, void* patches, int64_t n, int32_t H, int32_t W, int32_t C,
                   int32_t P, float vmin, float vmax, float in_min, float in_max, int32_t clip_values,
                   void* stream) {
  return launch_patchify_u8(image, patches, n, H, W, C, P, vmin, vmax, in_min, in_max, clip_values, S(stream));
}
int bv_embed_fwd(const int32_t* ids, const float* table, const float* pos, void* out,
                 int out_dtype, int64_t n, int32_t L, int32_t d, int32_t vocab, void* stream) {
  return launch_embed_fwd(ids, table, pos, out, out_dtype, n, L, d, vocab, S(stream));
}
int bv_embed_bwd(const int32_t* ids, const void* dy, int dy_dtype, float* dtable, float* dpos,
                 int64_t n, int32_t L, int32_t d, int32_t vocab, void* stream) {
  return launch_embed_bwd(ids, dy, dy_dtype, dtable, dpos, n, L, d, vocab, S(stream));
}
int bv_colsum(const void* x, int x_dtype, float* out, int64_t rows, int64_t cols, int64_t ld,
              void* stream) {
  return launch_colsum(x, x_dtype, out, rows, cols, ld, S(stream));
}
int bv_cast(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n, void* stream) {
  return launch_cast(src, src_dtype, dst, dst_dtype, n, S(stream));
}
int bv_l2norm_fwd(const void* x, int x_dtype, float* z, float* norm, int64_t n, int32_t d,
                  float eps, void* stream) {
  return launch_l2norm_fwd(x, x_dtype, z, norm, n, d, eps, S(stream));
}
int bv_l2norm_bwd(const float* dz, const float* z, const float* norm, void* dx, int dx_dtype,
                  int64_t n, int32_t d, float eps, void* stream) {
  return launch_l2norm_bwd(dz, z, norm, dx, dx_dtype, n, d, eps, S(stream));
}
int bv_pool_fwd(const void* x, int x_dtype, void* y, int y_dtype, int64_t n, int32_t N, int32_t d,
                int32_t mode, int32_t tok, void* stream) {
  return launch_pool(x, x_dtype, y, y_dtype, n, N, d, mode, tok, S(stream));
}
int bv_pool_bwd(const void* dy, int dy_dtype, void* dx, int dx_dtype, int64_t n, int32_t N,
                int32_t d, int32_t mode, int32_t tok, void* stream) {
  return launch_pool_bwd(dy, dy_dtype, dx, dx_dtype, n, N, d, mode, tok, S(stream));
}
int bv_pool_max_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, void* dx, int dx_dtype,
                    int64_t n, int32_t N, int32_t d, void* stream) {
  return launch_pool_max_bwd(dy, dy_dtype, x, x_dtype, dx, dx_dtype, n, N, d, S(stream));
}
int bv_broadcast_row(const void* x, int x_dtype, const float* row, void* y, int y_dtype,
                     int64_t rows, int32_t d, void* stream) {
  return launch_add_rows(x, x_dtype, row, y, y_dtype, rows, d, S(stream));
}
int bv_tanh_fwd(const void* x, void* y, int dtype, int64_t n, void* stream) {
  return launch_tanh_fwd(x, y, dtype, n, S(stream));
}
int bv_tanh_bwd(const void* dy, const void* y, void* dx, int dtype, int64_t n, void* stream) {
  return launch_tanh_bwd(dy, y, dx, dtype, n, S(stream));
}
int bv_gelu_fwd(const void* x, void* y, int dtype, int64_t n, void* stream) {
  return launch_gelu_fwd(x, y, dtype, n, S(stream));
}
int bv_mixup(const float* x, float* out, int64_t n, int64_t row_elems, float a, void* stream) {
  return launch_mixup(x, out, n, row_elems, a, S(stream));
}
int bv_axpby(const void* x, const void* y, void* out, int dtype, float a, float b, int64_t n,
             void* stream) {
  return launch_axpby(x, y, out, dtype, a, b, n, S(stream));
}
int bv_untranspose_add(const void* y, const void* res, void* out, int64_t n, int32_t N, int32_t d,
                       void* stream) {
  return launch_untranspose_add(y, res, out, n, N, d, S(stream));
}
int bv_concat_cls(const void* x, const float* cls, void* out, int64_t n, int32_t N0, int32_t d,
                  void* stream) {
  return launch_concat_cls(x, cls, out, n, N0, d, S(stream));
}
int bv_drop_cls(const void* x, void* out, int64_t n, int32_t N0, int32_t d, void* stream) {
  return launch_drop_cls(x, out, n, N0, d, S(stream));
}
int bv_row_select(const void* a, const void* b, const float* mask, void* out, int64_t n, int32_t N,
                  int32_t d, void* stream) {
  return launch_row_select(a, b, mask, out, n, N, d, S(stream));
}
int bv_transpose_tokens(const void* x, void* y, int64_t n, int32_t N, int32_t d, void* stream) {
  return launch_transpose_tokens(x, y, n, N, d, S(stream));
}

int bv_siglip_loss(const float* dots, int64_t n, int64_t B, int64_t ld, int64_t row_offset,
                   const float* t_param, const float* b_param, int64_t global_B, void* G,
                   int64_t ldg, float* loss, float* dt, float* db, float* partials_ws,
                   void* stream) {
  return launch_siglip_loss_ew(dots, n, B, ld, row_offset, t_param, b_param, global_B, G, ldg,
                               loss, dt, db, partials_ws, S(stream));
}
int bv_softmax_contrastive_loss(const float* dots, int64_t n, int64_t B, int64_t ld, int64_t row_offset,
                                const float* t_param, int64_t global_B, float weight, void* G, int64_t ldg,
                                float* loss, float* dt, float* ncorrect, float* rows_ws, void* stream) {
  return launch_softmax_contrastive(dots, n, B, ld, row_offset, t_param, global_B, weight, G, ldg, loss, dt,
                                    ncorrect, rows_ws, S(stream));
}
int bv_sigmoid_xent(const float* logits, const float* labels, float* loss, float* dlogits,
                    float* row_loss_ws, int64_t n, int32_t C, void* stream) {
  return bv_sigmoid_xent_ld(logits, C, labels, C, loss, dlogits, C, row_loss_ws, n, C, stream);
}
int bv_sigmoid_xent_ld(const float* logits, int64_t ld_logits, const float* labels, int64_t ld_labels, float* loss,
                       float* dlogits, int64_t ld_dlogits, float* row_loss_ws, int64_t n, int32_t C, void* stream) {
  return launch_sigmoid_xent(logits, ld_logits, labels, ld_labels, loss, dlogits, ld_dlogits, row_loss_ws, n, C,
                             S(stream));
}
int bv_softmax_xent(const float* logits, const float* labels, float* loss, float* dlogits,
                    float* row_loss_ws, int64_t n, int32_t C, void* stream) {
  return bv_softmax_xent_ld(logits, C, labels, C, loss, dlogits, C, row_loss_ws, n, C, stream);
}
int bv_softmax_xent_ld(const float* logits, int64_t ld_logits, const float* labels, int64_t ld_labels, float* loss,
                       float* dlogits, int64_t ld_dlogits, float* row_loss_ws, int64_t n, int32_t C, void* stream) {
  return launch_softmax_xent(logits, ld_logits, labels, ld_labels, loss, dlogits, ld_dlogits, row_loss_ws, n, C,
                             S(stream));
}

int bv_adam_step(const bv_adam_args* a, void* stream) {
  if (!a) { set_error("bv_adam_step: null args"); return BV_ERR_INVALID; }
  AdamArgs g;
  g.params = a->params; g.grads = a->grads; g.mu = a->mu; g.nu = a->nu;
  g.params_bf16 = a->params_bf16; g.wd_mask = nullptr; g.n = a->n; g.mu_dtype = a->mu_dtype;
  g.lr = a->lr_eff; g.b1 = a->b1; g.b2 = a->b2; g.eps = a->eps; g.wd = a->wd_eff;
  g.grad_scale_host = a->grad_mult; g.gnorm_sq = a->gnorm_sq; g.clip_norm = a->clip_norm;
  g.step = a->step; g.upd_sq = a->upd_sq; g.param_sq = a->param_sq;
  return launch_adam(g, S(stream));
}
int bv_scale_step(float* params, const float* grads, void* params_bf16, int64_t n, float lr_eff,
                  float wd_eff, float grad_mult, float clip_norm, const float* gnorm_sq, float* upd_sq,
                  float* param_sq, void* stream) {
  return launch_scale_step(params, grads, params_bf16, n, lr_eff, wd_eff, grad_mult, clip_norm, gnorm_sq,
                           upd_sq, param_sq, S(stream));
}
int bv_adafactor_step(const bv_adafactor_args* a, void* stream) {
  if (!a) { set_error("bv_adafactor_step: null args"); return BV_ERR_INVALID; }
  AdafactorArgs g;
  g.params = a->params; g.grads = a->grads; g.params_bf16 = a->params_bf16;
  g.A = a->A; g.L = a->L; g.M = a->M; g.H = a->H; g.sA = a->sA; g.sL = a->sL; g.sM = a->sM;
  g.mode = a->mode; g.vfull = a->vfull; g.red_h = a->red_h; g.red_l = a->red_l; g.nrm = a->nrm;
  g.momentum = a->momentum; g.decay = a->decay; g.eps = a->eps; g.beta = a->beta; g.lr = a->lr_eff;
  g.wd = a->wd_eff; g.grad_mult = a->grad_mult; g.clip_norm = a->clip_norm; g.gnorm_sq = a->gnorm_sq;
  g.upd_sq = a->upd_sq; g.param_sq = a->param_sq;
  return launch_adafactor(g, S(stream));
}
int bv_sumsq(const float* x, float* out, int64_t n, void* stream) {
  return launch_sumsq(x, out, n, S(stream));
}
int bv_top1(const void* logits, int logits_dtype, int64_t rows, int32_t C, int64_t ld, int32_t* idx,
            const float* labels, int64_t ldl, const float* mask, float* top1_correct, float* sums,
            void* stream) {
  return launch_top1(logits, logits_dtype, rows, C, ld, idx, labels, ldl, mask, top1_correct, sums, S(stream));
}
int bv_retrieval_ranks(const float* dist, int64_t NI, int64_t NT, int64_t ld, const int32_t* corr,
                       int32_t* rank_t2i, int32_t* rank_i2t, void* stream) {
  return launch_retrieval_ranks(dist, NI, NT, ld, corr, rank_t2i, rank_i2t, S(stream));
}

int bv_sam_perturb(const float* w, const float* g, const float* g_sumsq, float rho, float eps, int32_t adaptive,
                   float* w_out, void* w_bf16, int64_t n, void* stream) {
  return launch_sam_perturb(w, g, g_sumsq, rho, eps, adaptive, w_out, w_bf16, n, S(stream));
}
int bv_sam_dots(const float* a, const float* b, float* out, float* ws, int64_t n, void* stream) {
  return launch_sam_dots(a, b, out, ws, n, S(stream));
}
int bv_gsam_combine(float* g_clean, const float* g_robust, const float* dot, const float* norm_sq, float alpha,
                    int32_t minimize_fp, int64_t n, void* stream) {
  return launch_gsam_combine(g_clean, g_robust, dot, norm_sq, alpha, minimize_fp, n, S(stream));
}

}  // extern "C"
