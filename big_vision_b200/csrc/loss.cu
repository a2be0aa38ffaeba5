// Loss kernels.
//  * SigLIP pairwise sigmoid loss (K14): trainers/proj/image_text/siglip.py:291-306,
//    explicit per-device form trainers/proj/image_text/_deprecated_contrastive.py:117-141.
//      x_ij   = (zimg_i . ztxt_j) * exp(t') + b
//      loglik = log_sigmoid(+x_ij) on the positive diagonal, log_sigmoid(-x_ij) elsewhere
//      loss   = (1/B) sum_i sum_j -loglik_ij            (B = GLOBAL batch, siglip.py:306)
//    The dot products come from the wgmma GEMM; this kernel fuses scale+bias, the
//    loss reduction and d loss/d dot (written as the bf16 operand of the two gradient
//    GEMMs) plus the scalar gradients of t' and b in one pass over the [n, B] slab.
//  * sigmoid_xent / softmax_xent (K15): utils.py:236-243, 276-281.
#include "common.cuh"
#include "host_utils.h"

namespace bv {
namespace {

__device__ __forceinline__ float log_sigmoid(float y) {
  // log sigma(y) = min(y, 0) - log1p(exp(-|y|))   (stable; matches jax.nn.log_sigmoid)
  return fminf(y, 0.f) - log1pf(__expf(-fabsf(y)));
}
__device__ __forceinline__ float sigmoid(float y) { return 1.f / (1.f + __expf(-y)); }

__global__ void __launch_bounds__(256)
siglip_loss_kernel(const float* __restrict__ dots, int64_t n, int64_t B, int64_t ld,
                   int64_t row_offset, const float* __restrict__ t_param,
                   const float* __restrict__ b_param, float inv_B, bf16* __restrict__ G,
                   int64_t ldg, float* __restrict__ partials) {
  __shared__ float sh[96];
  const float t = __expf(t_param[0]);
  const float bias = b_param ? b_param[0] : 0.f;
  float l_acc = 0.f, t_acc = 0.f, b_acc = 0.f;
  const int64_t groups = B / 4;
  const int64_t total = n * groups;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = idx / groups;
    const int64_t j0 = (idx % groups) * 4;
    const float4 dv = *reinterpret_cast<const float4*>(dots + i * ld + j0);
    const float d[4] = {dv.x, dv.y, dv.z, dv.w};
    float g[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float sgn = (j0 + e == row_offset + i) ? 1.f : -1.f;
      const float x = d[e] * t + bias;
      l_acc -= log_sigmoid(sgn * x);
      const float gx = -sgn * sigmoid(-sgn * x) * inv_B;    // d loss / d x
      b_acc += gx;
      t_acc += gx * d[e] * t;                                // d x / d t' = dot * exp(t')
      g[e] = gx * t;                                         // d loss / d dot
    }
    uint2 q;
    q.x = pack_bf16(g[0], g[1]);
    q.y = pack_bf16(g[2], g[3]);
    *reinterpret_cast<uint2*>(G + i * ldg + j0) = q;
  }
  // one partial per block and scalar, summed in a fixed order by finish_row_sums: the result never
  // depends on which block finished first (XLA's reductions are run-to-run deterministic too)
  float sums[3] = {l_acc * inv_B, t_acc, b_acc};
  block_sum(sums, sh);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = sums[0];
    partials[gridDim.x + blockIdx.x] = sums[1];
    partials[2 * gridDim.x + blockIdx.x] = sums[2];
  }
}

// One direction of the softmax (CLIP) contrastive loss, _deprecated_contrastive.py:80-101:
//   x_ij = dots_ij * exp(t'),  loss_i = logsumexp_j x_ij - x_i,pos(i),  pos(i) = row_offset + i
//   loss += weight/global_B * sum_i loss_i ;  G_ij = weight/global_B * (softmax_ij - [j == pos]) * exp(t')
//   dt'  += sum_ij (G_ij / exp(t')) * x_ij ;  ncorrect += #[argmax_j x_ij == pos(i)]   (first max wins)
// One warp per row; per-row partials (loss, dt', correct) go to `rows_ws` [3, n] and are summed in a
// fixed order by finish_row_sums (deterministic like the other losses).
__global__ void __launch_bounds__(256)
softmax_contrastive_kernel(const float* __restrict__ dots, int64_t n, int64_t B, int64_t ld, int64_t row_offset,
                           const float* __restrict__ t_param, float scale, bf16* __restrict__ G, int64_t ldg,
                           float* __restrict__ rows_ws) {
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= n) return;
  const float t = __expf(t_param[0]);
  const float* d = dots + row * ld;
  const int64_t pos = row_offset + row;
  float mx = -INFINITY;
  int64_t arg = 0;
  for (int64_t c = lane; c < B; c += 32) {
    const float x = d[c] * t;
    if (x > mx) { mx = x; arg = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float omx = __shfl_xor_sync(0xffffffffu, mx, o);
    const int64_t oarg = __shfl_xor_sync(0xffffffffu, arg, o);
    if (omx > mx || (omx == mx && oarg < arg)) { mx = omx; arg = oarg; }
  }
  float se = 0.f;
  for (int64_t c = lane; c < B; c += 32) se += __expf(d[c] * t - mx);
  se = warp_sum(se);
  const float lse = mx + logf(se);
  float dt_acc = 0.f;
  for (int64_t c = lane; c < B; c += 32) {
    const float x = d[c] * t;
    const float gx = (__expf(x - lse) - (c == pos ? 1.f : 0.f)) * scale;     // d loss / d x
    dt_acc += gx * x;
    G[row * ldg + c] = __float2bfloat16_rn(gx * t);                            // d loss / d dot
  }
  dt_acc = warp_sum(dt_acc);
  if (lane == 0) {
    const float xpos = (pos >= 0 && pos < B) ? d[pos] * t : 0.f;
    rows_ws[row] = (lse - xpos) * scale;
    rows_ws[n + row] = dt_acc;
    rows_ws[2 * n + row] = (arg == pos) ? 1.f : 0.f;
  }
}

// one warp per row.  Row strides ldx / ldy / ldd; the dlogits columns C..ldd-1 are written as zeros, so
// a head stored with padded columns can feed the [n, ldd] gradient straight to its GEMMs.
__global__ void __launch_bounds__(256)
sigmoid_xent_kernel(const float* __restrict__ logits, int64_t ldx, const float* __restrict__ labels, int64_t ldy,
                    float* __restrict__ dlogits, int64_t ldd,
                    float* __restrict__ row_loss, int64_t n, int C) {
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= n) return;
  const float inv_n = 1.f / static_cast<float>(n);
  float acc = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float x = logits[row * ldx + c], y = labels[row * ldy + c];
    acc -= y * log_sigmoid(x) + (1.f - y) * log_sigmoid(-x);
    if (dlogits) dlogits[row * ldd + c] = (sigmoid(x) - y) * inv_n;
  }
  if (dlogits) {
    for (int64_t c = C + lane; c < ldd; c += 32) dlogits[row * ldd + c] = 0.f;
  }
  acc = warp_sum(acc);
  if (lane == 0) row_loss[row] = acc * inv_n;
}

__global__ void __launch_bounds__(256)
softmax_xent_kernel(const float* __restrict__ logits, int64_t ldx, const float* __restrict__ labels, int64_t ldy,
                    float* __restrict__ dlogits, int64_t ldd,
                    float* __restrict__ row_loss, int64_t n, int C) {
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= n) return;
  const float inv_n = 1.f / static_cast<float>(n);
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, logits[row * ldx + c]);
  mx = warp_max(mx);
  float se = 0.f, sy = 0.f, sxy = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float x = logits[row * ldx + c] - mx, y = labels[row * ldy + c];
    se += __expf(x); sy += y; sxy += y * x;
  }
  se = warp_sum(se); sy = warp_sum(sy); sxy = warp_sum(sxy);
  const float lse = logf(se);
  // -sum y (x - lse) = lse * sum(y) - sum(y x)
  if (lane == 0) row_loss[row] = (lse * sy - sxy) * inv_n;
  if (dlogits) {
    for (int c = lane; c < C; c += 32) {
      const float x = logits[row * ldx + c] - mx, y = labels[row * ldy + c];
      dlogits[row * ldd + c] = (__expf(x - lse) * sy - y) * inv_n;
    }
    for (int64_t c = C + lane; c < ldd; c += 32) dlogits[row * ldd + c] = 0.f;
  }
}

}  // namespace
}  // namespace bv

extern "C" {

int bv_siglip_loss(const float* dots, int64_t n, int64_t B, int64_t ld, int64_t row_offset,
                   const float* t_param, const float* b_param, int64_t global_B, void* G,
                   int64_t ldg, float* loss, float* dt, float* db, float* partials,
                   void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0 || B <= 0 || B % 4 || ld % 4 || ldg % 4 || global_B <= 0) {
    set_error("bv_siglip_loss: need n,B > 0 and B, ld, ldg multiples of 4");
    return BV_ERR_INVALID;
  }
  if (partials == nullptr) {
    set_error("bv_siglip_loss: need the workspace of BV_LOSS_WS_FLOATS floats");
    return BV_ERR_INVALID;
  }
  unsigned blocks = grid_for(n * (B / 4), 256, num_sms() * 8);
  if (blocks > BV_LOSS_WS_FLOATS / 3) blocks = BV_LOSS_WS_FLOATS / 3;
  siglip_loss_kernel<<<blocks, 256, 0, s>>>(dots, n, B, ld, row_offset, t_param, b_param,
                                            1.0f / static_cast<float>(global_B), reinterpret_cast<bf16*>(G), ldg,
                                            partials);
  int rc = check_cuda(cudaGetLastError(), "siglip_loss_kernel launch");
  if (rc) return rc;
  float* const outs[3] = {loss, dt, db};
  return finish_row_sums(partials, 3, blocks, outs, 1.f, true, s);
}

int bv_softmax_contrastive_loss(const float* dots, int64_t n, int64_t B, int64_t ld, int64_t row_offset,
                                const float* t_param, int64_t global_B, float weight, void* G, int64_t ldg,
                                float* loss, float* dt, float* ncorrect, float* rows_ws, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0 || B <= 0 || global_B <= 0 || rows_ws == nullptr) {
    set_error("bv_softmax_contrastive_loss: need n, B > 0 and the [3, n] workspace");
    return BV_ERR_INVALID;
  }
  softmax_contrastive_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(
      dots, n, B, ld, row_offset, t_param, weight / static_cast<float>(global_B), reinterpret_cast<bf16*>(G), ldg,
      rows_ws);
  int rc = check_cuda(cudaGetLastError(), "softmax_contrastive_kernel launch");
  if (rc) return rc;
  float* const outs[3] = {loss, dt, ncorrect};
  return finish_row_sums(rows_ws, 3, n, outs, 1.f, true, s);
}

int bv_sigmoid_xent_ld(const float* logits, int64_t ldx, const float* labels, int64_t ldy, float* loss,
                       float* dlogits, int64_t ldd, float* row_loss, int64_t n, int32_t C, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (ldx < C || ldy < C || ldd < C) {
    set_error("bv_sigmoid_xent_ld: row strides must be >= C (ld_logits %lld, ld_labels %lld, ld_dlogits %lld, C %d)",
              static_cast<long long>(ldx), static_cast<long long>(ldy), static_cast<long long>(ldd), C);
    return BV_ERR_INVALID;
  }
  if (n <= 0) return BV_OK;
  if (row_loss == nullptr) {
    set_error("bv_sigmoid_xent_ld: need the [n] workspace");
    return BV_ERR_INVALID;
  }
  sigmoid_xent_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(logits, ldx, labels, ldy, dlogits, ldd,
                                                                        row_loss, n, C);
  int rc = check_cuda(cudaGetLastError(), "sigmoid_xent_kernel launch");
  if (rc) return rc;
  return finish_row_sums(row_loss, 1, n, &loss, 1.f, true, s);
}
int bv_softmax_xent_ld(const float* logits, int64_t ldx, const float* labels, int64_t ldy, float* loss,
                       float* dlogits, int64_t ldd, float* row_loss, int64_t n, int32_t C, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (ldx < C || ldy < C || ldd < C) {
    set_error("bv_softmax_xent_ld: row strides must be >= C (ld_logits %lld, ld_labels %lld, ld_dlogits %lld, C %d)",
              static_cast<long long>(ldx), static_cast<long long>(ldy), static_cast<long long>(ldd), C);
    return BV_ERR_INVALID;
  }
  if (n <= 0) return BV_OK;
  if (row_loss == nullptr) {
    set_error("bv_softmax_xent_ld: need the [n] workspace");
    return BV_ERR_INVALID;
  }
  softmax_xent_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(logits, ldx, labels, ldy, dlogits, ldd,
                                                                        row_loss, n, C);
  int rc = check_cuda(cudaGetLastError(), "softmax_xent_kernel launch");
  if (rc) return rc;
  return finish_row_sums(row_loss, 1, n, &loss, 1.f, true, s);
}

}  // extern "C"
