// Fused optimizer step over a flat parameter buffer.  Reference chain
// (optax.py:143-149): clip_by_global_norm -> scale_by_adam(b1,b2,eps,mu_dtype) ->
// scale(lr) -> add_decayed_weights(wd, mask) -> scale_by_schedule -> scale(-1),
// followed by optax.apply_updates (trainers/proj/image_text/siglip.py:312-313).
// One launch per (wd, lr-mult) parameter group updates fp32 master weights, both Adam
// moments, and the bf16 shadow copy the GEMMs read; it also accumulates the
// l2_params / l2_updates measurements (siglip.py:315-321).  HBM-bound:
// 4+4 (p) + 4 (g) + 2x(2|4) (mu) + 4+4 (nu) + 2 (bf16 shadow) bytes per element.
#include "common.cuh"
#include "host_utils.h"

namespace bv {
namespace {

template <bool MU_BF16>
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, void* __restrict__ mu,
            float* __restrict__ nu, bf16* __restrict__ p16, int64_t n, float lr, float b1,
            float b2, float eps, float wd, float bc1, float bc2, const float* __restrict__ gnorm_sq,
            float clip_norm, float grad_mult, float* __restrict__ upd_sq,
            float* __restrict__ param_sq) {
  __shared__ float sh[64];
  float gscale = grad_mult;
  if (clip_norm > 0.f && gnorm_sq != nullptr) {
    // optax.clip_by_global_norm: g if ||g|| < c else g / ||g|| * c
    const float gn = sqrtf(gnorm_sq[0]) * grad_mult;
    if (!(gn < clip_norm)) gscale *= clip_norm / gn;
  }
  float us = 0.f, ps = 0.f;
  const int64_t n4 = n / 4;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float4 pv = reinterpret_cast<float4*>(p)[i];
    const float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 nv = reinterpret_cast<float4*>(nu)[i];
    float m[4];
    if (MU_BF16) {
      const uint2 q = reinterpret_cast<const uint2*>(mu)[i];
      m[0] = bf16_lo(q.x); m[1] = bf16_hi(q.x); m[2] = bf16_lo(q.y); m[3] = bf16_hi(q.y);
    } else {
      const float4 q = reinterpret_cast<const float4*>(mu)[i];
      m[0] = q.x; m[1] = q.y; m[2] = q.z; m[3] = q.w;
    }
    float pp[4] = {pv.x, pv.y, pv.z, pv.w};
    const float gg[4] = {gv.x, gv.y, gv.z, gv.w};
    float vv[4] = {nv.x, nv.y, nv.z, nv.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float gr = gg[e] * gscale;
      m[e] = b1 * m[e] + (1.f - b1) * gr;
      vv[e] = b2 * vv[e] + (1.f - b2) * gr * gr;
      const float dir = (m[e] / bc1) / (sqrtf(vv[e] / bc2) + eps);
      const float upd = -(lr * dir + wd * pp[e]);
      pp[e] += upd;
      us += upd * upd;
      ps += pp[e] * pp[e];
      if (MU_BF16) m[e] = round_bf16(m[e]);
    }
    reinterpret_cast<float4*>(p)[i] = make_float4(pp[0], pp[1], pp[2], pp[3]);
    reinterpret_cast<float4*>(nu)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    if (MU_BF16) {
      uint2 q; q.x = pack_bf16(m[0], m[1]); q.y = pack_bf16(m[2], m[3]);
      reinterpret_cast<uint2*>(mu)[i] = q;
    } else {
      reinterpret_cast<float4*>(mu)[i] = make_float4(m[0], m[1], m[2], m[3]);
    }
    if (p16 != nullptr) {
      uint2 q; q.x = pack_bf16(pp[0], pp[1]); q.y = pack_bf16(pp[2], pp[3]);
      reinterpret_cast<uint2*>(p16)[i] = q;
    }
  }
  float sums[2] = {us, ps};
  block_sum(sums, sh);
  if (threadIdx.x == 0) {
    if (upd_sq) atomicAdd(upd_sq, sums[0]);
    if (param_sq) atomicAdd(param_sq, sums[1]);
  }
}

// optax.scale(step_size) as the inner transform of the same chain (the reference's optimizer tests
// use it, optax_test.py:103-299; it is plain SGD): p += -(lr * g' + wd * p), g' = clipped gradient.
__global__ void __launch_bounds__(256)
scale_step_kernel(float* __restrict__ p, const float* __restrict__ g, bf16* __restrict__ p16, int64_t n,
                  float lr, float wd, const float* __restrict__ gnorm_sq, float clip_norm,
                  float grad_mult, float* __restrict__ upd_sq, float* __restrict__ param_sq) {
  __shared__ float sh[64];
  float gscale = grad_mult;
  if (clip_norm > 0.f && gnorm_sq != nullptr) {
    const float gn = sqrtf(gnorm_sq[0]) * grad_mult;
    if (!(gn < clip_norm)) gscale *= clip_norm / gn;
  }
  float us = 0.f, ps = 0.f;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float pp = p[i];
    const float upd = -(lr * (g[i] * gscale) + wd * pp);
    pp += upd;
    us += upd * upd;
    ps += pp * pp;
    p[i] = pp;
    if (p16 != nullptr) p16[i] = __float2bfloat16_rn(pp);
  }
  float sums[2] = {us, ps};
  block_sum(sums, sh);
  if (threadIdx.x == 0) {
    if (upd_sq) atomicAdd(upd_sq, sums[0]);
    if (param_sq) atomicAdd(param_sq, sums[1]);
  }
}

// 8 blocks per SM, the grid's cap, all resident at once: at most 32 registers
__global__ void __launch_bounds__(256, 8)
sumsq_kernel(const float* __restrict__ x, float* __restrict__ out, int64_t n) {
  __shared__ float sh[32];
  float a = 0.f;
  const int64_t n4 = n / 4;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    a += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const float v = x[n4 * 4 + threadIdx.x]; a += v * v; }
  a = block_sum(a, sh);
  if (threadIdx.x == 0) atomicAdd(out, a);
}

}  // namespace
}  // namespace bv

extern "C" {

int bv_adam_step(const bv_adam_args* args, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!args) { set_error("bv_adam_step: null args"); return BV_ERR_INVALID; }
  const bv_adam_args& a = *args;
  if (a.n <= 0) return BV_OK;
  if (a.n % 4 != 0 || (reinterpret_cast<uintptr_t>(a.params) & 15) ||
      (reinterpret_cast<uintptr_t>(a.grads) & 15)) {
    set_error("bv_adam_step: group size must be a multiple of 4 elements and 16B aligned");
    return BV_ERR_INVALID;
  }
  if (a.step < 1) { set_error("bv_adam_step: step is 1-based"); return BV_ERR_INVALID; }
  const float bc1 = 1.f - powf(a.b1, static_cast<float>(a.step));
  const float bc2 = 1.f - powf(a.b2, static_cast<float>(a.step));
  const unsigned blocks = grid_for(a.n / 4, 256, num_sms() * 8);
  if (a.mu_dtype == DT_BF16) {
    adam_kernel<true><<<blocks, 256, 0, s>>>(
        a.params, a.grads, a.mu, a.nu, reinterpret_cast<bf16*>(a.params_bf16), a.n, a.lr_eff, a.b1,
        a.b2, a.eps, a.wd_eff, bc1, bc2, a.gnorm_sq, a.clip_norm, a.grad_mult, a.upd_sq, a.param_sq);
  } else {
    adam_kernel<false><<<blocks, 256, 0, s>>>(
        a.params, a.grads, a.mu, a.nu, reinterpret_cast<bf16*>(a.params_bf16), a.n, a.lr_eff, a.b1,
        a.b2, a.eps, a.wd_eff, bc1, bc2, a.gnorm_sq, a.clip_norm, a.grad_mult, a.upd_sq, a.param_sq);
  }
  return check_cuda(cudaGetLastError(), "adam_kernel launch");
}

int bv_scale_step(float* params, const float* grads, void* params_bf16, int64_t n, float lr, float wd,
                  float grad_mult, float clip_norm, const float* gnorm_sq, float* upd_sq, float* param_sq,
                  void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return BV_OK;
  scale_step_kernel<<<grid_for(n, 256, num_sms() * 8), 256, 0, s>>>(
      params, grads, reinterpret_cast<bf16*>(params_bf16), n, lr, wd, gnorm_sq, clip_norm, grad_mult, upd_sq,
      param_sq);
  return check_cuda(cudaGetLastError(), "scale_step_kernel launch");
}

int bv_sumsq(const float* x, float* out, int64_t n, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return BV_OK;
  sumsq_kernel<<<grid_for(n / 4, 256, num_sms() * 8), 256, 0, s>>>(x, out, n);
  return check_cuda(cudaGetLastError(), "sumsq_kernel launch");
}

}  // extern "C"


// =====================================================================================================
// BV-Adafactor (big_vision/optax.py:187-214): optax.scale_by_factored_rms(factored=True, decay_rate=0.8,
// min_dim_size_to_factor=32, epsilon=1e-30, decay_rate_fn = min(beta2_cap, 1 - (t+1)^-0.8)) -> [clip_by_
// block_rms] -> optax.ema(momentum, debias=False, accumulator bf16), inside the same outer chain as Adam.
// optax (un-vendored dependency of the reference, requirements.txt:8) factors the second moment of a
// tensor with >= 2 dims whose second-largest dim is >= min_dim_size_to_factor over its two largest axes
// d0 (largest) and d1:   R0 = ema(mean_{d0}(g^2 + eps)),  R1 = ema(mean_{d1}(g^2 + eps)),
//                        u  = g * (R0 / mean_{d1}(R0))^-1/2 * R1^-1/2 ;
// everything else keeps a full second moment v = ema(g^2 + eps), u = g * v^-1/2.
// Every reference tensor on this path is a strided view [A, L, M, H] of the flat buffer (H contiguous,
// {d0, d1} = {L, H}): Dense [in, out] = [1, in, 1, out]; DenseGeneral q/k/v [d, h, dh] = [1, d, h, dh];
// out [h, dh, d] = [h, dh, 1, d]; scan-stacked tensors carry their depth in A.
// =====================================================================================================
namespace bv {
namespace {

struct View4 { int64_t A, L, M, H; int64_t sA, sL, sM; };   // element strides; H has stride 1

__device__ __forceinline__ float clip_scale(const float* gnorm_sq, float clip_norm, float grad_mult) {
  float gscale = grad_mult;
  if (clip_norm > 0.f && gnorm_sq != nullptr) {
    const float gn = sqrtf(gnorm_sq[0]) * grad_mult;
    if (!(gn < clip_norm)) gscale *= clip_norm / gn;
  }
  return gscale;
}

// out[a, l, m] = decay * out + (1 - decay) * mean_h((g * gs)^2 + eps): one warp per output
__global__ void __launch_bounds__(256)
af_reduce_h_kernel(const float* __restrict__ g, View4 v, float* __restrict__ out, float decay, float eps,
                   const float* __restrict__ gnorm_sq, float clip_norm, float grad_mult) {
  const float gs = clip_scale(gnorm_sq, clip_norm, grad_mult);
  const int lane = threadIdx.x & 31;
  const int64_t total = v.A * v.L * v.M;
  for (int64_t o = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5; o < total;
       o += (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5) {
    const int64_t m = o % v.M, l = (o / v.M) % v.L, a = o / (v.M * v.L);
    const float* row = g + a * v.sA + l * v.sL + m * v.sM;
    float acc = 0.f;
    for (int64_t h = lane; h < v.H; h += 32) { const float x = row[h] * gs; acc += x * x + eps; }
    acc = warp_sum(acc);
    if (lane == 0) out[o] = decay * out[o] + (1.f - decay) * (acc / static_cast<float>(v.H));
  }
}
// out[a, m, h] = decay * out + (1 - decay) * mean_l((g * gs)^2 + eps): one thread per output
__global__ void __launch_bounds__(256)
af_reduce_l_kernel(const float* __restrict__ g, View4 v, float* __restrict__ out, float decay, float eps,
                   const float* __restrict__ gnorm_sq, float clip_norm, float grad_mult) {
  const float gs = clip_scale(gnorm_sq, clip_norm, grad_mult);
  const int64_t total = v.A * v.M * v.H;
  for (int64_t o = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; o < total;
       o += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t h = o % v.H, m = (o / v.H) % v.M, a = o / (v.H * v.M);
    const float* col = g + a * v.sA + m * v.sM + h;
    float acc = 0.f;
    for (int64_t l = 0; l < v.L; ++l) { const float x = col[l * v.sL] * gs; acc += x * x + eps; }
    out[o] = decay * out[o] + (1.f - decay) * (acc / static_cast<float>(v.L));
  }
}
// out[o, i] = mean_r x[o, r, i]  (x contiguous [O, R, I]): the normaliser mean_{d1}(R0); tiny
__global__ void __launch_bounds__(256)
af_mean_kernel(const float* __restrict__ x, float* __restrict__ out, int64_t O, int64_t R, int64_t I) {
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < O * I;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = t % I, o = t / I;
    float acc = 0.f;
    for (int64_t r = 0; r < R; ++r) acc += x[(o * R + r) * I + i];
    out[t] = acc / static_cast<float>(R);
  }
}

// The update itself.  mode 0: unfactored (vfull updated here); mode 1: d0 = H (R0 = red_h [A,L,M],
// normaliser nrm [A,M], R1 = red_l [A,M,H]); mode 2: d0 = L (R0 = red_l [A,M,H], nrm [A,M], R1 = red_h).
template <bool MOM>
__global__ void __launch_bounds__(256)
af_apply_kernel(float* __restrict__ p, const float* __restrict__ g, bf16* __restrict__ p16, View4 v, int mode,
                float* __restrict__ vfull, const float* __restrict__ red_h, const float* __restrict__ red_l,
                const float* __restrict__ nrm, bf16* __restrict__ mom, float decay, float eps, float beta,
                float lr, float wd, const float* __restrict__ gnorm_sq, float clip_norm, float grad_mult,
                float* __restrict__ upd_sq, float* __restrict__ param_sq) {
  __shared__ float sh[64];
  const float gs = clip_scale(gnorm_sq, clip_norm, grad_mult);
  float us = 0.f, ps = 0.f;
  const int64_t total = v.A * v.L * v.M * v.H;
  for (int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t h = t % v.H, m = (t / v.H) % v.M, l = (t / (v.H * v.M)) % v.L, a = t / (v.H * v.M * v.L);
    const int64_t off = a * v.sA + l * v.sL + m * v.sM + h;
    const float gr = g[off] * gs;
    float u;
    if (mode == 0) {
      const float nv = decay * vfull[t] + (1.f - decay) * (gr * gr + eps);
      vfull[t] = nv;
      u = gr * rsqrtf(nv);
    } else {
      const float rh = red_h[(a * v.L + l) * v.M + m], rl = red_l[(a * v.M + m) * v.H + h];
      const float nm = nrm[a * v.M + m];
      u = (mode == 1) ? gr * rsqrtf(rh / nm) * rsqrtf(rl) : gr * rsqrtf(rl / nm) * rsqrtf(rh);
    }
    if (MOM) {
      const float mo = beta * __bfloat162float(mom[t]) + (1.f - beta) * u;   // optax.ema, debias=False
      mom[t] = __float2bfloat16_rn(mo);                                      // accumulator dtype bf16
      u = mo;
    }
    float pp = p[off];
    const float upd = -(lr * u + wd * pp);
    pp += upd;
    p[off] = pp;
    if (p16 != nullptr) p16[off] = __float2bfloat16_rn(pp);
    us += upd * upd;
    ps += pp * pp;
  }
  float sums[2] = {us, ps};
  block_sum(sums, sh);
  if (threadIdx.x == 0) {
    if (upd_sq) atomicAdd(upd_sq, sums[0]);
    if (param_sq) atomicAdd(param_sq, sums[1]);
  }
}

inline unsigned af_blocks(int64_t work) { return grid_for(work, 256, num_sms() * 8); }

}  // namespace
}  // namespace bv

extern "C" {

int bv_adafactor_step(const bv_adafactor_args* args, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!args) { set_error("bv_adafactor_step: null args"); return BV_ERR_INVALID; }
  const bv_adafactor_args& a = *args;
  View4 v{a.A, a.L, a.M, a.H, a.sA, a.sL, a.sM};
  if (a.A <= 0 || a.L <= 0 || a.M <= 0 || a.H <= 0 || a.mode < 0 || a.mode > 2) {
    set_error("bv_adafactor_step: bad view or mode");
    return BV_ERR_INVALID;
  }
  const int64_t n = a.A * a.L * a.M * a.H;
  if (a.mode != 0) {
    if (!a.red_h || !a.red_l || !a.nrm) { set_error("bv_adafactor_step: factored state missing"); return BV_ERR_INVALID; }
    af_reduce_h_kernel<<<af_blocks(a.A * a.L * a.M * 32), 256, 0, s>>>(a.grads, v, a.red_h, a.decay, a.eps, a.gnorm_sq,
                                                                     a.clip_norm, a.grad_mult);
    af_reduce_l_kernel<<<af_blocks(a.A * a.M * a.H), 256, 0, s>>>(a.grads, v, a.red_l, a.decay, a.eps, a.gnorm_sq,
                                                                a.clip_norm, a.grad_mult);
    // normaliser of R0 over the d1 axis: mode 1: R0 = red_h [A, L, M] -> mean over L; mode 2: R0 = red_l
    // [A, M, H] -> mean over H
    if (a.mode == 1) af_mean_kernel<<<af_blocks(a.A * a.M), 256, 0, s>>>(a.red_h, a.nrm, a.A, a.L, a.M);
    else af_mean_kernel<<<af_blocks(a.A * a.M), 256, 0, s>>>(a.red_l, a.nrm, a.A * a.M, a.H, 1);
  } else if (!a.vfull) {
    set_error("bv_adafactor_step: vfull missing");
    return BV_ERR_INVALID;
  }
  if (a.momentum != nullptr) {
    af_apply_kernel<true><<<af_blocks(n), 256, 0, s>>>(
        a.params, a.grads, reinterpret_cast<bf16*>(a.params_bf16), v, a.mode, a.vfull, a.red_h, a.red_l, a.nrm,
        reinterpret_cast<bf16*>(a.momentum), a.decay, a.eps, a.beta, a.lr_eff, a.wd_eff, a.gnorm_sq, a.clip_norm,
        a.grad_mult, a.upd_sq, a.param_sq);
  } else {
    af_apply_kernel<false><<<af_blocks(n), 256, 0, s>>>(
        a.params, a.grads, reinterpret_cast<bf16*>(a.params_bf16), v, a.mode, a.vfull, a.red_h, a.red_l, a.nrm,
        nullptr, a.decay, a.eps, a.beta, a.lr_eff, a.wd_eff, a.gnorm_sq, a.clip_norm, a.grad_mult, a.upd_sq,
        a.param_sq);
  }
  return check_cuda(cudaGetLastError(), "adafactor kernels launch");
}

}  // extern "C"
