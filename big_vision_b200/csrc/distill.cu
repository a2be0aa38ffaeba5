// Distillation kernels (include/bv_b200_distill.h; reference trainers/proj/distill/distill.py:217-248 and
// evaluators/proj/distill/distance.py:35-67).
//
// distill_loss_kernel turns the student's and one teacher's logits into the distance, its gradient and
// the step's measurements.  One CTA per row, two passes over the row:
//   pass 1  online (max, sum exp) of the student and the teacher, at temperature 1 and at t, and for
//           `hard` the teacher's first maximal index;
//   pass 2  the loss terms, the two entropies, the two task losses and the gradient.
// HBM traffic is one read of s, u (and labels) and one write of ds; the second read of a row follows
// the first from the same CTA and is meant to hit L2.  Rows wider than kWideRow run in CTAs of 1024
// threads: at the kernel's register count that is one row per SM in flight, so the rows between their
// two reads (132 * 3 * 4 C bytes, 35 MB at C = 21,843) fit the 50 MB L2, and 85 elements per thread
// become 21.
// Per-row results go to rows_ws and a fixed-order finishing pass averages them: no atomics, so the
// scalars are bit-identical from run to run.
#include "../../include/bv_b200_distill.h"

#include <limits.h>

#include "common.cuh"
#include "host_utils.h"

namespace bv {
namespace {

constexpr int kWideRow = 4096;
constexpr float kLogClip = -18.420680743952367f;   // log(1e-8): log(max(p, 1e-8)) = max(log p, log 1e-8)

// (max, sum exp(x - max), sum exp((x - max) / t)) of the elements seen so far
struct Soft { float m, z1, zt; };

template <bool T1, int V>
__device__ __forceinline__ void soft_add(Soft& a, const float (&x)[V], int cnt, float inv_t) {
  float vmax = x[0];
#pragma unroll
  for (int e = 1; e < V; ++e) if (e < cnt) vmax = fmaxf(vmax, x[e]);
  if (vmax > a.m) {
    const float d = a.m - vmax;             // -inf on the first chunk: exp gives 0 and z is 0
    a.z1 *= __expf(d);
    if (!T1) a.zt *= __expf(d * inv_t);
    a.m = vmax;
  }
#pragma unroll
  for (int e = 0; e < V; ++e) {
    if (e < cnt) {
      const float d = x[e] - a.m;
      a.z1 += __expf(d);
      if (!T1) a.zt += __expf(d * inv_t);
    }
  }
}

template <bool T1>
__device__ __forceinline__ Soft soft_merge(const Soft& a, const Soft& b, float inv_t) {
  Soft r;
  r.m = fmaxf(a.m, b.m);
  // a side that has seen nothing has m = -inf and z = 0; (a.m == r.m) keeps -inf - -inf out of exp
  const float da = a.m - r.m, db = b.m - r.m;
  const float sa = a.m == r.m ? 1.f : expf(da), sb = b.m == r.m ? 1.f : expf(db);
  r.z1 = a.z1 * sa + b.z1 * sb;
  r.zt = 0.f;
  if (!T1) r.zt = a.zt * (a.m == r.m ? 1.f : expf(da * inv_t)) + b.zt * (b.m == r.m ? 1.f : expf(db * inv_t));
  return r;
}

template <bool T1>
__device__ __forceinline__ Soft warp_soft(Soft a, float inv_t) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Soft b;
    b.m = __shfl_xor_sync(0xffffffffu, a.m, o);
    b.z1 = __shfl_xor_sync(0xffffffffu, a.z1, o);
    b.zt = __shfl_xor_sync(0xffffffffu, a.zt, o);
    a = soft_merge<T1>(a, b, inv_t);
  }
  return a;
}

// Block total of a Soft, the same bits in every thread: warp butterflies, then each warp re-reduces the
// warp totals.  sh: 3 * 32 floats.
template <bool T1>
__device__ __forceinline__ Soft block_soft(Soft a, float inv_t, float* sh) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  a = warp_soft<T1>(a, inv_t);
  if (lane == 0) { sh[warp] = a.m; sh[32 + warp] = a.z1; sh[64 + warp] = a.zt; }
  __syncthreads();
  Soft b = {-INFINITY, 0.f, 0.f};
  if (lane < nw) { b.m = sh[lane]; b.z1 = sh[32 + lane]; b.zt = sh[64 + lane]; }
  b = warp_soft<T1>(b, inv_t);
  __syncthreads();
  return b;
}

__device__ __forceinline__ float block_sum(float v, float* sh) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  v = warp_sum(v);
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  v = warp_sum(lane < nw ? sh[lane] : 0.f);
  __syncthreads();
  return v;
}

__device__ __forceinline__ int block_sum(int v, int* sh) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  v = lane < nw ? sh[lane] : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  return v;
}

// Block argmax with jnp.argmax's tie rule (the first maximal index), the same in every thread.
__device__ __forceinline__ int block_argmax(float best, int arg, float* shv, int* shi) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int round = 0; round < 2; ++round) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, arg, o);
      if (ov > best || (ov == best && oi < arg)) { best = ov; arg = oi; }
    }
    if (round == 0) {
      if (lane == 0) { shv[warp] = best; shi[warp] = arg; }
      __syncthreads();
      best = lane < nw ? shv[lane] : -INFINITY;
      arg = lane < nw ? shi[lane] : INT_MAX;
    }
  }
  __syncthreads();
  return arg;
}

// x[0 .. cnt) = p[c .. c + cnt): one 16-byte load for a whole chunk of 4
template <int V>
__device__ __forceinline__ void load_chunk(const float* __restrict__ p, int c, int cnt, float (&x)[V]) {
  if (V == 4 && cnt == 4) {
    const float4 v = *reinterpret_cast<const float4*>(p + c);
    x[0] = v.x; x[V > 1 ? 1 : 0] = v.y; x[V > 2 ? 2 : 0] = v.z; x[V > 3 ? 3 : 0] = v.w;
  } else {
#pragma unroll
    for (int e = 0; e < V; ++e) x[e] = e < cnt ? p[c + e] : 0.f;
  }
}

struct DistillArgs {
  const float* s; const float* u; const float* y;
  int64_t lds, ldu, ldy;
  float* d; int64_t ldd;
  float* rows;               // [BV_DISTILL_OUTPUTS, n], or [n] distances when !meas
  int64_t n; int C;
  float t, ls;
  int accumulate, meas;
};

// V: elements per load (4 needs 16-byte aligned rows).  T1: t == 1, the tempered sums are the plain
// ones.  HARD: the teacher's smoothed one-hot argmax instead of its tempered softmax (always with T1).
template <int V, bool T1, bool HARD>
__global__ void __launch_bounds__(1024, 1)
distill_loss_kernel(const DistillArgs a) {
  __shared__ float sh[96];
  __shared__ int shi[32];
  const int64_t row = blockIdx.x;
  const int C = a.C, tid = threadIdx.x, nthr = blockDim.x;
  const float* __restrict__ s = a.s + row * a.lds;
  const float* __restrict__ u = a.u + row * a.ldu;
  const float* __restrict__ y = a.y ? a.y + row * a.ldy : nullptr;
  const float inv_t = T1 ? 1.f : 1.f / a.t;
  const int chunks = (C + V - 1) / V;

  Soft ss = {-INFINITY, 0.f, 0.f}, su = {-INFINITY, 0.f, 0.f};
  float best = -INFINITY;
  int arg = INT_MAX;
  for (int ch = tid; ch < chunks; ch += nthr) {
    const int c = ch * V, cnt = min(V, C - c);
    float xs[V], xu[V];
    load_chunk<V>(s, c, cnt, xs);
    load_chunk<V>(u, c, cnt, xu);
    soft_add<T1, V>(ss, xs, cnt, inv_t);
    soft_add<T1, V>(su, xu, cnt, inv_t);
    if (HARD) {
#pragma unroll
      for (int e = 0; e < V; ++e) if (e < cnt && xu[e] > best) { best = xu[e]; arg = c + e; }
    }
  }
  ss = block_soft<T1>(ss, inv_t, sh);
  su = block_soft<T1>(su, inv_t, sh);
  if (HARD) arg = block_argmax(best, arg, sh, shi);

  const float lzs1 = logf(ss.z1), lzu1 = logf(su.z1);
  const float lzst = T1 ? lzs1 : logf(ss.zt), lzut = T1 ? lzu1 : logf(su.zt);
  // distance.py:45-47: the pseudo-label and its label smoothing
  const float on = HARD && a.ls != 0.f ? 1.f - a.ls : 1.f;
  const float off = HARD && a.ls != 0.f ? a.ls / static_cast<float>(C - 1) : 0.f;
  const float gscale = (HARD ? 1.f : a.t) / static_cast<float>(a.n);
  float* __restrict__ d = a.d ? a.d + row * a.ldd : nullptr;

  float dist = 0.f, ent_s = 0.f, ent_u = 0.f, task_s = 0.f, task_u = 0.f;
  for (int ch = tid; ch < chunks; ch += nthr) {
    const int c = ch * V, cnt = min(V, C - c);
    float xs[V], xu[V], yv[V], g[V];
    load_chunk<V>(s, c, cnt, xs);
    load_chunk<V>(u, c, cnt, xu);
    if (y) load_chunk<V>(y, c, cnt, yv);
#pragma unroll
    for (int e = 0; e < V; ++e) {
      g[e] = 0.f;
      if (e < cnt) {
        const float ds = xs[e] - ss.m, du = xu[e] - su.m;
        const float lq1 = ds - lzs1, lp1 = du - lzu1;            // log_softmax at temperature 1
        const float q1 = __expf(lq1), p1 = __expf(lp1);
        if (a.meas) {
          ent_s -= q1 * lq1;                                     // distill.py:232-233
          ent_u -= p1 * lp1;
          if (y) { task_s -= yv[e] * lq1; task_u -= yv[e] * lp1; }   // distill.py:235-236
        }
        if (HARD) {
          const float pl = (c + e == arg) ? on : off;
          dist -= pl * lq1;
          g[e] = (q1 - pl) * gscale;
        } else {
          const float lq = T1 ? lq1 : ds * inv_t - lzst, lp = T1 ? lp1 : du * inv_t - lzut;
          const float q = T1 ? q1 : __expf(lq), p = T1 ? p1 : __expf(lp);
          // utils.py:279-280: -p log_softmax(s / t) + p log(clip(p, 1e-8)), term by term so that equal
          // logits cancel exactly
          dist += p * (fmaxf(lp, kLogClip) - lq);
          g[e] = (q - p) * gscale;
        }
      }
    }
    if (d) {
      if (V == 4 && cnt == 4) {
        float4* dp = reinterpret_cast<float4*>(d + c);
        float4 o = make_float4(g[0], g[V > 1 ? 1 : 0], g[V > 2 ? 2 : 0], g[V > 3 ? 3 : 0]);
        if (a.accumulate) { const float4 old = *dp; o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w; }
        *dp = o;
      } else {
#pragma unroll
        for (int e = 0; e < V; ++e) if (e < cnt) d[c + e] = a.accumulate ? d[c + e] + g[e] : g[e];
      }
    }
  }
  if (d && !a.accumulate) {
    for (int64_t c = C + tid; c < a.ldd; c += nthr) d[c] = 0.f;
  }

  dist = block_sum(dist, sh);
  if (a.meas) {
    ent_s = block_sum(ent_s, sh); ent_u = block_sum(ent_u, sh);
    task_s = block_sum(task_s, sh); task_u = block_sum(task_u, sh);
  }
  if (tid == 0) {
    if (HARD) {
      // + sum pl log(clip(pl, 1e-8)): one class at `on`, C - 1 at `off`
      dist += on * fmaxf(logf(on), kLogClip);
      if (off != 0.f) dist += static_cast<float>(C - 1) * (off * fmaxf(logf(off), kLogClip));
    } else {
      dist *= a.t * a.t;
    }
    a.rows[BV_DISTILL_DISTANCE * a.n + row] = dist;
    if (a.meas) {
      a.rows[BV_DISTILL_ENTROPY_STUDENT * a.n + row] = ent_s;
      a.rows[BV_DISTILL_ENTROPY_TEACHER * a.n + row] = ent_u;
      a.rows[BV_DISTILL_TASK_STUDENT * a.n + row] = task_s;
      a.rows[BV_DISTILL_TASK_TEACHER * a.n + row] = task_u;
    }
  }
}

// out[k] = (1 / n) sum_i rows[k * n + i] for k = blockIdx.x: thread t sums t, t + 256, ... in index
// order, then a fixed shared-memory tree.
__global__ void __launch_bounds__(256)
distill_finish_kernel(const float* __restrict__ rows, int64_t n, float* __restrict__ out) {
  __shared__ float sh[256];
  const int k = blockIdx.x;
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += 256) acc += rows[k * n + i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (static_cast<int>(threadIdx.x) < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[k] = sh[0] / static_cast<float>(n);
}

// The kinds of dist() that are neither `kl` nor `hard`; one CTA of 256 threads per row.
__global__ void __launch_bounds__(256)
distance_kernel(const float* __restrict__ sp, int64_t lds, const float* __restrict__ up, int64_t ldu, int kind,
                float epsilon, int k, void* __restrict__ out, int C) {
  __shared__ float sh[96];
  __shared__ int shi[32];
  const int64_t row = blockIdx.x;
  const float* __restrict__ s = sp + row * lds;
  const float* __restrict__ u = up + row * ldu;
  const int tid = threadIdx.x;
  if (kind == BV_DIST_AGREE) {
    float best = -INFINITY;
    int arg = INT_MAX;
    for (int c = tid; c < C; c += 256) if (u[c] > best) { best = u[c]; arg = c; }
    arg = block_argmax(best, arg, sh, shi);
    const float sa = s[arg];
    int before = 0;        // classes that lax.top_k orders before `arg`: larger, or equal with a lower index
    for (int c = tid; c < C; c += 256) before += (s[c] > sa || (s[c] == sa && c < arg)) ? 1 : 0;
    before = block_sum(before, shi);
    if (tid == 0) reinterpret_cast<int32_t*>(out)[row] = before < k ? 1 : 0;
    return;
  }
  float acc = 0.f;
  if (kind == BV_DIST_LOGSOFTMAX_EUCLIDEAN) {
    Soft ss = {-INFINITY, 0.f, 0.f}, su = {-INFINITY, 0.f, 0.f};
    for (int c = tid; c < C; c += 256) {
      const float xs[1] = {s[c]}, xu[1] = {u[c]};
      soft_add<true, 1>(ss, xs, 1, 1.f);
      soft_add<true, 1>(su, xu, 1, 1.f);
    }
    ss = block_soft<true>(ss, 1.f, sh);
    su = block_soft<true>(su, 1.f, sh);
    const float ls = ss.m + logf(ss.z1), lu = su.m + logf(su.z1);
    for (int c = tid; c < C; c += 256) {
      const float df = (s[c] - ls) - (u[c] - lu);
      acc += df * df;
    }
  } else {
    for (int c = tid; c < C; c += 256) {
      const float df = s[c] - u[c];
      acc += df * df;
    }
  }
  acc = block_sum(acc, sh);
  if (tid == 0) reinterpret_cast<float*>(out)[row] = kind == BV_DIST_L2 ? acc : sqrtf(acc + epsilon);
}

inline bool vec_ok(const void* p, int64_t ld) {
  return p == nullptr || ((reinterpret_cast<uintptr_t>(p) & 15) == 0 && ld % 4 == 0);
}

int launch_rows(const DistillArgs& a, bool hard, cudaStream_t s) {
  const bool vec = vec_ok(a.s, a.lds) && vec_ok(a.u, a.ldu) && vec_ok(a.y, a.ldy) && vec_ok(a.d, a.ldd);
  const bool t1 = a.t == 1.f;
  const unsigned grid = static_cast<unsigned>(a.n), threads = a.C > kWideRow ? 1024 : 256;
  if (hard) {
    if (vec) distill_loss_kernel<4, true, true><<<grid, threads, 0, s>>>(a);
    else distill_loss_kernel<1, true, true><<<grid, threads, 0, s>>>(a);
  } else if (t1) {
    if (vec) distill_loss_kernel<4, true, false><<<grid, threads, 0, s>>>(a);
    else distill_loss_kernel<1, true, false><<<grid, threads, 0, s>>>(a);
  } else {
    if (vec) distill_loss_kernel<4, false, false><<<grid, threads, 0, s>>>(a);
    else distill_loss_kernel<1, false, false><<<grid, threads, 0, s>>>(a);
  }
  return check_cuda(cudaGetLastError(), "distill_loss_kernel launch");
}

// Argument checks shared by the two entry points.  > 0: nothing to do.
int check_rows(const char* fn, const void* student, int64_t lds, const void* teacher, int64_t ldu, int kind, float t,
               float ls, int64_t n, int C) {
  if (n < 0 || n > INT_MAX || C < 1 || lds < C || ldu < C) {
    set_error("%s: need 0 <= n < 2^31, C >= 1 and row strides >= C (n %lld, C %d, ld_student %lld, ld_teacher %lld)",
              fn, static_cast<long long>(n), C, static_cast<long long>(lds), static_cast<long long>(ldu));
    return BV_ERR_INVALID;
  }
  if (n > 0 && (!student || !teacher)) { set_error("%s: null logits", fn); return BV_ERR_INVALID; }
  if (kind == BV_DIST_KL && !(t > 0.f)) { set_error("%s: kl needs a temperature t > 0", fn); return BV_ERR_INVALID; }
  if (kind == BV_DIST_HARD && (ls < 0.f || ls > 1.f || (ls != 0.f && C < 2))) {
    set_error("%s: hard needs 0 <= ls <= 1, and C >= 2 to smooth over the other classes", fn);
    return BV_ERR_INVALID;
  }
  return n == 0 ? 1 : BV_OK;
}

}  // namespace
}  // namespace bv

extern "C" {

int bv_distill_loss(const float* student, int64_t ld_student, const float* teacher, int64_t ld_teacher,
                    const float* labels, int64_t ld_labels, int32_t kind, float t, float ls, int32_t accumulate,
                    float* dlogits, int64_t ld_dlogits, float* out, float* rows_ws, int64_t n, int32_t C,
                    void* stream) {
  using namespace bv;
  if (kind != BV_DIST_KL && kind != BV_DIST_HARD) {
    set_error("bv_distill_loss: kind %d has no training kernel (built: kl, hard)", kind);
    return BV_ERR_UNSUPPORTED;
  }
  const int rc = check_rows("bv_distill_loss", student, ld_student, teacher, ld_teacher, kind, t, ls, n, C);
  if (rc < 0) return rc;
  if ((labels && ld_labels < C) || (dlogits && ld_dlogits < C)) {
    set_error("bv_distill_loss: row strides must be >= C (ld_labels %lld, ld_dlogits %lld, C %d)",
              static_cast<long long>(ld_labels), static_cast<long long>(ld_dlogits), C);
    return BV_ERR_INVALID;
  }
  if (!out || !rows_ws) { set_error("bv_distill_loss: null out or rows_ws"); return BV_ERR_INVALID; }
  if (rc > 0) return BV_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const DistillArgs a = {student, teacher, labels, ld_student, ld_teacher, ld_labels, dlogits, ld_dlogits, rows_ws,
                         n, C, kind == BV_DIST_HARD ? 1.f : t, ls, accumulate, 1};
  const int lrc = launch_rows(a, kind == BV_DIST_HARD, s);
  if (lrc) return lrc;
  distill_finish_kernel<<<BV_DISTILL_OUTPUTS, 256, 0, s>>>(rows_ws, n, out);
  return check_cuda(cudaGetLastError(), "distill_finish_kernel launch");
}

int bv_distance(const float* student, int64_t ld_student, const float* teacher, int64_t ld_teacher, int32_t kind,
                float epsilon, float t, float ls, int32_t k, void* out, int64_t n, int32_t C, void* stream) {
  using namespace bv;
  if (kind < BV_DIST_EUCLIDEAN || kind > BV_DIST_AGREE) {
    set_error("bv_distance: unknown kind of distance %d", kind);
    return BV_ERR_INVALID;
  }
  const int rc = check_rows("bv_distance", student, ld_student, teacher, ld_teacher, kind, t, ls, n, C);
  if (rc < 0) return rc;
  if (!out) { set_error("bv_distance: null out"); return BV_ERR_INVALID; }
  if (kind == BV_DIST_AGREE && k < 1) { set_error("bv_distance: agree needs k >= 1"); return BV_ERR_INVALID; }
  if (rc > 0) return BV_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (kind == BV_DIST_KL || kind == BV_DIST_HARD) {
    const DistillArgs a = {student, teacher, nullptr, ld_student, ld_teacher, 0, nullptr, 0,
                           static_cast<float*>(out), n, C, kind == BV_DIST_HARD ? 1.f : t, ls, 0, 0};
    return launch_rows(a, kind == BV_DIST_HARD, s);
  }
  distance_kernel<<<static_cast<unsigned>(n), 256, 0, s>>>(student, ld_student, teacher, ld_teacher, kind, epsilon, k,
                                                          out, C);
  return check_cuda(cudaGetLastError(), "distance_kernel launch");
}

}  // extern "C"
