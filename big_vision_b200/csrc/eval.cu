// Integer evaluation paths (SURVEY 8f rank 2): exact index arithmetic, HBM-bound single passes.
//  * top-1: evaluators/classification.py:46-52 -- top1_idx = argmax(logits, axis=1);
//    top1_correct = take_along_axis(labels, top1_idx); mask *= labels.max(axis=1);
//    ncorrect = sum(top1_correct * mask); nseen = sum(mask).  Also the zero-shot classifier's
//    best_txt = (zimg @ ztxt.T).argmax(axis=1)
//    (evaluators/proj/image_text/discriminative_classifier.py:284-288) on the GEMM's output.
//    argmax returns the FIRST maximal index and treats NaN as maximal, as jnp.argmax does.
//  * retrieval: evaluators/proj/image_text/image_text_retrieval.py:23-85.  The reference sorts
//    (argsort) and tests membership in the first k entries; here the position of the positive in
//    that order is COUNTED instead -- rank = #{entries that sort before it} -- which gives the
//    same integers without a sort.  Ties sort by index (a stable argsort).
#include "common.cuh"
#include "host_utils.h"

#include <limits.h>

namespace bv {
namespace {

// (value, index) ordering of argmax: NaN beats everything, then larger value, then lower index
__device__ __forceinline__ bool argmax_better(float v, int c, float bv, int bc) {
  const bool vn = v != v, bn = bv != bv;
  if (vn != bn) return vn;
  if (!vn && v != bv) return v > bv;
  return c < bc;
}

__device__ __forceinline__ float load_logit(const void* p, int dtype, int64_t off) {
  if (dtype == DT_BF16) return __bfloat162float(reinterpret_cast<const bf16*>(p)[off]);
  return reinterpret_cast<const float*>(p)[off];
}

// one warp per row
__global__ void __launch_bounds__(256)
top1_kernel(const void* __restrict__ logits, int dtype, int64_t rows, int C, int64_t ld,
            int32_t* __restrict__ idx_out, const float* __restrict__ labels, int64_t ldl,
            const float* __restrict__ mask, float* __restrict__ top1_correct,
            float* __restrict__ sums) {
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  float best = -INFINITY;
  int bidx = INT_MAX;
  for (int c = lane; c < C; c += 32) {
    const float v = load_logit(logits, dtype, row * ld + c);
    if (bidx == INT_MAX || argmax_better(v, c, best, bidx)) { best = v; bidx = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oc = __shfl_xor_sync(0xffffffffu, bidx, o);
    if (oc != INT_MAX && (bidx == INT_MAX || argmax_better(ov, oc, best, bidx))) { best = ov; bidx = oc; }
  }
  if (lane == 0 && idx_out != nullptr) idx_out[row] = bidx;
  if (labels == nullptr) return;
  // mask *= labels.max(axis=1): rows whose labels are all zero do not count
  float lmax = -INFINITY;
  for (int c = lane; c < C; c += 32) lmax = fmaxf(lmax, labels[row * ldl + c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  if (lane == 0) {
    const float m = (mask != nullptr ? mask[row] : 1.0f) * lmax;
    const float hit = labels[row * ldl + bidx];
    if (top1_correct != nullptr) top1_correct[row] = hit;
    if (sums != nullptr) {
      atomicAdd(sums + 0, hit * m);     // ncorrect
      atomicAdd(sums + 1, m);           // nseen
    }
  }
}

// text -> image: for text column j with positive image p = corr[j],
//   rank[j] = #{ i : d[i,j] < d[p,j]  or  (d[i,j] == d[p,j] and i < p) }
// A block owns 32 consecutive columns (lane = column, so every row read is one coalesced 128 B
// line) and its 8 warps split the rows.
__global__ void __launch_bounds__(256)
rank_t2i_kernel(const float* __restrict__ d, int64_t NI, int64_t NT, int64_t ld,
                const int32_t* __restrict__ corr, int32_t* __restrict__ rank) {
  __shared__ int cnt[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t j = static_cast<int64_t>(blockIdx.x) * 32 + lane;
  if (threadIdx.x < 32) cnt[threadIdx.x] = 0;
  __syncthreads();
  int c = 0;
  bool ok = false;
  if (j < NT) {
    const int64_t p = corr[j];
    ok = p >= 0 && p < NI;
    if (ok) {
      const float dp = d[p * ld + j];
      for (int64_t i = warp; i < NI; i += 8) {
        const float v = d[i * ld + j];
        c += (v < dp || (v == dp && i < p)) ? 1 : 0;
      }
    }
  }
  atomicAdd(&cnt[lane], c);
  __syncthreads();
  if (warp == 0 && j < NT) rank[j] = ok ? cnt[lane] : INT_MAX;
}

// image -> text: for image row i the best positive is the (distance, index)-smallest text j with
// corr[j] == i; rank[i] = #{ j' : d[i,j'] sorts before it }.  INT_MAX when the row has no text.
__global__ void __launch_bounds__(256)
rank_i2t_kernel(const float* __restrict__ d, int64_t NI, int64_t NT, int64_t ld,
                const int32_t* __restrict__ corr, int32_t* __restrict__ rank) {
  __shared__ float s_val[8];
  __shared__ long long s_idx[8];
  __shared__ int s_cnt;
  const int64_t i = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* row = d + i * ld;
  float bv = INFINITY;
  long long bj = -1;
  for (int64_t j = threadIdx.x; j < NT; j += blockDim.x) {
    if (corr[j] == i) {
      const float v = row[j];
      if (bj < 0 || v < bv || (v == bv && j < bj) || (bv != bv && v == v)) { bv = v; bj = j; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const long long oj = __shfl_xor_sync(0xffffffffu, bj, o);
    if (oj >= 0 && (bj < 0 || ov < bv || (ov == bv && oj < bj) || (bv != bv && ov == ov))) { bv = ov; bj = oj; }
  }
  if (lane == 0) { s_val[warp] = bv; s_idx[warp] = bj; }
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  bv = s_val[0]; bj = s_idx[0];
  for (int w = 1; w < 8; ++w) {
    const float ov = s_val[w];
    const long long oj = s_idx[w];
    if (oj >= 0 && (bj < 0 || ov < bv || (ov == bv && oj < bj) || (bv != bv && ov == ov))) { bv = ov; bj = oj; }
  }
  if (bj < 0) {
    if (threadIdx.x == 0) rank[i] = INT_MAX;
    return;
  }
  int c = 0;
  for (int64_t j = threadIdx.x; j < NT; j += blockDim.x) {
    const float v = row[j];
    c += (v < bv || (v == bv && j < bj)) ? 1 : 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) atomicAdd(&s_cnt, c);
  __syncthreads();
  if (threadIdx.x == 0) rank[i] = s_cnt;
}

}  // namespace
}  // namespace bv

extern "C" {

int bv_top1(const void* logits, int dtype, int64_t rows, int32_t C, int64_t ld, int32_t* idx,
            const float* labels, int64_t ldl, const float* mask, float* top1_correct, float* sums,
            void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows < 0 || C <= 0 || ld < C || (labels != nullptr && ldl < C)) {
    set_error("bv_top1: need rows >= 0, C >= 1 and row strides >= C");
    return BV_ERR_INVALID;
  }
  if (dtype != DT_F32 && dtype != DT_BF16) { set_error("bv_top1: bad dtype"); return BV_ERR_INVALID; }
  if (rows == 0) return BV_OK;
  const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
  top1_kernel<<<grid, 256, 0, s>>>(logits, dtype, rows, C, ld, idx, labels, ldl, mask, top1_correct, sums);
  return check_cuda(cudaGetLastError(), "top1_kernel launch");
}

int bv_retrieval_ranks(const float* dist, int64_t NI, int64_t NT, int64_t ld, const int32_t* corr,
                       int32_t* rank_t2i, int32_t* rank_i2t, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (NI <= 0 || NT <= 0 || ld < NT) {
    set_error("bv_retrieval_ranks: need NI, NT >= 1 and ld >= NT");
    return BV_ERR_INVALID;
  }
  if (rank_t2i != nullptr) {
    rank_t2i_kernel<<<static_cast<unsigned>((NT + 31) / 32), 256, 0, s>>>(dist, NI, NT, ld, corr, rank_t2i);
    int rc = check_cuda(cudaGetLastError(), "rank_t2i_kernel launch");
    if (rc) return rc;
  }
  if (rank_i2t != nullptr) {
    rank_i2t_kernel<<<static_cast<unsigned>(NI), 256, 0, s>>>(dist, NI, NT, ld, corr, rank_i2t);
    return check_cuda(cudaGetLastError(), "rank_i2t_kernel launch");
  }
  return BV_OK;
}

}  // extern "C"
