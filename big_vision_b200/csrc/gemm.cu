// Warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] = epilogue( alpha * sum_k A(m,k) * B(n,k) )
//
// A and B are bf16 and each may be stored K-major (rows = M/N, K contiguous) or
// MN-major (rows = K, M/N contiguous); both go HBM -> smem by TMA (128B swizzle)
// and smem -> tensor core by wgmma descriptors (the transpose bits select the
// major-ness), accumulating fp32 in registers.  This one kernel serves every dense
// contraction of the hot path:
//   forward  Y  = X  W      A = X  (K-major),  B = W  [K,N] (MN-major)    K1,K4,K6,K7,K8,K11
//   dgrad    dX = dY W^T    A = dY (K-major),  B = W  [K,N] (K-major)
//   wgrad    dW = X^T dY    A = X  (MN-major), B = dY (MN-major), split-K, fp32 reduce-add
// (reference call sites: flax Dense/DenseGeneral under models/vit.py:72-77,93-98,
//  176-178,212-214,261,272; models/mlp_mixer.py:35-37,72,82).
//
// One CTA owns one 128 x BN output tile (x one K split).  Roles (384 threads): warpgroup 0 is the
// TMA producer (one thread issues, the rest give their registers back with setmaxnreg), warpgroups
// 1 and 2 each run m64 x BN x 16 wgmma on their half of the rows from a STAGES-deep ring of shared
// memory, then apply the epilogue straight from the accumulator registers.
#include "common.cuh"
#include "host_utils.h"
#include "kernels.h"

#include <atomic>

#include <stdlib.h>

namespace bv {

namespace {

constexpr int BM = 128;          // rows per CTA (two consumer warpgroups of 64)
constexpr int BK = 64;           // 64 bf16 = 128 B = one swizzle row
constexpr int A_STAGE_BYTES = BM * BK * 2;   // 16 KB
constexpr int NUM_THREADS = 384;

// epilogue families (template parameter)
enum : int { EF_BIAS = 0, EF_GELU = 1, EF_RESID = 2, EF_DGELU = 3 };

template <int BN>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int SMEM_LIMIT = 232448 - 2048;         // 227 KB minus barriers / align slack
  static constexpr int STAGES_FIT = SMEM_LIMIT / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 8 ? 8 : STAGES_FIT;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFFSET + 256 + 1024;  // + barriers + align slack
};

struct GemmDev {
  int M, N, K;
  int kblocks_total, kblocks_per_split;
  int a_mn, b_mn;        // 1 = MN-major
  int reduce_out;        // 1 = atomic add into D (split-K / grad accumulation)
  float alpha;
  const float* bias;
  const bf16* aux;
  void* d; void* d2;
  long long ldd, ldd2, ldaux;
  float* colsum;         // optional bias-gradient accumulator (bf16 outputs only)
  int aux_row_mod;
};

// The consumer warpgroup's main loop.  The transpose bits of wgmma are immediates, so each operand
// layout pair is its own instantiation (a branch between wgmma issues would make ptxas serialise them).
template <int BN, int STAGES, int STAGE_BYTES, int TA, int TB>
__device__ __forceinline__ void mainloop(float (&acc)[BN / 2], uint32_t base, uint32_t bar_base, int cw, int kb0,
                                         int kb1) {
  // 128B-swizzled operand tiles: K-major rows of 128 B (8-row groups 1024 B apart, K step 32 B);
  // MN-major boxes of 64 (M|N) x 64 (K), 8 KB each (K step 16 rows = 2048 B)
  constexpr uint32_t a_lbo = TA ? 8192u : 16u, b_lbo = TB ? 8192u : 16u;
  constexpr uint32_t a_kstep = TA ? 2048u : 32u, b_kstep = TB ? 2048u : 32u;
  int stage = 0;
  uint32_t phase = 0;
  int prev_stage = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(bar_base + 8u * stage, phase);
    const uint32_t a_s = base + stage * STAGE_BYTES + cw * 8192;
    const uint32_t b_s = base + stage * STAGE_BYTES + A_STAGE_BYTES;
    const uint64_t adesc = wgmma_desc_sw128(a_s, a_lbo, 1024u), bdesc = wgmma_desc_sw128(b_s, b_lbo, 1024u);
    wgmma_fence_regs(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t a = adesc + k * (a_kstep >> 4), b = bdesc + k * (b_kstep >> 4);
      const int accumulate = (kb > kb0 || k > 0) ? 1 : 0;    // the first MMA overwrites the registers
      if constexpr (BN == 256) wgmma_ss_n256<TA, TB>(acc, a, b, accumulate);
      else wgmma_ss_n128<TA, TB>(acc, a, b, accumulate);
    }
    wgmma_commit();
    wgmma_fence_regs(acc);
    // keep this k block's MMAs in flight; the previous one has retired -> its slot is free
    wgmma_wait<1>();
    if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_base + 8u * (STAGES + prev_stage));
    prev_stage = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_base + 8u * (STAGES + prev_stage));
}

template <int BN, bool OUT_F32, int EF>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmDev p) {
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;
  const uint32_t bar_base = base + C::BAR_OFFSET;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };

  const int wg = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);
  const int n0 = static_cast<int>(blockIdx.x) * BN;
  const int m0 = static_cast<int>(blockIdx.y) * BM;
  const int kb0 = static_cast<int>(blockIdx.z) * p.kblocks_per_split;
  const int kb1 = min(kb0 + p.kblocks_per_split, p.kblocks_total);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);     // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ========================= TMA producer =========================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(empty_bar(stage), phase ^ 1u);
        const uint32_t a_s = base + stage * C::STAGE_BYTES;
        const uint32_t b_s = a_s + A_STAGE_BYTES;
        const uint32_t fb = full_bar(stage);
        mbar_expect_tx(fb, C::STAGE_BYTES);
        const int k0 = kb * BK;
        if (p.a_mn) {
#pragma unroll
          for (int j = 0; j < BM / 64; ++j) tma_load_2d(a_s + j * 8192, &tmA, fb, m0 + 64 * j, k0);
        } else {
          tma_load_2d(a_s, &tmA, fb, k0, m0);
        }
        if (p.b_mn) {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(b_s + j * 8192, &tmB, fb, n0 + 64 * j, k0);
        } else {
          tma_load_2d(b_s, &tmB, fb, k0, n0);
        }
        if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ========================= consumers: warpgroups 1, 2 =========================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = wg - 1;                        // which 64-row half of the tile
  float acc[BN / 2];
  constexpr int S = C::STAGES, SB = C::STAGE_BYTES;
  if (p.a_mn) {
    if (p.b_mn) mainloop<BN, S, SB, 1, 1>(acc, base, bar_base, cw, kb0, kb1);
    else mainloop<BN, S, SB, 1, 0>(acc, base, bar_base, cw, kb0, kb1);
  } else {
    if (p.b_mn) mainloop<BN, S, SB, 0, 1>(acc, base, bar_base, cw, kb0, kb1);
    else mainloop<BN, S, SB, 0, 0>(acc, base, bar_base, cw, kb0, kb1);
  }

  // ========================= epilogue from registers =========================
  // Accumulator layout (per warp w of the warpgroup, lane l): element 4j + e sits at row
  // 16w + l/4 + 8*(e >> 1), column 8j + 2*(l%4) + (e & 1).
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int row0 = m0 + cw * 64 + warp * 16 + (lane >> 2);
  const int pM = p.M, pN = p.N;
  const float alpha = p.alpha;
  const bool reduce = p.reduce_out != 0;
  constexpr bool HAS_AUX = (EF == EF_RESID || EF == EF_DGELU);
  float cs[BN / 8][2];
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * (lane & 3);
    cs[j][0] = cs[j][1] = 0.f;
    if (col >= pN) continue;
    const bool pair = col + 1 < pN;
    float b0 = 0.f, b1 = 0.f;
    if (p.bias != nullptr) {
      b0 = __ldg(p.bias + col);
      if (pair) b1 = __ldg(p.bias + col + 1);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      if (row >= pM) continue;
      float v0 = acc[4 * j + 2 * h] * alpha + b0, v1 = acc[4 * j + 2 * h + 1] * alpha + b1;
      float a0 = 0.f, a1 = 0.f;
      if (HAS_AUX) {
        const long long ar = p.aux_row_mod > 0 ? (row % p.aux_row_mod) : row;
        const bf16* ap = p.aux + ar * p.ldaux + col;
        if (pair) {
          const uint32_t q = *reinterpret_cast<const uint32_t*>(ap);
          a0 = bf16_lo(q); a1 = bf16_hi(q);
        } else {
          a0 = __bfloat162float(*ap);
        }
      }
      float pre0 = 0.f, pre1 = 0.f;
      if (EF == EF_GELU) {
        pre0 = round_bf16(v0); pre1 = round_bf16(v1);
        v0 = gelu_tanh_fast(pre0); v1 = gelu_tanh_fast(pre1);
      } else if (EF == EF_RESID) {
        v0 = (OUT_F32 ? v0 : round_bf16(v0)) + a0;
        v1 = (OUT_F32 ? v1 : round_bf16(v1)) + a1;
      } else if (EF == EF_DGELU) {
        v0 *= gelu_tanh_grad_fast(a0);
        v1 *= gelu_tanh_grad_fast(a1);
      }
      if (OUT_F32) {
        float* dp = static_cast<float*>(p.d) + row * p.ldd + col;
        if (reduce) {
          atomicAdd(dp, v0);
          if (pair) atomicAdd(dp + 1, v1);
        } else if (pair) {
          *reinterpret_cast<float2*>(dp) = make_float2(v0, v1);
        } else {
          *dp = v0;
        }
      } else {
        bf16* dp = static_cast<bf16*>(p.d) + row * p.ldd + col;
        const __nv_bfloat162 o = __floats2bfloat162_rn(v0, v1);
        if (reduce) {
          if (pair) atomicAdd(reinterpret_cast<__nv_bfloat162*>(dp), o);
          else atomicAdd(dp, o.x);
        } else if (pair) {
          *reinterpret_cast<__nv_bfloat162*>(dp) = o;
        } else {
          *dp = o.x;
        }
        cs[j][0] += __low2float(o);
        cs[j][1] += pair ? __high2float(o) : 0.f;
        if (EF == EF_GELU) {
          bf16* d2 = static_cast<bf16*>(p.d2) + row * p.ldd2 + col;
          const __nv_bfloat162 q = __floats2bfloat162_rn(pre0, pre1);
          if (pair) *reinterpret_cast<__nv_bfloat162*>(d2) = q;
          else *d2 = q.x;
        }
      }
    }
  }
  if (!OUT_F32 && p.colsum != nullptr) {
    // bias gradient fused into the producer: column sums of the stored (bf16-rounded) values; the
    // eight lanes that share a column pair are summed with shuffles, then one atomic per warp
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float s = cs[j][e];
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        s += __shfl_xor_sync(0xffffffffu, s, 8);
        s += __shfl_xor_sync(0xffffffffu, s, 16);
        cs[j][e] = s;
      }
      const int col = n0 + 8 * j + 2 * (lane & 3);
      if (lane < 4) {
        if (col < pN) atomicAdd(p.colsum + col, cs[j][0]);
        if (col + 1 < pN) atomicAdd(p.colsum + col + 1, cs[j][1]);
      }
    }
  }
}

template <int BN, bool OUT_F32, int EF>
int launch_cfg(const GemmArgs& g, cudaStream_t stream) {
  using C = Cfg<BN>;
  CUtensorMap tmA, tmB;
  int rc;
  const CUtensorMapDataType bf = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if (g.a_mn) rc = make_tmap_2d(&tmA, bf, g.A, g.M, g.K, g.lda * 2, 64, 64);
  else        rc = make_tmap_2d(&tmA, bf, g.A, g.K, g.M, g.lda * 2, 64, BM);
  if (rc) return rc;
  if (g.b_mn) rc = make_tmap_2d(&tmB, bf, g.B, g.N, g.K, g.ldb * 2, 64, 64);
  else        rc = make_tmap_2d(&tmB, bf, g.B, g.K, g.N, g.ldb * 2, 64, BN);
  if (rc) return rc;

  GemmDev p;
  p.M = (int)g.M; p.N = (int)g.N; p.K = (int)g.K;
  const int num_m = (int)((g.M + BM - 1) / BM);
  const int num_n = (int)((g.N + BN - 1) / BN);
  p.kblocks_total = (int)((g.K + BK - 1) / BK);
  int splits = g.splits;
  if (splits <= 0) {
    // auto (reduce-add outputs only, i.e. the weight gradients): the split count whose work units fill
    // whole waves of the grid best (one CTA per SM).  Each extra split costs one more fp32 reduce-add
    // of the output tile, negligible against a K of 10^5.
    splits = 1;
    if (g.reduce_out) {
      const int slots = num_sms();
      const int tiles = num_m * num_n;
      int smax = p.kblocks_total / 16;
      if (smax > 32) smax = 32;
      double best = -1.0;
      for (int sp = 1; sp <= smax; ++sp) {
        const int units = tiles * sp;
        const int waves = (units + slots - 1) / slots;
        const double eff = static_cast<double>(units) / (static_cast<double>(waves) * slots) - 0.002 * sp;
        if (eff > best + 1e-9) { best = eff; splits = sp; }
      }
    }
  }
  if (splits > p.kblocks_total) splits = p.kblocks_total;
  if (splits < 1) splits = 1;
  if (splits > 1 && !g.reduce_out) {
    set_error("bv_gemm: split-K requires reduce_out=1");
    return BV_ERR_INVALID;
  }
  p.kblocks_per_split = (p.kblocks_total + splits - 1) / splits;
  splits = (p.kblocks_total + p.kblocks_per_split - 1) / p.kblocks_per_split;
  if (splits > 65535 || num_m > 65535) { set_error("bv_gemm: grid too large"); return BV_ERR_INVALID; }
  p.a_mn = g.a_mn; p.b_mn = g.b_mn; p.reduce_out = g.reduce_out;
  p.alpha = g.alpha;
  p.bias = g.bias;
  p.colsum = g.colsum;
  p.aux = reinterpret_cast<const bf16*>(g.aux);
  p.ldaux = g.ldaux;
  p.aux_row_mod = g.aux_row_mod;
  p.d = g.D; p.d2 = g.D2;
  p.ldd = g.ldd; p.ldd2 = g.ldd2;

  auto kern = gemm_kernel<BN, OUT_F32, EF>;
  // The dynamic-shared-memory opt-in is a per-DEVICE attribute of the kernel: cache it per device
  // (one process may drive several GPUs from several host threads; the flags are atomics and a
  // duplicate set by two racing threads is harmless).
  static std::atomic<bool> attr_set[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = -1;
  if (dev < 0 || !attr_set[dev].load(std::memory_order_acquire)) {
    rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES),
                    "cudaFuncSetAttribute(gemm)");
    if (rc) return rc;
    if (dev >= 0) attr_set[dev].store(true, std::memory_order_release);
  }
  kern<<<dim3(num_n, num_m, splits), NUM_THREADS, C::SMEM_BYTES, stream>>>(tmA, tmB, p);
  return check_cuda(cudaGetLastError(), "gemm_kernel launch");
}

template <int BN>
int dispatch_epi(const GemmArgs& g, cudaStream_t s) {
  const bool f32 = (g.out_dtype == DT_F32);
  switch (g.epi) {
    case EPI_NONE:
    case EPI_BIAS:
      return f32 ? launch_cfg<BN, true, EF_BIAS>(g, s) : launch_cfg<BN, false, EF_BIAS>(g, s);
    case EPI_BIAS_RESID:
      return f32 ? launch_cfg<BN, true, EF_RESID>(g, s) : launch_cfg<BN, false, EF_RESID>(g, s);
    case EPI_BIAS_GELU:
      return launch_cfg<BN, false, EF_GELU>(g, s);
    case EPI_DGELU:
      if (f32) { set_error("bv_gemm: DGELU epilogue writes bf16"); return BV_ERR_INVALID; }
      if (g.aux_row_mod > 0) { set_error("bv_gemm: DGELU takes a row-aligned aux"); return BV_ERR_INVALID; }
      return launch_cfg<BN, false, EF_DGELU>(g, s);
  }
  set_error("bv_gemm: bad epilogue %d", g.epi);
  return BV_ERR_INVALID;
}

}  // namespace

int launch_gemm(const GemmArgs& g, cudaStream_t stream) {
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) { set_error("bv_gemm: empty problem"); return BV_ERR_INVALID; }
  // N need not be a multiple of 8 as long as the row strides are (TMA clips the loads)
  // the epilogue stores bf16 pairs / fp32 pairs straight from registers
  if (g.out_dtype == DT_BF16 && ((reinterpret_cast<uintptr_t>(g.D) & 15) || (g.ldd % 8))) {
    set_error("bv_gemm: bf16 output must be 16B aligned with ldd %% 8 == 0"); return BV_ERR_INVALID;
  }
  if (g.out_dtype == DT_F32 && ((reinterpret_cast<uintptr_t>(g.D) & 7) || (g.ldd % 2))) {
    set_error("bv_gemm: fp32 output must be 8B aligned with an even ldd"); return BV_ERR_INVALID;
  }
  if (g.M > 0x7fffffffLL || g.N > 0x7fffffffLL || g.K > 0x7fffffffLL) {
    set_error("bv_gemm: dimension exceeds int32"); return BV_ERR_INVALID;
  }
  if (g.epi < EPI_NONE || g.epi > EPI_DGELU) { set_error("bv_gemm: bad epilogue %d", g.epi); return BV_ERR_INVALID; }
  if ((g.epi == EPI_BIAS_RESID || g.epi == EPI_DGELU) && g.aux == nullptr) {
    set_error("bv_gemm: epilogue %d needs aux", g.epi); return BV_ERR_INVALID;
  }
  if (g.aux != nullptr && ((reinterpret_cast<uintptr_t>(g.aux) & 15) || (g.ldaux % 8))) {
    set_error("bv_gemm: aux must be 16B aligned with ldaux %% 8 == 0"); return BV_ERR_INVALID;
  }
  if (g.bias != nullptr && (reinterpret_cast<uintptr_t>(g.bias) & 15)) {
    set_error("bv_gemm: bias must be 16B aligned"); return BV_ERR_INVALID;
  }
  if (g.epi == EPI_BIAS_GELU && (g.out_dtype != DT_BF16 || g.D2 == nullptr || g.reduce_out)) {
    set_error("bv_gemm: BIAS_GELU needs bf16 output, D2 and no reduce"); return BV_ERR_INVALID;
  }
  if (g.epi == EPI_BIAS_GELU && ((reinterpret_cast<uintptr_t>(g.D2) & 15) || (g.ldd2 % 8))) {
    set_error("bv_gemm: D2 must be 16B aligned with ldd2 %% 8 == 0"); return BV_ERR_INVALID;
  }
  if (g.out_dtype != DT_F32 && g.out_dtype != DT_BF16) { set_error("bv_gemm: bad out dtype"); return BV_ERR_INVALID; }
  if (g.colsum != nullptr && (g.out_dtype != DT_BF16 || g.reduce_out)) {
    set_error("bv_gemm: colsum needs a plain bf16 output"); return BV_ERR_INVALID;
  }
  int bn = g.block_n;
  if (bn == 0) bn = (g.N > 128) ? 256 : 128;
  if (bn == 256) return dispatch_epi<256>(g, stream);
  if (bn == 128) return dispatch_epi<128>(g, stream);
  set_error("bv_gemm: block_n must be 0, 128 or 256");
  return BV_ERR_INVALID;
}

}  // namespace bv
