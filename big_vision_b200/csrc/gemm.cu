// Warp-specialised, persistent wgmma GEMM for sm_90a.
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
// The grid is persistent: min(work units, SMs) CTAs, each running a static sequence of work units
// (one 128 x BN output tile x one K split; gemm_sched.h).  Roles (384 threads): warpgroup 0 is the
// TMA producer (one thread issues, the rest give their registers back with setmaxnreg), warpgroups
// 1 and 2 are the consumers, fed from a STAGES-deep ring of shared memory.  At BN = 128 they
// ping-pong: the CTA's units alternate between them, a warpgroup runs all 128 rows of its unit
// (two m64 x 128 x 16 wgmma per k16 step), and one warpgroup's epilogue runs while the other's MMAs
// keep the tensor cores busy.  At BN = 256 they cooperate: both run every unit, each m64 x 256 x 16 on
// its half of the rows.  The ring's barriers live for the whole CTA and the producer runs ahead
// across units, so the next tile's loads overlap this tile's epilogue.  Plain bf16 outputs leave
// through shared memory and TMA stores; a row-aligned aux operand (residual, gelu' pre-activation)
// arrives by TMA into the same staging buffers during the main loop.  fp32 and bf16 reduce-add
// outputs store from the registers.
#include "common.cuh"
#include "conv_gemm.h"
#include "gemm_sched.h"
#include "host_utils.h"

#include <atomic>
#include <type_traits>

#include <stdlib.h>
#include <string.h>

namespace bv {

namespace {

constexpr int BM = 128;          // rows per tile: two 64-row halves
constexpr int BK = 64;           // 64 bf16 = 128 B = one swizzle row
constexpr int A_STAGE_BYTES = BM * BK * 2;   // 16 KB
constexpr int NUM_THREADS = 384;
constexpr int SUB_BYTES = 64 * 64 * 2;       // one 64 x 64 bf16 output sub-tile, 128B-swizzled

// epilogue families (template parameter).  EF_RESID_ROWMOD is the residual whose aux rows wrap
// (aux_row_mod > 0, the position embedding): a tile's row window can wrap around it, so it is not one
// TMA box and its TMA-store kernel reads aux from global memory in the accumulator layout.
// EF_GELU_ACT is EF_GELU without the pre-activation output (forward-only MLPs): one staging buffer
// per sub-tile, so it keeps the stage count of EF_BIAS.
enum : int { EF_BIAS = 0, EF_GELU = 1, EF_RESID = 2, EF_DGELU = 3, EF_RESID_ROWMOD = 4, EF_GELU_ACT = 5 };
// output modes (template parameter): fp32 from the registers, bf16 reduce-add from the registers,
// plain bf16 by TMA store
enum : int { OM_F32 = 0, OM_BF16_ADD = 1, OM_BF16_TMA = 2 };

template <int BN, int OM, int EF>
struct Cfg {
  // BN = 128: ping-pong, each consumer warpgroup runs both 64-row halves of its own units.
  // BN = 256: cooperative, each consumer warpgroup runs one half of every unit.
  static constexpr bool PINGPONG = BN == 128;
  static constexpr int HALVES = PINGPONG ? 2 : 1;
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  // TMA-store staging of bf16 outputs, each buffer holding one 64 x 64 sub-tile of every output (GELU
  // writes two).  Per consumer warpgroup either two buffers (one fills while the other's store is in
  // flight), or, when aux is loaded by TMA, one buffer per sub-tile of the warpgroup's part of the
  // unit, so that the whole unit's aux is prefetched during its main loop.
  static constexpr bool AUX_TMA = OM == OM_BF16_TMA && (EF == EF_RESID || EF == EF_DGELU);
  static constexpr int OUTS = OM != OM_BF16_TMA ? 0 : (EF == EF_GELU ? 2 : 1);
  static constexpr int BUF_BYTES = OUTS * SUB_BYTES;
  static constexpr int BUFS = AUX_TMA ? HALVES * BN / 64 : 2;
  static constexpr int STAGING_BYTES = 2 * BUFS * BUF_BYTES;
  static constexpr int SMEM_LIMIT = 232448 - 2048;         // 227 KB minus barriers / align slack
  static constexpr int STAGES_FIT = (SMEM_LIMIT - STAGING_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 8 ? 8 : STAGES_FIT;
  static constexpr int STAGING_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = STAGING_OFFSET + STAGING_BYTES;
  // barriers: full and empty per stage, then (AUX_TMA) one per staging buffer of each warpgroup, then
  // (PINGPONG) one per warpgroup that completes a phase when all of its unit's k blocks have landed
  static constexpr int AUX_BAR = 2 * STAGES;
  static constexpr int ISSUED_BAR = AUX_BAR + (AUX_TMA ? 2 * BUFS : 0);
  static constexpr int SMEM_BYTES = BAR_OFFSET + 256 + 1024;  // + barriers + align slack
  static_assert(STAGES >= 3, "shared-memory budget leaves fewer than 3 stages");
  static_assert(8 * (ISSUED_BAR + 2) <= 256, "barriers overflow their 256 bytes");
};

struct GemmDev {
  GemmSched s;
  int M, N;
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

// What the producer loads per k block (template parameter).  PROD_GEMM: the 2-D tiles of A and B.  The
// convolution modes (conv_gemm.h) read A from an NHWC activation by TMA in im2col mode, so no im2col matrix
// is ever written: PROD_CONV is the forward / data gradient, whose k block (tap, 64-channel block) loads 128
// output pixels x 64 channels of the tap-shifted input (A K-major) and the tap's rows of the kernel (B);
// PROD_WGRAD is the kernel gradient, whose M rows are (tap, input channel) and whose k block is 64 output
// pixels: A is two 64-pixel x 64-channel im2col boxes (MN-major), B the 64 pixels' rows of dy (MN-major).
enum : int { PROD_GEMM = 0, PROD_CONV = 1, PROD_WGRAD = 2 };

struct ConvDev {
  int gh, gw;              // the output-pixel grid whose row-major order (img, y, x) the pixel index runs over
  int lw, lh, es;          // input base position of grid point (x, y) = (lw + es * x, lh + es * y)
  int cblocks, cin;        // 64-channel blocks per tap (PROD_CONV); channels per tap of M (PROD_WGRAD)
  int ntaps;
  uint16_t offw[kConvMaxTaps], offh[kConvMaxTaps];   // the tap's shift of the base position
  int brow[kConvMaxTaps];  // PROD_CONV: first row of the tap's kernel slice in the 2-D map of B
};

// the input base position (w, h) and image of output pixel m
__device__ __forceinline__ void conv_base(const ConvDev& cv, int m, int& img, int& bw, int& bh) {
  const int t = m / cv.gw, x = m - t * cv.gw;
  img = t / cv.gh;
  const int y = t - img * cv.gh;
  bw = cv.lw + cv.es * x;
  bh = cv.lh + cv.es * y;
}

// The consumer warpgroup's main loop over one unit's k blocks, for the H 64-row halves h0 .. h0 + H - 1
// of the tile; acc[h] holds half h0 + h.  `ps` is the running ring position, carried from unit to
// unit.  The transpose bits of wgmma are immediates, so each operand layout pair is its own
// instantiation (a branch between wgmma issues would make ptxas serialise them).  `after_first` runs
// once, after the first k block's MMAs are committed, so that whatever it waits for overlaps them;
// `after_last` runs once, after the last k block's MMAs are committed.
template <int BN, int H, int STAGES, int STAGE_BYTES, int TA, int TB, typename F, typename G>
__device__ __forceinline__ void mainloop(float (&acc)[H][BN / 2], uint32_t base, uint32_t bar_base, int h0,
                                         PipeState& ps, int kb0, int kb1, F&& after_first, G&& after_last) {
  // 128B-swizzled operand tiles: K-major rows of 128 B (8-row groups 1024 B apart, K step 32 B);
  // MN-major boxes of 64 (M|N) x 64 (K), 8 KB each (K step 16 rows = 2048 B).  Either way rows
  // 64 .. 127 of the A tile start 8 KB after row 0.
  constexpr uint32_t a_lbo = TA ? 8192u : 16u, b_lbo = TB ? 8192u : 16u;
  constexpr uint32_t a_kstep = TA ? 2048u : 32u, b_kstep = TB ? 2048u : 32u;
  int prev_stage = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(bar_base + 8u * ps.stage, ps.phase);
    const uint32_t a_s = base + ps.stage * STAGE_BYTES + h0 * 8192;
    const uint32_t b_s = base + ps.stage * STAGE_BYTES + A_STAGE_BYTES;
    const uint64_t bdesc = wgmma_desc_sw128(b_s, b_lbo, 1024u);
    uint64_t adesc[H];
#pragma unroll
    for (int h = 0; h < H; ++h) {
      adesc[h] = wgmma_desc_sw128(a_s + h * 8192, a_lbo, 1024u);
      wgmma_fence_regs(acc[h]);
    }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t b = bdesc + k * (b_kstep >> 4);
      const int accumulate = (kb > kb0 || k > 0) ? 1 : 0;    // the first MMA overwrites the registers
#pragma unroll
      for (int h = 0; h < H; ++h) {
        const uint64_t a = adesc[h] + k * (a_kstep >> 4);
        if constexpr (BN == 256) wgmma_ss_n256<TA, TB>(acc[h], a, b, accumulate);
        else wgmma_ss_n128<TA, TB>(acc[h], a, b, accumulate);
      }
    }
    wgmma_commit();
#pragma unroll
    for (int h = 0; h < H; ++h) wgmma_fence_regs(acc[h]);
    if (kb == kb0) after_first();
    if (kb == kb1 - 1) after_last();
    // keep this k block's MMAs in flight; the previous one has retired -> its slot is free
    wgmma_wait<1>();
    if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_base + 8u * (STAGES + prev_stage));
    prev_stage = ps.stage;
    ps.advance(STAGES);
  }
  // every MMA of the unit has retired, so the last slot is free before the epilogue starts
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < H; ++h) wgmma_fence_regs(acc[h]);
  if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_base + 8u * (STAGES + prev_stage));
}

// The aux pair (col, col + 1) of one row, read from global memory in the accumulator layout (col + 1
// only if `pair`); aux_row_mod > 0 wraps the row.  The register epilogues and EF_RESID_ROWMOD use it.
__device__ __forceinline__ void aux_global(const GemmDev& p, int row, int col, bool pair, float& a0, float& a1) {
  const long long ar = p.aux_row_mod > 0 ? (row % p.aux_row_mod) : row;
  const bf16* ap = p.aux + ar * p.ldaux + col;
  if (pair) {
    const uint32_t q = *reinterpret_cast<const uint32_t*>(ap);
    a0 = bf16_lo(q); a1 = bf16_hi(q);
  } else {
    a0 = __bfloat162float(*ap);
    a1 = 0.f;
  }
}

// alpha, bias and the element-wise op of the epilogue on one column pair (col, col + 1) of one row.
// a0/a1: the aux pair (residual or gelu' pre-activation).  pre0/pre1: GELU's pre-activation
// (bf16-rounded).
template <bool OUT_F32, int EF>
__device__ __forceinline__ void epi_math(float alpha, float c0, float c1, float b0, float b1, float a0, float a1,
                                         float& v0, float& v1, float& pre0, float& pre1) {
  v0 = c0 * alpha + b0;
  v1 = c1 * alpha + b1;
  pre0 = pre1 = 0.f;
  if (EF == EF_GELU || EF == EF_GELU_ACT) {
    pre0 = round_bf16(v0); pre1 = round_bf16(v1);
    v0 = gelu_tanh_fast(pre0); v1 = gelu_tanh_fast(pre1);
  } else if (EF == EF_RESID || EF == EF_RESID_ROWMOD) {
    v0 = (OUT_F32 ? v0 : round_bf16(v0)) + a0;
    v1 = (OUT_F32 ? v1 : round_bf16(v1)) + a1;
  } else if (EF == EF_DGELU) {
    v0 *= gelu_tanh_grad_fast(a0);
    v1 *= gelu_tanh_grad_fast(a1);
  }
}

// Accumulator layout (per warp w of the warpgroup, lane l): element 4j + e sits at row
// 16w + l/4 + 8*(e >> 1), column 8j + 2*(l%4) + (e & 1).

// Bias gradient fused into the producer: s0/s1 are one thread's sums of the stored (bf16-rounded)
// values in columns col and col + 1; the eight lanes that share a column pair are summed with
// shuffles, then one atomic per warp and column.
__device__ __forceinline__ void colsum_add(float* colsum, int N, float s0, float s1, int col, int lane) {
  s0 += __shfl_xor_sync(0xffffffffu, s0, 4);
  s0 += __shfl_xor_sync(0xffffffffu, s0, 8);
  s0 += __shfl_xor_sync(0xffffffffu, s0, 16);
  s1 += __shfl_xor_sync(0xffffffffu, s1, 4);
  s1 += __shfl_xor_sync(0xffffffffu, s1, 8);
  s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
  if (lane < 4) {
    if (col < N) atomicAdd(colsum + col, s0);
    if (col + 1 < N) atomicAdd(colsum + col + 1, s1);
  }
}

// Epilogue straight from the registers: fp32 outputs, and bf16 reduce-add outputs (gradient
// accumulation; never with colsum).  Under split-K every unit adds its partial into D, so bias and a
// residual are added only by the unit of the first split (kb0 == 0); gelu' scales every partial.
// r0 is the first row of the warpgroup's 64-row half.
template <int BN, bool OUT_F32, int EF>
__device__ __forceinline__ void epilogue_regs(const GemmDev& p, const float (&acc)[BN / 2], int r0, int n0,
                                              int kb0) {
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int row0 = r0 + warp * 16 + (lane >> 2);
  const int pM = p.M, pN = p.N;
  const float alpha = p.alpha;
  const bool reduce = p.reduce_out != 0;
  const bool first = kb0 == 0;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * (lane & 3);
    if (col >= pN) continue;
    const bool pair = col + 1 < pN;
    float b0 = 0.f, b1 = 0.f;
    if (p.bias != nullptr && first) {
      b0 = __ldg(p.bias + col);
      if (pair) b1 = __ldg(p.bias + col + 1);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      if (row >= pM) continue;
      float v0, v1, pre0, pre1, a0 = 0.f, a1 = 0.f;
      if ((EF == EF_RESID && first) || EF == EF_DGELU) aux_global(p, row, col, pair, a0, a1);
      epi_math<OUT_F32, EF>(alpha, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], b0, b1, a0, a1, v0, v1, pre0, pre1);
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
        // the pair, or (last column of an odd N) its low half, as one predicated reduction: two branches
        // here, one per case, make ptxas spill the 128 accumulators of a ping-pong unit
        bf16* dp = static_cast<bf16*>(p.d) + row * p.ldd + col;
        const uint32_t o = pack_bf16(v0, v1);
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            ".reg .b16 lo, hi;\n"
            "setp.ne.u32 p, %2, 0;\n"
            "mov.b32 {lo, hi}, %1;\n"
            "@p red.global.add.noftz.bf16x2 [%0], %1;\n"
            "@!p red.global.add.noftz.bf16 [%0], lo;\n"
            "}\n" ::"l"(dp), "r"(o), "r"(pair ? 1u : 0u)
            : "memory");
      }
    }
  }
}

// Epilogue through shared memory for plain bf16 outputs, for one 64-row half of the tile (first row
// r0): the warpgroup writes each 64-column sub-tile of those rows into a 128B-swizzled staging buffer
// (the 16-byte chunk index XOR the row mod 8, so the 8 rows of one store instruction hit different
// banks), and one thread stores it with
// TMA, which clips rows >= M and columns >= N8 = N rounded down to a multiple of 8.  TMA writes the
// innermost dimension in whole 16-byte chunks, so a map of width N with N % 8 != 0 would write the
// chunk's columns N .. round_up(N, 8) - 1 of a strided output; the N % 8 columns past N8 are copied
// from the staging buffer by the threads instead.
//
// Without a TMA-loaded aux the two buffers alternate; `nstore` counts the warpgroup's sub-tiles across
// units, and the issuing thread waits until the store that last read a buffer is done reading before
// the buffer is refilled.  With one (EF_RESID, EF_DGELU), sub-tile c of the half uses buffer c after
// `staging`, which already holds the aux sub-tile (issue_aux_loads, same swizzle): each thread waits
// on the buffer's barrier (phase `aux_parity`), reads its aux pair at the offset where it then writes
// its output pair, and the output overwrites the aux in place.
template <int BN, int EF, int BUF_BYTES>
__device__ __forceinline__ void epilogue_tma(const GemmDev& p, const CUtensorMap* tmD, const CUtensorMap* tmD2,
                                             const float (&acc)[BN / 2], int r0, int n0, int cw, uint32_t staging,
                                             uint32_t& nstore, uint32_t aux_bar, uint32_t aux_parity) {
  constexpr bool AUX_TMA = (EF == EF_RESID || EF == EF_DGELU);
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const bool leader = (threadIdx.x & 127) == 0;
  const int rl0 = warp * 16 + (lane >> 2);       // row within the half
  const int row0 = r0 + rl0;
  const int pM = p.M, pN = p.N, pN8 = p.N & ~7;
  const float alpha = p.alpha;
#pragma unroll
  for (int c = 0; c < BN / 64; ++c) {
    uint32_t buf;
    if constexpr (AUX_TMA) {
      buf = staging + c * BUF_BYTES;
      mbar_wait(aux_bar + 8u * c, aux_parity);
    } else {
      buf = staging + (nstore & 1u) * BUF_BYTES;
      if (leader) tma_store_wait_read<1>();
      named_bar_sync(1 + cw, 128);
    }
    float cs[8][2];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int j = 8 * c + jj;
      const int col = n0 + 8 * j + 2 * (lane & 3);
      cs[jj][0] = cs[jj][1] = 0.f;
      const bool cin = col < pN, pair = col + 1 < pN;
      float b0 = 0.f, b1 = 0.f;
      if (cin && p.bias != nullptr) {
        b0 = __ldg(p.bias + col);
        if (pair) b1 = __ldg(p.bias + col + 1);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rl = rl0 + 8 * h, row = row0 + 8 * h;
        const uint32_t off = rl * 128 + ((jj ^ (rl & 7)) << 4) + (lane & 3) * 4;
        float v0 = 0.f, v1 = 0.f, pre0 = 0.f, pre1 = 0.f;
        const bool in = cin && row < pM;
        if (in) {
          float a0 = 0.f, a1 = 0.f;
          if constexpr (AUX_TMA) {
            // without `pair`, a1 is the box's zero fill past column N and is never stored
            uint32_t q;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(q) : "r"(buf + off));
            a0 = bf16_lo(q); a1 = bf16_hi(q);
          } else if constexpr (EF == EF_RESID_ROWMOD) {
            aux_global(p, row, col, pair, a0, a1);
          }
          epi_math<false, EF>(alpha, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], b0, b1, a0, a1, v0, v1, pre0, pre1);
        }
        const __nv_bfloat162 o = __floats2bfloat162_rn(v0, v1);
        if (in) {
          cs[jj][0] += __low2float(o);
          cs[jj][1] += pair ? __high2float(o) : 0.f;
        }
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(buf + off), "r"(*reinterpret_cast<const uint32_t*>(&o))
                     : "memory");
        if (EF == EF_GELU) {
          const __nv_bfloat162 q = __floats2bfloat162_rn(pre0, pre1);
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(buf + SUB_BYTES + off),
                       "r"(*reinterpret_cast<const uint32_t*>(&q))
                       : "memory");
        }
      }
    }
    // make the generic-proxy writes visible to the TMA engine, then hand the buffer to one thread
    fence_proxy_async();
    named_bar_sync(1 + cw, 128);
    if (leader) {
      if (n0 + 64 * c < pN8 && r0 < pM) {     // sub-tiles wholly past N8 are not stored
        tma_store_2d(tmD, buf, n0 + 64 * c, r0);
        if (EF == EF_GELU) tma_store_2d(tmD2, buf + SUB_BYTES, n0 + 64 * c, r0);
      }
      tma_store_commit();
    }
    // The sub-tile holding the partial chunk (N % 8 != 0): its N - N8 columns go from the staging
    // buffer to global memory here, one row of D (and of D2) per thread.  The branch is uniform over
    // the warpgroup, and its barrier keeps the buffer from being refilled before every read is done.
    const int tail0 = pN8 - (n0 + 64 * c);
    if (pN8 < pN && tail0 >= 0 && tail0 < 64) {
      const int t = threadIdx.x & 127, rl = t & 63, out = t >> 6;
      const int row = r0 + rl;
      if (row < pM && (out == 0 || EF == EF_GELU)) {
        const uint32_t src = buf + out * SUB_BYTES + rl * 128 + (((tail0 >> 3) ^ (rl & 7)) << 4);
        uint16_t* dst = reinterpret_cast<uint16_t*>(out ? p.d2 : p.d) + row * (out ? p.ldd2 : p.ldd) + pN8;
#pragma unroll 1
        for (int e = 0; e < pN - pN8; ++e) {
          uint16_t u;
          asm volatile("ld.shared.u16 %0, [%1];" : "=h"(u) : "r"(src + 2 * e));
          dst[e] = u;
        }
      }
      named_bar_sync(1 + cw, 128);
    }
    if (!AUX_TMA) ++nstore;
    if (p.colsum != nullptr) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        colsum_add(p.colsum, pN, cs[jj][0], cs[jj][1], n0 + 8 * (8 * c + jj) + 2 * (lane & 3), lane);
    }
  }
}

// Run by the warpgroup's leader thread, which owns the warpgroup's bulk-store groups: once every store
// of the warpgroup's previous unit has finished reading its staging buffer, TMA-load the aux sub-tiles
// (64 rows x 64 columns, 128B-swizzled like the outputs) of the H halves h0 .. h0 + H - 1 of this unit
// into buffers 0 .. H * BN/64 - 1, half by half.  A sub-tile wholly past N, or a half whose 64 rows
// are all past M, is never stored, so its aux is not loaded; a plain arrival completes the barrier's
// phase instead, which keeps every barrier's phase equal to the warpgroup's unit count and the
// consumers' wait unconditional.
template <int BN, int H>
__device__ __forceinline__ void issue_aux_loads(const CUtensorMap* tmAux, int M, int N, int m0, int n0, int h0,
                                                uint32_t staging, uint32_t aux_bar) {
  tma_store_wait_read<0>();
#pragma unroll
  for (int h = 0; h < H; ++h) {
    const int r0 = m0 + 64 * (h0 + h);
#pragma unroll
    for (int c = 0; c < BN / 64; ++c) {
      const int b = h * (BN / 64) + c;
      const uint32_t bar = aux_bar + 8u * b;
      if (n0 + 64 * c < N && r0 < M) {
        mbar_expect_tx(bar, SUB_BYTES);        // the full box, zero fill included
        tma_load_2d(staging + b * SUB_BYTES, tmAux, bar, n0 + 64 * c, r0);
      } else {
        mbar_arrive(bar);
      }
    }
  }
}

// The convolution modes take a ConvDev; the plain GEMM an empty placeholder.
struct NoConv {};
template <int PROD>
using ConvParam = std::conditional_t<PROD == PROD_GEMM, NoConv, ConvDev>;

template <int BN, int OM, int EF, int PROD>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmD2,
            const __grid_constant__ CUtensorMap tmAux, const GemmDev p, const __grid_constant__ ConvParam<PROD> cv) {
  using C = Cfg<BN, OM, EF>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;
  const uint32_t bar_base = base + C::BAR_OFFSET;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };

  const int wg = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);
  const int units = p.s.units;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (C::AUX_TMA) tma_prefetch_desc(&tmAux);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), C::PINGPONG ? 1 : 2);     // one arrival per warpgroup that reads the stage
    }
    if (C::AUX_TMA) {
      for (int b = 0; b < 2 * C::BUFS; ++b) mbar_init(bar_base + 8u * (C::AUX_BAR + b), 1);
    }
    if (C::PINGPONG) {
      for (int b = 0; b < 2; ++b) mbar_init(bar_base + 8u * (C::ISSUED_BAR + b), 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ========================= TMA producer =========================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      PipeState ps;
      for (int u = blockIdx.x; u < units; u += gridDim.x) {
        const WorkUnit w = gemm_work_unit(p.s, u, BM, BN);
        if constexpr (PROD == PROD_GEMM) {
          for (int kb = w.kb0; kb < w.kb1; ++kb) {
            mbar_wait(empty_bar(ps.stage), ps.phase ^ 1u);
            const uint32_t a_s = base + ps.stage * C::STAGE_BYTES;
            const uint32_t b_s = a_s + A_STAGE_BYTES;
            const uint32_t fb = full_bar(ps.stage);
            mbar_expect_tx(fb, C::STAGE_BYTES);
            const int k0 = kb * BK;
            if (p.a_mn) {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(a_s + j * 8192, &tmA, fb, w.m0 + 64 * j, k0);
            } else {
              tma_load_2d(a_s, &tmA, fb, k0, w.m0);
            }
            if (p.b_mn) {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_2d(b_s + j * 8192, &tmB, fb, w.n0 + 64 * j, k0);
            } else {
              tma_load_2d(b_s, &tmB, fb, k0, w.n0);
            }
            ps.advance(C::STAGES);
          }
        } else {
          int img = 0, bw = 0, bh = 0;
          if constexpr (PROD == PROD_CONV) conv_base(cv, w.m0, img, bw, bh);
          for (int kb = w.kb0; kb < w.kb1; ++kb) {
            mbar_wait(empty_bar(ps.stage), ps.phase ^ 1u);
            const uint32_t a_s = base + ps.stage * C::STAGE_BYTES;
            const uint32_t b_s = a_s + A_STAGE_BYTES;
            const uint32_t fb = full_bar(ps.stage);
            mbar_expect_tx(fb, C::STAGE_BYTES);
            const int k0 = kb * BK;
            if constexpr (PROD == PROD_CONV) {
              const int tap = kb / cv.cblocks, c0 = (kb - tap * cv.cblocks) * BK, brow = cv.brow[tap];
              tma_load_im2col_4d(a_s, &tmA, fb, c0, bw, bh, img, cv.offw[tap], cv.offh[tap]);
              if (p.b_mn) {
#pragma unroll
                for (int j = 0; j < BN / 64; ++j) tma_load_2d(b_s + j * 8192, &tmB, fb, w.n0 + 64 * j, brow + c0);
              } else {
                tma_load_2d(b_s, &tmB, fb, c0, brow + w.n0);
              }
            } else {
              conv_base(cv, k0, img, bw, bh);
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) {
                // a box past the last tap (M = taps x cin is a multiple of 64) loads tap 0; its rows are not stored
                const int m = w.m0 + 64 * j, t = m / cv.cin, tap = t < cv.ntaps ? t : 0;
                tma_load_im2col_4d(a_s + j * 8192, &tmA, fb, m - t * cv.cin, bw, bh, img, cv.offw[tap],
                                   cv.offh[tap]);
              }
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_2d(b_s + j * 8192, &tmB, fb, w.n0 + 64 * j, k0);
            }
            ps.advance(C::STAGES);
          }
        }
      }
    }
    return;
  }

  // ========================= consumers: warpgroups 1, 2 =========================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = wg - 1;
  constexpr int H = C::HALVES;
  const int h0 = C::PINGPONG ? 0 : cw;          // the warpgroup's first 64-row half of a tile
  const uint32_t staging = base + C::STAGING_OFFSET + cw * C::BUFS * C::BUF_BYTES;
  const uint32_t aux_bar = bar_base + 8u * (C::AUX_BAR + cw * C::BUFS);
  const bool leader = (threadIdx.x & 127) == 0;
  uint32_t nstore = 0;
  PipeState ps;
  ConsumerWalk walk(blockIdx.x, gridDim.x, C::PINGPONG ? cw : -1);
  WorkUnit w;
  constexpr int S = C::STAGES, SB = C::STAGE_BYTES;
  for (int j = 0; walk.next(p.s, BM, BN, S, ps, w); ++j) {
    // Ping-pong: this warpgroup's ring position skipped the other warpgroup's previous unit without
    // waiting, and a parity wait on a full barrier is only sound once that barrier's previous phase has
    // completed.  So wait until every k block of that unit has landed (the other warpgroup's
    // (j + cw - 1)-th unit; warpgroup 0's first unit has none).  This also orders the two main loops.
    if constexpr (C::PINGPONG) {
      const int prev = j + cw - 1;
      if (prev >= 0) mbar_wait(bar_base + 8u * (C::ISSUED_BAR + 1 - cw), prev & 1);
    }
    // the leader's wait for the previous unit's stores overlaps the first k block's MMAs
    auto after_first = [&]() {
      if constexpr (C::AUX_TMA) {
        if (leader) issue_aux_loads<BN, H>(&tmAux, p.M, p.N, w.m0, w.n0, h0, staging, aux_bar);
      }
    };
    auto after_last = [&]() {
      if constexpr (C::PINGPONG) {
        if (leader) mbar_arrive(bar_base + 8u * (C::ISSUED_BAR + cw));
      }
    };
    float acc[H][BN / 2];
    if (p.a_mn) {
      if (p.b_mn) mainloop<BN, H, S, SB, 1, 1>(acc, base, bar_base, h0, ps, w.kb0, w.kb1, after_first, after_last);
      else mainloop<BN, H, S, SB, 1, 0>(acc, base, bar_base, h0, ps, w.kb0, w.kb1, after_first, after_last);
    } else {
      if (p.b_mn) mainloop<BN, H, S, SB, 0, 1>(acc, base, bar_base, h0, ps, w.kb0, w.kb1, after_first, after_last);
      else mainloop<BN, H, S, SB, 0, 0>(acc, base, bar_base, h0, ps, w.kb0, w.kb1, after_first, after_last);
    }

#pragma unroll
    for (int h = 0; h < H; ++h) {
      const int r0 = w.m0 + 64 * (h0 + h);
      if constexpr (OM == OM_BF16_TMA) {
        const int b = C::AUX_TMA ? h * (BN / 64) : 0;
        epilogue_tma<BN, EF, C::BUF_BYTES>(p, &tmD, &tmD2, acc[h], r0, w.n0, cw, staging + b * C::BUF_BYTES, nstore,
                                           aux_bar + 8u * b, j & 1);
      } else {
        epilogue_regs<BN, OM == OM_F32, EF>(p, acc[h], r0, w.n0, w.kb0);
      }
    }
  }
  // the staging buffers must outlive every bulk store that reads them
  if (OM == OM_BF16_TMA && leader) tma_store_wait<0>();
}

// The dynamic-shared-memory opt-in is a per-DEVICE attribute of the kernel: cache it per device and
// instantiation (one process may drive several GPUs from several host threads; the flags are atomics and a
// duplicate set by two racing threads is harmless).
template <int BN, int OM, int EF, int PROD>
int opt_in_smem() {
  auto kern = gemm_kernel<BN, OM, EF, PROD>;
  const int bytes = Cfg<BN, OM, EF>::SMEM_BYTES;
  static std::atomic<bool> attr_set[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = -1;
  if (dev < 0 || !attr_set[dev].load(std::memory_order_acquire)) {
    const int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes),
                              "cudaFuncSetAttribute(gemm)");
    if (rc) return rc;
    if (dev >= 0) attr_set[dev].store(true, std::memory_order_release);
  }
  return BV_OK;
}

template <int BN, int OM, int EF>
int launch_cfg(const bv_gemm_args& g, cudaStream_t stream) {
  using C = Cfg<BN, OM, EF>;
  CUtensorMap tmA, tmB, tmD, tmD2, tmAux;
  int rc;
  const CUtensorMapDataType bf = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if (g.a_mn) rc = make_tmap_2d(&tmA, bf, g.A, g.M, g.K, g.lda * 2, 64, 64);
  else        rc = make_tmap_2d(&tmA, bf, g.A, g.K, g.M, g.lda * 2, 64, BM);
  if (rc) return rc;
  if (g.b_mn) rc = make_tmap_2d(&tmB, bf, g.B, g.N, g.K, g.ldb * 2, 64, 64);
  else        rc = make_tmap_2d(&tmB, bf, g.B, g.K, g.N, g.ldb * 2, 64, BN);
  if (rc) return rc;

  GemmDev p;
  const long long tiles = ((g.M + BM - 1) / BM) * ((g.N + BN - 1) / BN);
  if (tiles * ((g.K + BK - 1) / BK) > 0x7fffffffLL) { set_error("bv_gemm: problem too large"); return BV_ERR_INVALID; }
  if (!gemm_make_sched(g.M, g.N, g.K, BM, BN, BK, g.splits, g.reduce_out != 0, num_sms(), &p.s)) {
    set_error("bv_gemm: split-K requires reduce_out=1");
    return BV_ERR_INVALID;
  }
  p.M = (int)g.M; p.N = (int)g.N;
  p.a_mn = g.a_mn; p.b_mn = g.b_mn; p.reduce_out = g.reduce_out;
  p.alpha = g.alpha;
  p.bias = g.epilogue == BV_EPI_NONE ? nullptr : g.bias;     // BV_EPI_NONE ignores bias (bv_b200.h)
  p.colsum = g.colsum;
  p.aux = reinterpret_cast<const bf16*>(g.aux);
  p.ldaux = g.ldaux;
  p.aux_row_mod = g.aux_row_mod;
  p.d = g.D; p.d2 = g.D2;
  p.ldd = g.ldd; p.ldd2 = g.ldd2;
  // the output maps span M x N8 (N rounded down to a multiple of 8; epilogue_tma stores the columns
  // past N8 with plain stores), so TMA leaves the rows past M and the columns past N of a strided
  // output alone.  With N < 8 there is no map: every column is stored that way.
  memset(&tmD, 0, sizeof(tmD));
  memset(&tmD2, 0, sizeof(tmD2));
  memset(&tmAux, 0, sizeof(tmAux));
  const long long n8 = g.N & ~7LL;
  if (OM == OM_BF16_TMA && n8 > 0) {
    rc = make_tmap_2d(&tmD, bf, g.D, n8, g.M, g.ldd * 2, 64, 64);
    if (rc) return rc;
    if (EF == EF_GELU) {
      rc = make_tmap_2d(&tmD2, bf, g.D2, n8, g.M, g.ldd2 * 2, 64, 64);
      if (rc) return rc;
    }
  }
  // aux is read through the same M x N window and box as the output it is staged with (the checks in
  // bv_gemm give TMA's 16-byte base and row-stride alignment)
  if (C::AUX_TMA) {
    rc = make_tmap_2d(&tmAux, bf, g.aux, g.N, g.M, g.ldaux * 2, 64, 64);
    if (rc) return rc;
  }

  auto kern = gemm_kernel<BN, OM, EF, PROD_GEMM>;
  rc = opt_in_smem<BN, OM, EF, PROD_GEMM>();
  if (rc) return rc;
  const int grid = p.s.units < num_sms() ? p.s.units : num_sms();
  kern<<<grid, NUM_THREADS, C::SMEM_BYTES, stream>>>(tmA, tmB, tmD, tmD2, tmAux, p, NoConv{});
  return check_cuda(cudaGetLastError(), "gemm_kernel launch");
}

// Plain bf16 outputs leave by TMA store; fp32 outputs and bf16 reduce-add outputs keep the register
// epilogue.  bf16 reduce-adds (gradient accumulation into bf16, not on the training step's path) run
// the ping-pong kernel (BN = 128) whatever BN is asked for: cooperative at 256, their atomics make
// ptxas spill the accumulators inside the persistent loop.
template <int BN>
int dispatch_epi(const bv_gemm_args& g, cudaStream_t s) {
  const bool f32 = (g.out_dtype == DT_F32), add = !f32 && g.reduce_out;
  switch (g.epilogue) {
    case BV_EPI_NONE:
    case BV_EPI_BIAS:
      return f32 ? launch_cfg<BN, OM_F32, EF_BIAS>(g, s)
                 : add ? launch_cfg<128, OM_BF16_ADD, EF_BIAS>(g, s) : launch_cfg<BN, OM_BF16_TMA, EF_BIAS>(g, s);
    case BV_EPI_BIAS_RESID:
      if (f32) return launch_cfg<BN, OM_F32, EF_RESID>(g, s);
      if (add) return launch_cfg<128, OM_BF16_ADD, EF_RESID>(g, s);
      return g.aux_row_mod > 0 ? launch_cfg<BN, OM_BF16_TMA, EF_RESID_ROWMOD>(g, s)
                               : launch_cfg<BN, OM_BF16_TMA, EF_RESID>(g, s);
    case BV_EPI_BIAS_GELU:     // never a reduce-add (refused in bv_gemm)
      return launch_cfg<BN, OM_BF16_TMA, EF_GELU>(g, s);
    case BV_EPI_BIAS_GELU_ACT:
      return launch_cfg<BN, OM_BF16_TMA, EF_GELU_ACT>(g, s);
    case BV_EPI_DGELU:
      if (f32) { set_error("bv_gemm: DGELU epilogue writes bf16"); return BV_ERR_INVALID; }
      if (g.aux_row_mod > 0) { set_error("bv_gemm: DGELU takes a row-aligned aux"); return BV_ERR_INVALID; }
      return add ? launch_cfg<128, OM_BF16_ADD, EF_DGELU>(g, s) : launch_cfg<BN, OM_BF16_TMA, EF_DGELU>(g, s);
  }
  set_error("bv_gemm: bad epilogue %d", g.epilogue);
  return BV_ERR_INVALID;
}

template <int BN, int OM, int EF, int PROD>
int launch_conv_cfg(const ConvGemm& g, cudaStream_t stream) {
  using C = Cfg<BN, OM, EF>;
  const bool wgrad = PROD == PROD_WGRAD;
  const long long pixels = g.n * g.gh * g.gw;
  const long long M = wgrad ? (long long)g.ntaps * g.c : pixels;
  const long long K = wgrad ? pixels : (long long)g.ntaps * g.c;
  const CUtensorMapDataType bf = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap tmA, tmB, tmD, tmD2, tmAux;
  memset(&tmD, 0, sizeof(tmD));
  memset(&tmD2, 0, sizeof(tmD2));
  memset(&tmAux, 0, sizeof(tmAux));
  int rc = make_tmap_im2col_nhwc(&tmA, g.x, g.n, g.h, g.w, g.c, g.lw, g.lh, g.lw + g.stride * (g.gw - 1) - (g.w - 1),
                                 g.lh + g.stride * (g.gh - 1) - (g.h - 1), g.stride, wgrad ? 64 : BM);
  if (rc) return rc;
  if (wgrad || g.b_mn) rc = make_tmap_2d(&tmB, bf, g.b, g.b_cols, g.b_rows, (uint64_t)g.b_cols * 2, 64, 64);
  else rc = make_tmap_2d(&tmB, bf, g.b, g.b_cols, g.b_rows, (uint64_t)g.b_cols * 2, 64, BN);
  if (rc) return rc;

  GemmDev p;
  if ((M + BM - 1) / BM * ((g.N + BN - 1) / BN) * ((K + BK - 1) / BK) > 0x7fffffffLL || M > 0x7fffffffLL) {
    set_error("bv_conv: problem too large");
    return BV_ERR_INVALID;
  }
  gemm_make_sched(M, g.N, K, BM, BN, BK, wgrad ? 0 : 1, wgrad, num_sms(), &p.s);
  p.M = (int)M; p.N = g.N;
  p.a_mn = wgrad ? 1 : 0;
  p.b_mn = wgrad ? 1 : g.b_mn;
  p.reduce_out = wgrad ? 1 : 0;
  p.alpha = 1.f;
  p.bias = nullptr;
  p.colsum = nullptr;
  p.aux = reinterpret_cast<const bf16*>(g.resid);
  p.ldaux = g.N;
  p.aux_row_mod = 0;
  p.d = g.out; p.d2 = nullptr;
  p.ldd = g.N; p.ldd2 = 0;
  if (OM == OM_BF16_TMA) {
    rc = make_tmap_2d(&tmD, bf, g.out, g.N, M, (uint64_t)g.N * 2, 64, 64);
    if (rc) return rc;
  }
  if (C::AUX_TMA) {
    rc = make_tmap_2d(&tmAux, bf, g.resid, g.N, M, (uint64_t)g.N * 2, 64, 64);
    if (rc) return rc;
  }
  ConvDev cv;
  memset(&cv, 0, sizeof(cv));
  cv.gh = g.gh; cv.gw = g.gw; cv.lw = g.lw; cv.lh = g.lh; cv.es = g.stride;
  cv.cblocks = g.c / BK; cv.cin = g.c; cv.ntaps = g.ntaps;
  for (int t = 0; t < g.ntaps; ++t) {
    cv.offw[t] = (uint16_t)g.taps[t].ow;
    cv.offh[t] = (uint16_t)g.taps[t].oh;
    cv.brow[t] = g.taps[t].brow;
  }
  auto kern = gemm_kernel<BN, OM, EF, PROD>;
  rc = opt_in_smem<BN, OM, EF, PROD>();
  if (rc) return rc;
  const int grid = p.s.units < num_sms() ? p.s.units : num_sms();
  kern<<<grid, NUM_THREADS, C::SMEM_BYTES, stream>>>(tmA, tmB, tmD, tmD2, tmAux, p, cv);
  return check_cuda(cudaGetLastError(), "gemm_kernel (convolution) launch");
}

}  // namespace

// Forward and data gradient: bf16 outputs on the ping-pong kernel, with the residual epilogue when resid is
// given.  Kernel gradient: fp32 reduce-add, cooperative at BN = 256 when N > 128, as bv_gemm's fp32 outputs.
int conv_gemm(const ConvGemm& g, cudaStream_t s) {
  if (g.wgrad) {
    return g.N > 128 ? launch_conv_cfg<256, OM_F32, EF_BIAS, PROD_WGRAD>(g, s)
                     : launch_conv_cfg<128, OM_F32, EF_BIAS, PROD_WGRAD>(g, s);
  }
  return g.resid ? launch_conv_cfg<128, OM_BF16_TMA, EF_RESID, PROD_CONV>(g, s)
                 : launch_conv_cfg<128, OM_BF16_TMA, EF_BIAS, PROD_CONV>(g, s);
}

}  // namespace bv

extern "C" {

int bv_gemm(const bv_gemm_args* args, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!args) { set_error("bv_gemm: null args"); return BV_ERR_INVALID; }
  const bv_gemm_args& g = *args;
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) { set_error("bv_gemm: empty problem"); return BV_ERR_INVALID; }
  // N need not be a multiple of 8 as long as the row strides are (TMA clips the loads and stores)
  if (g.out_dtype == DT_BF16 && ((reinterpret_cast<uintptr_t>(g.D) & 15) || (g.ldd % 8))) {
    set_error("bv_gemm: bf16 output must be 16B aligned with ldd %% 8 == 0"); return BV_ERR_INVALID;
  }
  if (g.out_dtype == DT_F32 && ((reinterpret_cast<uintptr_t>(g.D) & 7) || (g.ldd % 2))) {
    set_error("bv_gemm: fp32 output must be 8B aligned with an even ldd"); return BV_ERR_INVALID;
  }
  if (g.M > 0x7fffffffLL || g.N > 0x7fffffffLL || g.K > 0x7fffffffLL) {
    set_error("bv_gemm: dimension exceeds int32"); return BV_ERR_INVALID;
  }
  if (g.epilogue < BV_EPI_NONE || g.epilogue > BV_EPI_BIAS_GELU_ACT) {
    set_error("bv_gemm: bad epilogue %d", g.epilogue); return BV_ERR_INVALID;
  }
  if ((g.epilogue == BV_EPI_BIAS_RESID || g.epilogue == BV_EPI_DGELU) && g.aux == nullptr) {
    set_error("bv_gemm: epilogue %d needs aux", g.epilogue); return BV_ERR_INVALID;
  }
  if (g.aux != nullptr && ((reinterpret_cast<uintptr_t>(g.aux) & 15) || (g.ldaux % 8))) {
    set_error("bv_gemm: aux must be 16B aligned with ldaux %% 8 == 0"); return BV_ERR_INVALID;
  }
  if (g.bias != nullptr && (reinterpret_cast<uintptr_t>(g.bias) & 15)) {
    set_error("bv_gemm: bias must be 16B aligned"); return BV_ERR_INVALID;
  }
  if (g.epilogue == BV_EPI_BIAS_GELU && (g.out_dtype != DT_BF16 || g.D2 == nullptr || g.reduce_out)) {
    set_error("bv_gemm: BIAS_GELU needs bf16 output, D2 and no reduce"); return BV_ERR_INVALID;
  }
  if (g.epilogue == BV_EPI_BIAS_GELU && ((reinterpret_cast<uintptr_t>(g.D2) & 15) || (g.ldd2 % 8))) {
    set_error("bv_gemm: D2 must be 16B aligned with ldd2 %% 8 == 0"); return BV_ERR_INVALID;
  }
  if (g.epilogue == BV_EPI_BIAS_GELU_ACT && (g.out_dtype != DT_BF16 || g.reduce_out)) {
    set_error("bv_gemm: BIAS_GELU_ACT needs bf16 output and no reduce"); return BV_ERR_INVALID;
  }
  if (g.out_dtype != DT_F32 && g.out_dtype != DT_BF16) { set_error("bv_gemm: bad out dtype"); return BV_ERR_INVALID; }
  if (g.colsum != nullptr && (g.out_dtype != DT_BF16 || g.reduce_out)) {
    set_error("bv_gemm: colsum needs a plain bf16 output"); return BV_ERR_INVALID;
  }
  // The tile width picks the kernel's structure (Cfg): 128 ping-pongs, 256 is cooperative.  Ping-pong
  // hides each tile's epilogue under the other warpgroup's MMAs, but its 128 x 128 tiles bring a third
  // more operand bytes from L2 per FLOP than 128 x 256.  The fp32 outputs (split-K weight gradients,
  // K ~ 10^5 with a light register epilogue) lose more by that than they gain, so they run cooperative
  // at 256 (DESIGN §5); every bf16 output ping-pongs.  N <= 128 is one 128-wide tile.
  int bn = g.block_n;
  if (bn == 0) bn = (g.N > 128 && g.out_dtype == DT_F32) ? 256 : 128;
  if (bn == 256) return dispatch_epi<256>(g, s);
  if (bn == 128) return dispatch_epi<128>(g, s);
  set_error("bv_gemm: block_n must be 0, 128 or 256");
  return BV_ERR_INVALID;
}

}  // extern "C"
