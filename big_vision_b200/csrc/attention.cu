// Scaled-dot-product attention forward / backward on sm_90a wgmma (K5, and the MAP head's
// 1-query attention, K10).  Reference: flax.linen.MultiHeadDotProductAttention as called at
// models/vit.py:93-98 (self-attention, no mask, no dropout) and models/vit.py:176-178 (MAPHead
// probe attention): q is scaled by 1/sqrt(dh), softmax over keys, weights times v.  Head dims 64,
// 72, 80, 96 and 104 are built (the size table of models/vit.py:284-303: 64 for Ti, S, M, B and L,
// 72 for So400m, 80 for H, 96 for g-opt and G-opt, 104 for G); mu (16), g (88) and e (112) are not.
// Every kernel is a template on the head dim DH.
//
// q/k/v/o are strided views into the fused QKV GEMM output: element (b, t, h*DH+j) at
// base + b*batch_stride + t*row_stride + h*DH + j; TMA descriptors read them in place (no head
// transpose, no padding copies; rows past N are zero-filled).  At DH = 64 the map is 3-D
// [cols, tokens, batch] and a tile is one 64-column box.  At DH > 64 the head dim is a dimension of
// its own, [DH, H, tokens, batch], and a tile is two 128B-swizzled 64-column boxes side by side:
// columns 0-63 and 64-127, the second zero-filled by TMA past DH.  The contractions over the head
// dim (S = Q K^T, S^T = K Q^T, dP^T = V dO^T) run in k16 steps up to round_up(DH, 16) and so meet
// zeros, never the next head's columns.  The products whose N is the head dim (O += P V, dV, dK,
// dQ) are single n = DH wgmmas across both boxes (MN-major operand, leading byte offset = one box).
//
// Key-padding mask (dh = 64 only; head_dim | BV_ATTN_KEY_MASK, the mask appended to the arguments,
// include/bv_b200.h): an optional uint8 [B, Nk] row per batch, nonzero = attend.  The forward
// and the two backward kernels take it as a template flag MASK; without it they are the unmasked
// kernels unchanged.  A masked key takes the path of a key past Nk (score -inf in the forward, P = 0 in
// the backward), wherever it sits in its 64-key block.  A query whose keys are all masked gets O = 0,
// lse = 0 and zero gradients.
//
// Attention-probability dropout (key-masked dh = 64 only; head_dim | BV_ATTN_KEY_MASK | BV_ATTN_DROPOUT,
// include/bv_dropout.h): template flag DROP.  The mask is regenerated in each of the forward, dQ and dK / dV
// kernels from the Philox stream of the header, never stored.  A warp's 64 x 64 tile needs 64 Philox blocks
// (one per row and 16-key group); each lane draws two and turns them into 16-bit keep masks, and the lanes
// exchange those by shuffle (keep_rows, keep_cols).  The forward keeps l and lse of the undropped softmax,
// multiplies V by P o Z and divides O by l (1 - rate); the backward applies Z / (1 - rate) to dP (dQ, dK) and
// to P (dV).  Without DROP the kernels are unchanged.
//
// Every kernel runs one warpgroup per CTA on 64-row tiles and streams the other operand in 64-row
// blocks through a two-slot TMA ring, so any sequence length works with the same code:
//   forward   (b, h, 64 queries):  S = Q K^T (smem x smem), online softmax in registers,
//             O += P V with P as the register A operand of wgmma.
//   backward, after delta = rowsum(O o dO), two kernels that each own their outputs and sum over
//   the streamed blocks in a fixed order inside one wgmma accumulator (bit-reproducible, no
//   cross-CTA reduction, no workspace):
//     dQ      (b, h, 64 queries):  S = Q K^T, dP = dO V^T, P = exp(scale S - lse),
//             dS = P o (dP - delta), dQ += dS K with dS as the register A operand.
//     dK, dV  (b, h, 64 keys):     S^T = K Q^T, dP^T = V dO^T, P^T and dS^T in registers,
//             dV += P^T dO, dK += dS^T Q (register A operands).
//   S and dP are computed twice, once per kernel: 7 instead of 5 64 x 64 x DH products per tile
//   pair, which is cheaper than the HBM traffic of summing per-key-block dQ partials across CTAs.
#include "../../include/bv_dropout.h"

#include <math.h>

#include "common.cuh"
#include "host_utils.h"

namespace bv {

namespace {

constexpr int T = 64;                      // rows per tile (queries or keys)
constexpr int BOX_BYTES = T * 64 * 2;      // 8 KB: 64 rows x 128 B, 128B-swizzled
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;
constexpr int THREADS = 128;

// Per-head-dim geometry.  Shared memory: 1024-aligned tiles, then three mbarriers (+ alignment slack);
// the forward holds Q and two K / V slots, the dQ kernel Q, dO and two K / V slots, the dK / dV
// kernel K, V and two Q / dO slots.
template <int DH>
struct Geo {
  static_assert(DH == 64 || DH == 72 || DH == 80 || DH == 96 || DH == 104, "head dims 64, 72, 80, 96, 104");
  static constexpr int TILE_BYTES = DH > 64 ? 2 * BOX_BYTES : BOX_BYTES;   // a [64 rows x DH] tile
  static constexpr int KSTEPS = (DH + 15) / 16;                            // k16 steps over the head dim
  static_assert(KSTEPS >= 4 && KSTEPS <= 8, "one or two 64-column boxes");
  static constexpr int R = DH / 2;                                         // fp32 registers of a [64 x DH] accumulator
  static constexpr int FWD_SMEM = 5 * TILE_BYTES + 1024 + 64;
  static constexpr int BWD_SMEM = 6 * TILE_BYTES + 1024 + 64;
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

int make_tmap_bnd(CUtensorMap* m, const void* ptr, int dh, int H, int64_t N, int64_t B, int64_t ld, int64_t bs) {
  if (dh == 64) {
    uint64_t dims[3] = {static_cast<uint64_t>(H) * 64, static_cast<uint64_t>(N), static_cast<uint64_t>(B)};
    uint64_t strides[2] = {static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(bs) * 2};
    uint32_t box[3] = {64, T, 1};
    return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, ptr, dims, strides, box, true);
  }
  // [dh, H, N, B] with a head stride of dh * 2 bytes (a multiple of 16 since dh % 8 == 0)
  uint64_t dims[4] = {static_cast<uint64_t>(dh), static_cast<uint64_t>(H), static_cast<uint64_t>(N),
                      static_cast<uint64_t>(B)};
  uint64_t strides[3] = {static_cast<uint64_t>(dh) * 2, static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(bs) * 2};
  uint32_t box[4] = {64, 1, T, 1};
  return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, ptr, dims, strides, box, true);
}

// one [64 rows x DH] tile of head h from row `row` of batch b (TILE_BYTES transaction bytes)
template <int DH>
__device__ __forceinline__ void load_tile(uint32_t dst, const CUtensorMap* m, uint32_t bar, int h, int row, int b) {
  if constexpr (DH == 64) {
    tma_load_3d(dst, m, bar, h * DH, row, b);
  } else {
    tma_load_4d(dst, m, bar, 0, h, row, b);
    tma_load_4d(dst + BOX_BYTES, m, bar, 64, h, row, b);
  }
}

// Descriptors of a 64 x 64 bf16 box: K-major (rows = M|N, the 64 columns are the contraction) or
// MN-major (rows = the contraction, the 64 columns are M|N; the next 64 columns are the next box,
// 8 KB on).  One k step of 16 is 32 B or 16 rows.
__device__ __forceinline__ uint64_t desc_k(uint32_t tile) { return wgmma_desc_sw128(tile, 16u, 1024u); }
__device__ __forceinline__ uint64_t desc_mn(uint32_t tile) { return wgmma_desc_sw128(tile, 8192u, 1024u); }
constexpr uint64_t KSTEP_K = 32 >> 4, KSTEP_MN = 2048 >> 4;

// D[64 x DH] += A[64 x 16] (register fragment) * B[DH x 16]^T: the wgmma of N = DH
template <int TB, int R>
__device__ __forceinline__ void wgmma_rs_dh(float (&d)[R], const uint32_t (&a)[4], uint64_t b, int scale_d) {
  if constexpr (R == 32) wgmma_rs_n64<TB>(d, a, b, scale_d);
  else if constexpr (R == 36) wgmma_rs_n72<TB>(d, a, b, scale_d);
  else if constexpr (R == 40) wgmma_rs_n80<TB>(d, a, b, scale_d);
  else if constexpr (R == 48) wgmma_rs_n96<TB>(d, a, b, scale_d);
  else wgmma_rs_n104<TB>(d, a, b, scale_d);
}

// S[64 x 64] = A B^T over the head dimension (zero-padded to a multiple of 16), both tiles K-major
template <int DH>
__device__ __forceinline__ void mma_tile_kk(float (&d)[32], uint32_t a_tile, uint32_t b_tile) {
  const uint64_t a = desc_k(a_tile), b = desc_k(b_tile);
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_ss_n64<0, 0>(d, a + k * KSTEP_K, b + k * KSTEP_K, k > 0 ? 1 : 0);
  if constexpr (DH > 64) {
    const uint64_t a1 = desc_k(a_tile + BOX_BYTES), b1 = desc_k(b_tile + BOX_BYTES);
#pragma unroll
    for (int k = 0; k < Geo<DH>::KSTEPS - 4; ++k) wgmma_ss_n64<0, 0>(d, a1 + k * KSTEP_K, b1 + k * KSTEP_K, 1);
  }
}
// D[64 x DH] += P[64 x 64] (register fragments) * B, B an MN-major tile (rows = contraction)
template <int R>
__device__ __forceinline__ void mma_tile_rs(float (&d)[R], const uint32_t (&p)[4][4], uint32_t b_tile) {
  const uint64_t b = desc_mn(b_tile);
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_rs_dh<1>(d, p[k], b + k * KSTEP_MN, 1);
}

// accumulator element 4j + e of lane l in warp w: row 16w + l/4 + 8*(e >> 1), column 8j + 2*(l%4) + (e & 1).
// The register A fragment of k step kk (columns 16kk..16kk+15) is then {j = 2kk: e01, e23; j = 2kk+1: e01, e23}.
__device__ __forceinline__ void to_frags(const float (&s)[32], uint32_t (&p)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    p[kk][0] = pack_bf16(s[8 * kk + 0], s[8 * kk + 1]);
    p[kk][1] = pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
    p[kk][2] = pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
    p[kk][3] = pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
  }
}

template <int R>
__device__ __forceinline__ void zero(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) d[i] = 0.f;
}

// the attended keys of the 64-key block at k0, shifted to this thread's columns: bit 8c + e is key
// k0 + 8c + 2*(lane%4) + e, i.e. accumulator element 4c + e (and 4c + 2 + e) of the S = Q K^T tile.
// A key is attended when it is below Nk and its mask byte is nonzero.
__device__ __forceinline__ uint64_t attended_keys(const uint8_t* mask_row, int k0, int Nk, int lane) {
  const int a = k0 + lane, b = a + 32;
  const uint32_t lo = __ballot_sync(0xffffffffu, a < Nk && mask_row[a] != 0);
  const uint32_t hi = __ballot_sync(0xffffffffu, b < Nk && mask_row[b] != 0);
  return ((static_cast<uint64_t>(hi) << 32) | lo) >> (2 * (lane & 3));
}

// the attention dropout of a DROP kernel (include/bv_dropout.h)
struct DropDev {
  uint64_t seed, step, site;
  long long row0;                          // global row of (b, h, q) = (0, 0, 0)
  uint32_t thresh;                         // a probability is dropped when its 16-bit lane < thresh
  float keep, rkeep;                       // 1 - rate and 1 / (1 - rate), fp32
};

// keep bits of the 16 keys 16 kblk .. 16 kblk + 15 of global row `row`: bit t = key 16 kblk + t is kept
__device__ __forceinline__ uint32_t keep16(const DropDev& d, long long row, int kblk) {
  uint64_t w[4] = {static_cast<uint64_t>(kblk) + 1, d.step, d.site, static_cast<uint64_t>(row) + 1};
  philox4x64_10(w, d.seed, 0);
  uint32_t bits = 0;
#pragma unroll
  for (int t = 0; t < 16; ++t)
    bits |= static_cast<uint32_t>(((w[t >> 2] >> (16 * (t & 3))) & 0xffffu) >= d.thresh) << t;
  return bits;
}

// keep bits of this thread's 32 elements of a 64 x 64 tile whose rows are queries (S in the forward and the
// dQ kernel): bit i is element i, row `row` + 8 ((i >> 1) & 1), key 64 kb + 8 (i >> 2) + 2 (lane % 4) + (i & 1).
// Lane g of a quad draws key group g (16 keys) for the quad's two rows, and the quad shares them by shuffle.
__device__ __forceinline__ uint32_t keep_rows(const DropDev& d, long long row, int kb, int lane) {
  const int g = lane & 3;
  const uint32_t mine = keep16(d, row, 4 * kb + g) | (keep16(d, row + 8, 4 * kb + g) << 16);
  uint32_t keep = 0;
#pragma unroll
  for (int gg = 0; gg < 4; ++gg) {
    // bit 16 r + 8 h + e: key 16 gg + 8 h + 2 (lane % 4) + e of row r, i.e. element 8 gg + 4 h + 2 r + e
    const uint32_t m = __shfl_sync(0xffffffffu, mine, (lane & ~3) | gg) >> (2 * g);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int e = 0; e < 2; ++e) keep |= ((m >> (16 * r + 8 * h + e)) & 1u) << (8 * gg + 4 * h + 2 * r + e);
  }
  return keep;
}

// keep bits of this thread's 32 elements of a 64 x 64 tile whose rows are keys (S^T in the dK / dV kernel;
// the warp's 16 keys are the key group kblk): bit e is element e, key 16 kblk + lane / 4 + 8 ((e >> 1) & 1),
// query row0q + 8 (e >> 2) + 2 (lane % 4) + (e & 1).  Lane l draws queries l and l + 32, and each thread gathers
// its bits from the 8 lanes that drew its queries.
__device__ __forceinline__ uint32_t keep_cols(const DropDev& d, long long row0q, int kblk, int lane) {
  const uint32_t mine = keep16(d, row0q + lane, kblk) | (keep16(d, row0q + lane + 32, kblk) << 16);
  uint32_t keep = 0;
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      // bit 16 hi + 8 r: key lane / 4 + 8 r of query 8 (c + 4 hi) + 2 (lane % 4) + e
      const uint32_t m = __shfl_sync(0xffffffffu, mine, 8 * c + 2 * (lane & 3) + e) >> (lane >> 2);
#pragma unroll
      for (int hi = 0; hi < 2; ++hi)
#pragma unroll
        for (int r = 0; r < 2; ++r) keep |= ((m >> (16 * hi + 8 * r)) & 1u) << (4 * (c + 4 * hi) + 2 * r + e);
    }
  return keep;
}

// ============================================================================
// forward
// ============================================================================
struct FwdDev {
  int H, Nq, Nk, QT, NB;
  float scale_log2;
  float* lse;
  bf16* o;
  long long ldo, bso;
  const uint8_t* mask;                     // key mask [B, Nk] (MASK kernels only)
  long long bsmask;
  DropDev drop;                            // DROP kernels only
};

template <int DH, bool MASK, bool DROP>
__global__ void __launch_bounds__(THREADS)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const FwdDev p) {
  using G = Geo<DH>;
  constexpr int TILE_BYTES = G::TILE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t q_s = (smem_u32(smem_raw) + 1023u) & ~1023u, k_s = q_s + TILE_BYTES, v_s = q_s + 3 * TILE_BYTES;
  const uint32_t q_bar = q_s + 5 * TILE_BYTES;
  auto kv_bar = [&](int s) { return q_bar + 8u * (1 + s); };

  const int qt = static_cast<int>(blockIdx.x % p.QT);
  const int bh = static_cast<int>(blockIdx.x / p.QT);
  const int h = bh % p.H, b = bh / p.H;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  auto load_kv = [&](int j) {
    const int s = j & 1;
    mbar_expect_tx(kv_bar(s), 2 * TILE_BYTES);
    load_tile<DH>(k_s + s * TILE_BYTES, &tmK, kv_bar(s), h, j * T, b);
    load_tile<DH>(v_s + s * TILE_BYTES, &tmV, kv_bar(s), h, j * T, b);
  };
  if (tid == 0) {
    mbar_init(q_bar, 1);
    mbar_init(kv_bar(0), 1);
    mbar_init(kv_bar(1), 1);
    fence_barrier_init();
    mbar_expect_tx(q_bar, TILE_BYTES);
    load_tile<DH>(q_s, &tmQ, q_bar, h, qt * T, b);
    load_kv(0);
    if (p.NB > 1) load_kv(1);
  }
  __syncthreads();

  float o[G::R], s[32];
  zero(o);
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  // DROP: the global dropout row of this thread's first query
  const long long drow = DROP ? p.drop.row0 + static_cast<long long>(bh) * p.Nq + qt * T + 16 * warp + (lane >> 2) : 0;
  mbar_wait(q_bar, 0);
  for (int j = 0; j < p.NB; ++j) {
    const int slot = j & 1;
    mbar_wait(kv_bar(slot), (j >> 1) & 1);
    wgmma_fence();
    mma_tile_kk<DH>(s, q_s, k_s + slot * TILE_BYTES);
    wgmma_commit();
    uint32_t keep = 0;                   // drawn while the MMAs run
    if constexpr (DROP) keep = keep_rows(p.drop, drow, j, lane);
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    // online softmax in base 2 over this key block; keys past Nk (and masked keys) get probability 0
    const int kbase = j * T + 2 * (lane & 3);
    uint64_t live = 0;
    if constexpr (MASK) live = attended_keys(p.mask + b * p.bsmask, j * T, p.Nk, lane);
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int key = kbase + 8 * (i >> 2) + (i & 1);
      bool in;
      if constexpr (MASK) in = (live >> (8 * (i >> 2) + (i & 1))) & 1;
      else in = key < p.Nk;
      s[i] = in ? s[i] * p.scale_log2 : -INFINITY;
      mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
    }
    float corr[2], base[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      // with a mask, every key so far may be masked (mx = -inf): exponentiate against 0 instead, so
      // that the probabilities and the correction are 0, not NaN
      base[r] = MASK && mx[r] == -INFINITY ? 0.f : mx[r];
      corr[r] = ex2(m[r] - base[r]);     // 0 on the first block (m = -inf)
      m[r] = mx[r];
      l[r] *= corr[r];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = (i >> 1) & 1;
      s[i] = ex2(s[i] - (MASK ? base[r] : m[r]));
      l[r] += s[i];
      o[i] *= corr[r];
    }
#pragma unroll
    for (int i = 32; i < G::R; ++i) o[i] *= corr[(i >> 1) & 1];
    if constexpr (DROP) {                // l stays the undropped sum; P V takes P o Z
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = (keep >> i) & 1u ? s[i] : 0.f;
    }
    uint32_t pf[4][4];
    to_frags(s, pf);
    wgmma_fence_regs(o);
    wgmma_fence();
    mma_tile_rs(o, pf, v_s + slot * TILE_BYTES);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncthreads();                     // every warp is done with this slot
    if (tid == 0 && j + 2 < p.NB) load_kv(j + 2);
  }
  // normalise, store O (bf16) and the log-sum-exp (natural log of the scaled scores)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
  float inv[2] = {1.f / l[0], 1.f / l[1]};
  if constexpr (DROP) {                  // O = (P o Z) V / (l (1 - rate))
    inv[0] = 1.f / (l[0] * p.drop.keep);
    inv[1] = 1.f / (l[1] * p.drop.keep);
  }
  if constexpr (MASK) {                  // l = 0: no attended key, O = 0 and lse = 0
    inv[0] = l[0] > 0.f ? inv[0] : 0.f;
    inv[1] = l[1] > 0.f ? inv[1] : 0.f;
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = qt * T + 16 * warp + (lane >> 2) + 8 * r;
    if (q >= p.Nq) continue;
    bf16* orow = p.o + b * p.bso + static_cast<long long>(q) * p.ldo + h * DH + 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < DH / 8; ++jj)
      *reinterpret_cast<uint32_t*>(orow + 8 * jj) = pack_bf16(o[4 * jj + 2 * r] * inv[r], o[4 * jj + 2 * r + 1] * inv[r]);
    if ((lane & 3) == 0)
      p.lse[(static_cast<long long>(b) * p.H + h) * p.Nq + q] = MASK && l[r] == 0.f ? 0.f : (m[r] + __log2f(l[r])) * LN2;
  }
}

// ============================================================================
// backward
// ============================================================================
struct BwdDev {
  int H, Nq, Nk, QT, KT;
  float scale, scale_log2;
  const float* lse;
  const float* delta;
  bf16* dq; bf16* dk; bf16* dv;
  long long lddq, bsdq, lddk, bsdk, lddv, bsdv;
  float* dq_colsum; float* dk_colsum; float* dv_colsum;
  const uint8_t* mask;                     // key mask [B, Nk] (MASK kernels only)
  long long bsmask;
  DropDev drop;                            // DROP kernels only
};

// column sums of a [64 x DH] accumulator tile's stored (bf16-rounded) rows < nvalid: the eight lanes
// that share a column pair are summed with shuffles, then one atomic per warp and column
template <int R>
__device__ __forceinline__ void tile_colsum(const float (&d)[R], float mul, int row0, int nvalid, float* colsum,
                                            int lane) {
#pragma unroll
  for (int jj = 0; jj < R / 4; ++jj) {
    float c[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (row0 + 8 * r >= nvalid) continue;
      c[0] += round_bf16(d[4 * jj + 2 * r] * mul);
      c[1] += round_bf16(d[4 * jj + 2 * r + 1] * mul);
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      c[e] += __shfl_xor_sync(0xffffffffu, c[e], 4);
      c[e] += __shfl_xor_sync(0xffffffffu, c[e], 8);
      c[e] += __shfl_xor_sync(0xffffffffu, c[e], 16);
    }
    if (lane < 4) {
      atomicAdd(colsum + 8 * jj + 2 * lane, c[0]);
      atomicAdd(colsum + 8 * jj + 2 * lane + 1, c[1]);
    }
  }
}

// dQ of one (b, h, 64-query) block: the key blocks stream through the K / V ring and their dS K
// products accumulate in order in one register tile
template <int DH, bool MASK, bool DROP>
__global__ void __launch_bounds__(THREADS)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const BwdDev p) {
  using G = Geo<DH>;
  constexpr int TILE_BYTES = G::TILE_BYTES;
  // Q, dO (this CTA's query block), K / V ring of two
  extern __shared__ uint8_t smem_raw[];
  const uint32_t q_s = (smem_u32(smem_raw) + 1023u) & ~1023u, do_s = q_s + TILE_BYTES, k_s = q_s + 2 * TILE_BYTES,
                 v_s = q_s + 4 * TILE_BYTES;
  const uint32_t q_bar = q_s + 6 * TILE_BYTES;
  auto kv_bar = [&](int s) { return q_bar + 8u * (1 + s); };

  const int qt = static_cast<int>(blockIdx.x % p.QT);
  const int bh = static_cast<int>(blockIdx.x / p.QT);
  const int h = bh % p.H, b = bh / p.H;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  auto load_kv = [&](int j) {
    const int s = j & 1;
    mbar_expect_tx(kv_bar(s), 2 * TILE_BYTES);
    load_tile<DH>(k_s + s * TILE_BYTES, &tmK, kv_bar(s), h, j * T, b);
    load_tile<DH>(v_s + s * TILE_BYTES, &tmV, kv_bar(s), h, j * T, b);
  };
  if (tid == 0) {
    mbar_init(q_bar, 1);
    mbar_init(kv_bar(0), 1);
    mbar_init(kv_bar(1), 1);
    fence_barrier_init();
    mbar_expect_tx(q_bar, 2 * TILE_BYTES);
    load_tile<DH>(q_s, &tmQ, q_bar, h, qt * T, b);
    load_tile<DH>(do_s, &tmdO, q_bar, h, qt * T, b);
    load_kv(0);
    if (p.KT > 1) load_kv(1);
  }
  __syncthreads();

  float dq[G::R];
  zero(dq);
  // this thread's two queries (rows r = 0, 1): lse in base 2 and delta; +inf -> P = 0 past Nq
  const long long bhq = (static_cast<long long>(b) * p.H + h) * p.Nq;
  const int q0 = qt * T + 16 * warp + (lane >> 2);
  float lse2[2], dl[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + 8 * r;
    lse2[r] = q < p.Nq ? p.lse[bhq + q] * LOG2E : INFINITY;
    dl[r] = q < p.Nq ? p.delta[bhq + q] : 0.f;
  }
  const long long drow = DROP ? p.drop.row0 + bhq + q0 : 0;   // DROP: global dropout row of query q0
  mbar_wait(q_bar, 0);
  for (int j = 0; j < p.KT; ++j) {
    const int slot = j & 1;
    mbar_wait(kv_bar(slot), (j >> 1) & 1);
    const uint32_t kj = k_s + slot * TILE_BYTES, vj = v_s + slot * TILE_BYTES;
    float s[32], dp[32];
    wgmma_fence();
    mma_tile_kk<DH>(s, q_s, kj);          // S  = Q K^T
    mma_tile_kk<DH>(dp, do_s, vj);        // dP = dO V^T
    wgmma_commit();
    uint32_t keep = 0;                    // drawn while the MMAs run
    if constexpr (DROP) keep = keep_rows(p.drop, drow, j, lane);
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    wgmma_fence_regs(dp);
    // P = exp(scale S - lse), dS = P o (dP - delta); keys past Nk (zero-filled K rows) and masked keys
    // get P = 0
    const int kbase = j * T + 2 * (lane & 3);
    uint64_t live = 0;
    if constexpr (MASK) live = attended_keys(p.mask + b * p.bsmask, j * T, p.Nk, lane);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = (i >> 1) & 1;
      const int key = kbase + 8 * (i >> 2) + (i & 1);
      bool in;
      if constexpr (MASK) in = (live >> (8 * (i >> 2) + (i & 1))) & 1;
      else in = key < p.Nk;
      const float pr = in ? ex2(s[i] * p.scale_log2 - lse2[r]) : 0.f;
      if constexpr (DROP) dp[i] = (keep >> i) & 1u ? dp[i] * p.drop.rkeep : 0.f;   // Z o dP / (1 - rate)
      dp[i] = pr * (dp[i] - dl[r]);
    }
    uint32_t sf[4][4];
    to_frags(dp, sf);
    wgmma_fence_regs(dq);
    wgmma_fence();
    mma_tile_rs(dq, sf, kj);              // dQ += dS K
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dq);
    __syncthreads();                      // every warp is done with this slot
    if (tid == 0 && j + 2 < p.KT) load_kv(j + 2);
  }
  // dQ (scaled) for the queries of this block, and its fused column sum
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + 8 * r;
    if (q >= p.Nq) continue;
    bf16* qr = p.dq + b * p.bsdq + static_cast<long long>(q) * p.lddq + h * DH + 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < DH / 8; ++jj)
      *reinterpret_cast<uint32_t*>(qr + 8 * jj) = pack_bf16(dq[4 * jj + 2 * r] * p.scale, dq[4 * jj + 2 * r + 1] * p.scale);
  }
  if (p.dq_colsum != nullptr) tile_colsum(dq, p.scale, q0, p.Nq, p.dq_colsum + h * DH, lane);
}

// dK, dV of one (b, h, 64-key) block: the query blocks stream through the Q / dO ring
template <int DH, bool MASK, bool DROP>
__global__ void __launch_bounds__(THREADS)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const BwdDev p) {
  using G = Geo<DH>;
  constexpr int TILE_BYTES = G::TILE_BYTES;
  // K, V (this CTA's key block), Q / dO ring of two
  extern __shared__ uint8_t smem_raw[];
  const uint32_t k_s = (smem_u32(smem_raw) + 1023u) & ~1023u, v_s = k_s + TILE_BYTES, q_s = k_s + 2 * TILE_BYTES,
                 do_s = k_s + 4 * TILE_BYTES;
  const uint32_t kv_bar = k_s + 6 * TILE_BYTES;
  auto q_bar = [&](int s) { return kv_bar + 8u * (1 + s); };

  const int kt = static_cast<int>(blockIdx.x % p.KT);
  const int bh = static_cast<int>(blockIdx.x / p.KT);
  const int h = bh % p.H, b = bh / p.H;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  auto load_q = [&](int i) {
    const int s = i & 1;
    mbar_expect_tx(q_bar(s), 2 * TILE_BYTES);
    load_tile<DH>(q_s + s * TILE_BYTES, &tmQ, q_bar(s), h, i * T, b);
    load_tile<DH>(do_s + s * TILE_BYTES, &tmdO, q_bar(s), h, i * T, b);
  };
  if (tid == 0) {
    mbar_init(kv_bar, 1);
    mbar_init(q_bar(0), 1);
    mbar_init(q_bar(1), 1);
    fence_barrier_init();
    mbar_expect_tx(kv_bar, 2 * TILE_BYTES);
    load_tile<DH>(k_s, &tmK, kv_bar, h, kt * T, b);
    load_tile<DH>(v_s, &tmV, kv_bar, h, kt * T, b);
    load_q(0);
    if (p.QT > 1) load_q(1);
  }
  __syncthreads();

  float dk[G::R], dv[G::R];
  zero(dk);
  zero(dv);
  const long long bhq = (static_cast<long long>(b) * p.H + h) * p.Nq;
  const int key_row = 16 * warp + (lane >> 2);      // + 8r: this thread's rows of the key block
  bool live[2] = {true, true};                      // its two keys are attended (MASK)
  if constexpr (MASK) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int key = kt * T + key_row + 8 * r;
      live[r] = key < p.Nk && p.mask[b * p.bsmask + key] != 0;
    }
  }
  mbar_wait(kv_bar, 0);
  for (int i = 0; i < p.QT; ++i) {
    const int slot = i & 1;
    mbar_wait(q_bar(slot), (i >> 1) & 1);
    const uint32_t qi = q_s + slot * TILE_BYTES, doi = do_s + slot * TILE_BYTES;
    float st[32], dpt[32];
    wgmma_fence();
    mma_tile_kk<DH>(st, k_s, qi);        // S^T  = K Q^T
    mma_tile_kk<DH>(dpt, v_s, doi);      // dP^T = V dO^T
    wgmma_commit();
    // this thread's 16 queries: lse / delta, fetched while the MMAs run
    float lse2[16], dl[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const int q = i * T + 8 * (c >> 1) + 2 * (lane & 3) + (c & 1);
      lse2[c] = q < p.Nq ? p.lse[bhq + q] * LOG2E : INFINITY;   // +inf -> P = 0 for queries past Nq
      dl[c] = q < p.Nq ? p.delta[bhq + q] : 0.f;
    }
    uint32_t keep = 0;
    if constexpr (DROP) keep = keep_cols(p.drop, p.drop.row0 + bhq + i * T, 4 * kt + warp, lane);
    wgmma_wait<0>();
    wgmma_fence_regs(st);
    wgmma_fence_regs(dpt);
    // P^T = exp(scale S^T - lse), dS^T = P^T o (dP^T - delta)   (the scale of dS is applied at the end);
    // a masked key's row of P^T is 0
#pragma unroll
    for (int e = 0; e < 32; ++e) {
      const int c = 2 * (e >> 2) + (e & 1);
      st[e] = ex2(st[e] * p.scale_log2 - lse2[c]);
      if constexpr (MASK) st[e] = live[(e >> 1) & 1] ? st[e] : 0.f;
      if constexpr (DROP) {              // dS^T from Z o dP^T / (1 - rate); dV from Z o P^T / (1 - rate)
        const bool kept = (keep >> e) & 1u;
        dpt[e] = st[e] * ((kept ? dpt[e] * p.drop.rkeep : 0.f) - dl[c]);
        st[e] = kept ? st[e] * p.drop.rkeep : 0.f;
      } else {
        dpt[e] = st[e] * (dpt[e] - dl[c]);
      }
    }
    uint32_t pf[4][4], sf[4][4];
    to_frags(st, pf);
    to_frags(dpt, sf);
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    wgmma_fence();
    mma_tile_rs(dv, pf, doi);            // dV += P^T dO
    mma_tile_rs(dk, sf, qi);             // dK += dS^T Q
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    __syncthreads();                     // every warp is done with this Q / dO slot
    if (tid == 0 && i + 2 < p.QT) load_q(i + 2);
  }
  // dK (scaled), dV for the keys of this block, and their fused column sums
  const int k0 = kt * T + key_row;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = k0 + 8 * r;
    if (key >= p.Nk) continue;
    bf16* kr = p.dk + b * p.bsdk + static_cast<long long>(key) * p.lddk + h * DH + 2 * (lane & 3);
    bf16* vr = p.dv + b * p.bsdv + static_cast<long long>(key) * p.lddv + h * DH + 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < DH / 8; ++jj) {
      *reinterpret_cast<uint32_t*>(kr + 8 * jj) = pack_bf16(dk[4 * jj + 2 * r] * p.scale, dk[4 * jj + 2 * r + 1] * p.scale);
      *reinterpret_cast<uint32_t*>(vr + 8 * jj) = pack_bf16(dv[4 * jj + 2 * r], dv[4 * jj + 2 * r + 1]);
    }
  }
  if (p.dk_colsum != nullptr) tile_colsum(dk, p.scale, k0, p.Nk, p.dk_colsum + h * DH, lane);
  if (p.dv_colsum != nullptr) tile_colsum(dv, 1.f, k0, p.Nk, p.dv_colsum + h * DH, lane);
}

// delta[b,h,t] = sum_j O[b,t,h*DH+j] * dO[b,t,h*DH+j]: LANES lanes per (b, t, h) row, DH/8 of which load
// eight columns each (8 lanes at DH = 64, 16 above)
template <int DH>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ d_o, float* __restrict__ delta,
                  int64_t B, int H, int N, int64_t ldo, int64_t bso, int64_t lddo, int64_t bsdo) {
  constexpr int LOG2_LANES = DH == 64 ? 3 : 4, LANES = 1 << LOG2_LANES;
  const int64_t total = B * N * H;                    // head rows
  const int chunk = threadIdx.x & (LANES - 1);
  for (int64_t r = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> LOG2_LANES; r < total;
       r += (static_cast<int64_t>(gridDim.x) * blockDim.x) >> LOG2_LANES) {
    const int h = static_cast<int>(r % H);
    const int64_t bt = r / H;
    const int t = static_cast<int>(bt % N);
    const int64_t b = bt / N;
    float acc = 0.f;
    if (chunk < DH / 8) {
      const uint4 ao = ld_nc_na(reinterpret_cast<const uint4*>(o + b * bso + t * ldo + h * DH + chunk * 8));
      const uint4 ad = ld_nc_na(reinterpret_cast<const uint4*>(d_o + b * bsdo + t * lddo + h * DH + chunk * 8));
      acc = bf16_lo(ao.x) * bf16_lo(ad.x) + bf16_hi(ao.x) * bf16_hi(ad.x);
      acc += bf16_lo(ao.y) * bf16_lo(ad.y) + bf16_hi(ao.y) * bf16_hi(ad.y);
      acc += bf16_lo(ao.z) * bf16_lo(ad.z) + bf16_hi(ao.z) * bf16_hi(ad.z);
      acc += bf16_lo(ao.w) * bf16_lo(ad.w) + bf16_hi(ao.w) * bf16_hi(ad.w);
    }
#pragma unroll
    for (int off = 1; off < LANES; off <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (chunk == 0) delta[(b * H + h) * N + t] = acc;
  }
}

// the key mask of a call: head_dim | BV_ATTN_KEY_MASK means the arguments are followed by it
struct KeyMask {
  const uint8_t* mask = nullptr;
  int64_t bs = 0;
};

// the attention dropout of a call: head_dim | BV_ATTN_DROPOUT means the masked arguments are followed by a
// bv_dropout_key
struct AttnDrop {
  bool on = false;
  DropDev dev{};
};

// the dropout flag is accepted with the key mask at head dim 64 only, with a key that bv_dropout would accept
int check_drop(bool dropped, bool masked, int head_dim, const bv_dropout_key& k, AttnDrop* d, const char* who) {
  if (!dropped) return BV_OK;
  if (!masked) {
    set_error("%s: BV_ATTN_DROPOUT needs BV_ATTN_KEY_MASK", who);
    return BV_ERR_INVALID;
  }
  if (head_dim != 64) {
    set_error("%s: BV_ATTN_DROPOUT is supported at head_dim 64 only (got %d)", who, head_dim);
    return BV_ERR_INVALID;
  }
  if (!(k.rate >= 0.f && k.rate < 1.f)) {
    set_error("%s: dropout rate %g outside [0, 1)", who, static_cast<double>(k.rate));
    return BV_ERR_INVALID;
  }
  if (k.site == 0) {
    set_error("%s: dropout site 0 is Jet's noise stream; dropout sites start at 1", who);
    return BV_ERR_INVALID;
  }
  if (k.row0 < 0) {
    set_error("%s: dropout row0 must be >= 0 (got %lld)", who, static_cast<long long>(k.row0));
    return BV_ERR_INVALID;
  }
  d->on = true;
  d->dev.seed = k.seed;
  d->dev.step = k.step;
  d->dev.site = k.site;
  d->dev.row0 = k.row0;
  d->dev.thresh = static_cast<uint32_t>(nearbyint(static_cast<double>(k.rate) * 65536.0));
  d->dev.keep = 1.f - k.rate;
  d->dev.rkeep = 1.f / d->dev.keep;
  return BV_OK;
}

// head dims with kernels; every other one is refused before any CUDA call.  The key mask is built at
// head dim 64 only (BERT-Base and BERT-Large)
int check_head_dim(int head_dim, bool masked, const KeyMask& m, const char* who) {
  if (head_dim != 64 && head_dim != 72 && head_dim != 80 && head_dim != 96 && head_dim != 104) {
    set_error("%s: head_dim %d is not supported (supported head dims: 64, 72, 80, 96, 104)", who, head_dim);
    return BV_ERR_UNSUPPORTED;
  }
  if (masked && head_dim != 64) {
    set_error("%s: a key mask is supported at head_dim 64 only (got %d)", who, head_dim);
    return BV_ERR_INVALID;
  }
  if (masked && m.mask == nullptr) {
    set_error("%s: BV_ATTN_KEY_MASK needs a non-null key_mask", who);
    return BV_ERR_INVALID;
  }
  return BV_OK;
}

int check_attn(const bv_attn_args& a, const char* who) {
  if (a.B <= 0 || a.H <= 0 || a.Nq <= 0 || a.Nk <= 0 || a.Nq > 65536 || a.Nk > 65536) {
    set_error("%s: need 1 <= Nq,Nk <= 65536 and B,H >= 1 (got B=%lld H=%d Nq=%d Nk=%d)", who,
              (long long)a.B, a.H, a.Nq, a.Nk);
    return BV_ERR_INVALID;
  }
  const int64_t tiles = ((a.Nq > a.Nk ? a.Nq : a.Nk) + T - 1) / T;
  if (a.B * a.H * tiles > 0x7fffffffLL) {
    set_error("%s: too many (batch, head, tile) work units", who);
    return BV_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(a.o) & 15) || (a.ldo % 8) || (a.bso % 8)) {
    set_error("%s: o must be 16B aligned with strides that are multiples of 8", who);
    return BV_ERR_INVALID;
  }
  return BV_OK;
}

template <int DH>
int attention_fwd(const bv_attn_args& a, const KeyMask& km, const AttnDrop& dr, cudaStream_t s) {
  using G = Geo<DH>;
  int rc = check_attn(a, "bv_attention_fwd_hd");
  if (rc) return rc;
  FwdDev p;
  p.H = a.H; p.Nq = a.Nq; p.Nk = a.Nk;
  p.QT = (a.Nq + T - 1) / T;
  p.NB = (a.Nk + T - 1) / T;
  p.scale_log2 = a.scale * LOG2E;
  p.lse = a.lse;
  p.o = static_cast<bf16*>(a.o);
  p.ldo = a.ldo; p.bso = a.bso;
  p.mask = km.mask; p.bsmask = km.bs;
  p.drop = dr.dev;
  CUtensorMap tmQ, tmK, tmV;
  if ((rc = make_tmap_bnd(&tmQ, a.q, DH, a.H, a.Nq, a.B, a.ldq, a.bsq))) return rc;
  if ((rc = make_tmap_bnd(&tmK, a.k, DH, a.H, a.Nk, a.B, a.ldk, a.bsk))) return rc;
  if ((rc = make_tmap_bnd(&tmV, a.v, DH, a.H, a.Nk, a.B, a.ldv, a.bsv))) return rc;
  const long long grid = a.B * a.H * p.QT;
  auto kernel = attn_fwd_kernel<DH, false, false>;
  if constexpr (DH == 64) {
    if (km.mask != nullptr) kernel = dr.on ? attn_fwd_kernel<DH, true, true> : attn_fwd_kernel<DH, true, false>;
  }
  rc = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G::FWD_SMEM),
                  "cudaFuncSetAttribute(attn_fwd)");
  if (rc) return rc;
  kernel<<<static_cast<unsigned>(grid), THREADS, G::FWD_SMEM, s>>>(tmQ, tmK, tmV, p);
  return check_cuda(cudaGetLastError(), "attn_fwd_kernel launch");
}

template <int DH>
int attention_bwd(const bv_attn_bwd_args& g, const KeyMask& km, const AttnDrop& dr, cudaStream_t s) {
  using G = Geo<DH>;
  const bv_attn_args& a = g.fwd;
  int rc = check_attn(a, "bv_attention_bwd_hd");
  if (rc) return rc;
  if (a.lse == nullptr) { set_error("bv_attention_bwd_hd: lse required"); return BV_ERR_INVALID; }
  if (g.delta == nullptr) {
    set_error("bv_attention_bwd_hd: needs the delta [B,H,Nq] fp32 workspace");
    return BV_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(g.d_o) & 15) || (g.lddo % 8) || (g.bsdo % 8)) {
    set_error("bv_attention_bwd_hd: d_o must be 16B aligned with strides that are multiples of 8");
    return BV_ERR_INVALID;
  }
  const void* grads[3] = {g.dq, g.dk, g.dv};
  const int64_t lds[3] = {g.lddq, g.lddk, g.lddv}, bss[3] = {g.bsdq, g.bsdk, g.bsdv};
  for (int i = 0; i < 3; ++i) {
    if (grads[i] == nullptr || (reinterpret_cast<uintptr_t>(grads[i]) & 15) || (lds[i] % 8) || (bss[i] % 8)) {
      set_error("bv_attention_bwd_hd: dq / dk / dv must be non-null, 16B aligned, with strides that are multiples "
                "of 8");
      return BV_ERR_INVALID;
    }
  }
  // delta = rowsum(O o dO)
  {
    constexpr int lanes = DH == 64 ? 8 : 16;
    const int64_t head_rows = a.B * a.Nq * a.H;
    int64_t blocks = (head_rows * lanes + 255) / 256;
    const int64_t cap = static_cast<int64_t>(num_sms()) * 16;
    if (blocks > cap) blocks = cap;
    attn_delta_kernel<DH><<<static_cast<unsigned>(blocks), 256, 0, s>>>(
        reinterpret_cast<const bf16*>(a.o), reinterpret_cast<const bf16*>(g.d_o), g.delta, a.B, a.H, a.Nq,
        a.ldo, a.bso, g.lddo, g.bsdo);
    if ((rc = check_cuda(cudaGetLastError(), "attn_delta_kernel launch"))) return rc;
  }
  BwdDev p;
  p.H = a.H; p.Nq = a.Nq; p.Nk = a.Nk;
  p.QT = (a.Nq + T - 1) / T;
  p.KT = (a.Nk + T - 1) / T;
  p.scale = a.scale;
  p.scale_log2 = a.scale * LOG2E;
  p.lse = a.lse;
  p.delta = g.delta;
  p.dq = static_cast<bf16*>(g.dq); p.dk = static_cast<bf16*>(g.dk); p.dv = static_cast<bf16*>(g.dv);
  p.lddq = g.lddq; p.bsdq = g.bsdq; p.lddk = g.lddk; p.bsdk = g.bsdk; p.lddv = g.lddv; p.bsdv = g.bsdv;
  p.dq_colsum = g.dq_colsum; p.dk_colsum = g.dk_colsum; p.dv_colsum = g.dv_colsum;
  p.mask = km.mask; p.bsmask = km.bs;
  p.drop = dr.dev;
  CUtensorMap tmQ, tmK, tmV, tmdO;
  if ((rc = make_tmap_bnd(&tmQ, a.q, DH, a.H, a.Nq, a.B, a.ldq, a.bsq))) return rc;
  if ((rc = make_tmap_bnd(&tmK, a.k, DH, a.H, a.Nk, a.B, a.ldk, a.bsk))) return rc;
  if ((rc = make_tmap_bnd(&tmV, a.v, DH, a.H, a.Nk, a.B, a.ldv, a.bsv))) return rc;
  if ((rc = make_tmap_bnd(&tmdO, g.d_o, DH, a.H, a.Nq, a.B, g.lddo, g.bsdo))) return rc;
  // query blocks of one (b, h) are adjacent in the dQ grid (and key blocks in the dK / dV grid), so the
  // streamed K / V (Q / dO) tiles they share are served from L2
  auto dq_kernel = attn_bwd_dq_kernel<DH, false, false>;
  auto dkdv_kernel = attn_bwd_dkdv_kernel<DH, false, false>;
  if constexpr (DH == 64) {
    if (km.mask != nullptr && dr.on) {
      dq_kernel = attn_bwd_dq_kernel<DH, true, true>;
      dkdv_kernel = attn_bwd_dkdv_kernel<DH, true, true>;
    } else if (km.mask != nullptr) {
      dq_kernel = attn_bwd_dq_kernel<DH, true, false>;
      dkdv_kernel = attn_bwd_dkdv_kernel<DH, true, false>;
    }
  }
  rc = check_cuda(cudaFuncSetAttribute(dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G::BWD_SMEM),
                  "cudaFuncSetAttribute(attn_bwd_dq)");
  if (rc) return rc;
  dq_kernel<<<static_cast<unsigned>(a.B * a.H * p.QT), THREADS, G::BWD_SMEM, s>>>(tmQ, tmK, tmV, tmdO, p);
  if ((rc = check_cuda(cudaGetLastError(), "attn_bwd_dq_kernel launch"))) return rc;
  rc = check_cuda(cudaFuncSetAttribute(dkdv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G::BWD_SMEM),
                  "cudaFuncSetAttribute(attn_bwd_dkdv)");
  if (rc) return rc;
  dkdv_kernel<<<static_cast<unsigned>(a.B * a.H * p.KT), THREADS, G::BWD_SMEM, s>>>(tmQ, tmK, tmV, tmdO, p);
  rc = check_cuda(cudaGetLastError(), "attn_bwd_dkdv_kernel launch");
  return rc;
}

}  // namespace
}  // namespace bv

extern "C" {

int bv_attention_fwd_hd(const bv_attn_args* args, int32_t head_dim, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!args) { set_error("bv_attention_fwd_hd: null args"); return BV_ERR_INVALID; }
  const bool masked = (head_dim & BV_ATTN_KEY_MASK) != 0, dropped = (head_dim & BV_ATTN_DROPOUT) != 0;
  head_dim &= ~(BV_ATTN_KEY_MASK | BV_ATTN_DROPOUT);
  KeyMask km;
  if (masked) {     // args is the first member of a bv_attn_masked_args
    const bv_attn_masked_args* m = reinterpret_cast<const bv_attn_masked_args*>(args);
    km.mask = m->key_mask;
    km.bs = m->bsmask;
  }
  AttnDrop dr;      // with the dropout flag, that is the first member of a bv_attn_dropout_args
  int rc = check_drop(dropped, masked, head_dim,
                      dropped ? reinterpret_cast<const bv_attn_dropout_args*>(args)->drop : bv_dropout_key{}, &dr,
                      "bv_attention_fwd_hd");
  if (rc) return rc;
  rc = check_head_dim(head_dim, masked, km, "bv_attention_fwd_hd");
  if (rc) return rc;
  const bv_attn_args& a = *args;
  switch (head_dim) {
    case 72: return attention_fwd<72>(a, km, dr, s);
    case 80: return attention_fwd<80>(a, km, dr, s);
    case 96: return attention_fwd<96>(a, km, dr, s);
    case 104: return attention_fwd<104>(a, km, dr, s);
    default: return attention_fwd<64>(a, km, dr, s);
  }
}

int bv_attention_bwd_hd(const bv_attn_bwd_args* args, int32_t head_dim, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!args) { set_error("bv_attention_bwd_hd: null args"); return BV_ERR_INVALID; }
  const bool masked = (head_dim & BV_ATTN_KEY_MASK) != 0, dropped = (head_dim & BV_ATTN_DROPOUT) != 0;
  head_dim &= ~(BV_ATTN_KEY_MASK | BV_ATTN_DROPOUT);
  KeyMask km;
  if (masked) {     // args is the first member of a bv_attn_masked_bwd_args
    const bv_attn_masked_bwd_args* m = reinterpret_cast<const bv_attn_masked_bwd_args*>(args);
    km.mask = m->key_mask;
    km.bs = m->bsmask;
  }
  AttnDrop dr;      // with the dropout flag, that is the first member of a bv_attn_dropout_bwd_args
  int rc = check_drop(dropped, masked, head_dim,
                      dropped ? reinterpret_cast<const bv_attn_dropout_bwd_args*>(args)->drop : bv_dropout_key{}, &dr,
                      "bv_attention_bwd_hd");
  if (rc) return rc;
  rc = check_head_dim(head_dim, masked, km, "bv_attention_bwd_hd");
  if (rc) return rc;
  const bv_attn_bwd_args& g = *args;
  switch (head_dim) {
    case 72: return attention_bwd<72>(g, km, dr, s);
    case 80: return attention_bwd<80>(g, km, dr, s);
    case 96: return attention_bwd<96>(g, km, dr, s);
    case 104: return attention_bwd<104>(g, km, dr, s);
    default: return attention_bwd<64>(g, km, dr, s);
  }
}

}  // extern "C"
