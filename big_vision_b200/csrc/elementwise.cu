// HBM-bound helpers around the GEMM/attention kernels: patch extraction (K1's
// im2col), token embedding gather / scatter-add (K12), L2 normalisation (K13),
// pooling (K10), column sums (bias gradients), casts and small element-wise maps.
// Every kernel streams its operands once with 16-byte accesses where layout allows.
#include "common.cuh"
#include "host_utils.h"

namespace bv {
namespace {

__device__ __forceinline__ float ld_as_float(const void* p, int dt, int64_t i) {
  return dt == DT_BF16 ? __bfloat162float(reinterpret_cast<const bf16*>(p)[i])
                       : reinterpret_cast<const float*>(p)[i];
}
__device__ __forceinline__ void st_from_float(void* p, int dt, int64_t i, float v) {
  if (dt == DT_BF16) reinterpret_cast<bf16*>(p)[i] = __float2bfloat16_rn(v);
  else reinterpret_cast<float*>(p)[i] = v;
}

// ---------------------------------------------------------------------------
// patchify: image [n,H,W,C] fp32 (NHWC) -> patches [n*(H/P)*(W/P), Kp] bf16 with
// column order (ph, pw, c), the row-major flattening of the HWIO conv kernel
// (models/vit.py:212-214, nn.Conv(width, patch, strides=patch, padding="VALID")).
// Kp = round_up(P*P*C, 8); pad columns are zero.
// ---------------------------------------------------------------------------
__global__ void patchify_kernel(const float* __restrict__ img, bf16* __restrict__ out, int64_t n,
                                int H, int W, int C, int P, int Kp) {
  const int gh = H / P, gw = W / P;
  const int K = P * P * C, PC = P * C;
  const int groups = Kp / 8;
  const int64_t total = n * gh * gw * groups;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(idx % groups);
    const int64_t patch = idx / groups;
    const int px = static_cast<int>(patch % gw);
    const int py = static_cast<int>((patch / gw) % gh);
    const int64_t b = patch / (static_cast<int64_t>(gw) * gh);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = g * 8 + j;
      if (k < K) {
        const int ph = k / PC, o = k % PC;
        v[j] = __ldg(img + ((b * H + (py * P + ph)) * static_cast<int64_t>(W) + px * P) * C + o);
      } else {
        v[j] = 0.f;
      }
    }
    uint4 q;
    q.x = pack_bf16(v[0], v[1]); q.y = pack_bf16(v[2], v[3]);
    q.z = pack_bf16(v[4], v[5]); q.w = pack_bf16(v[6], v[7]);
    *reinterpret_cast<uint4*>(out + patch * Kp + g * 8) = q;
  }
}

// uint8 ingest: the same patch extraction straight from the decoded uint8 image, with the input
// pipeline's `value_range(vmin, vmax, in_min, in_max, clip)` (pp/ops_general.py:32-64) applied on
// the way -- fp32, every operation rounded separately like the TensorFlow op:
//   x = (float(u8) - in_min) / (in_max - in_min);  y = vmin + x * (vmax - vmin);  [clip to vmin..vmax]
// A quarter of the host->device bytes of the fp32 hand-off (input_pipeline.py:316-329 ships the
// already-converted fp32 image).  One thread per 8 output columns, as above.
__global__ void patchify_u8_kernel(const uint8_t* __restrict__ img, bf16* __restrict__ out, int64_t n,
                                   int H, int W, int C, int P, int Kp, float vmin, float vrange,
                                   float in_min, float in_span, int clip, float vmax) {
  const int gh = H / P, gw = W / P;
  const int K = P * P * C, PC = P * C;
  const int groups = Kp / 8;
  const int64_t total = n * gh * gw * groups;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(idx % groups);
    const int64_t patch = idx / groups;
    const int px = static_cast<int>(patch % gw);
    const int py = static_cast<int>((patch / gw) % gh);
    const int64_t b = patch / (static_cast<int64_t>(gw) * gh);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = g * 8 + j;
      if (k < K) {
        const int ph = k / PC, o = k % PC;
        const float x = static_cast<float>(
            __ldg(img + ((b * H + (py * P + ph)) * static_cast<int64_t>(W) + px * P) * C + o));
        float y = __fadd_rn(vmin, __fmul_rn(__fdiv_rn(__fsub_rn(x, in_min), in_span), vrange));
        if (clip) y = fminf(fmaxf(y, vmin), vmax);
        v[j] = y;
      } else {
        v[j] = 0.f;
      }
    }
    uint4 q;
    q.x = pack_bf16(v[0], v[1]); q.y = pack_bf16(v[2], v[3]);
    q.z = pack_bf16(v[4], v[5]); q.w = pack_bf16(v[6], v[7]);
    *reinterpret_cast<uint4*>(out + patch * Kp + g * 8) = q;
  }
}

// ---------------------------------------------------------------------------
// token embedding: out[b,l,:] = table[ids[b,l],:] + pos[l,:]
// (models/proj/image_text/text_transformer.py:63-70)
// ---------------------------------------------------------------------------
__global__ void embed_fwd_kernel(const int32_t* __restrict__ ids, const float* __restrict__ table,
                                 const float* __restrict__ pos, void* __restrict__ out, int out_dt,
                                 int64_t n, int L, int d, int vocab) {
  const int groups = d / 4;
  const int64_t total = n * L * groups;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(idx % groups);
    const int64_t tok = idx / groups;
    const int l = static_cast<int>(tok % L);
    int id = ids[tok];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const float4 e = __ldg(reinterpret_cast<const float4*>(table + static_cast<int64_t>(id) * d) + g);
    float4 pe = make_float4(0.f, 0.f, 0.f, 0.f);
    if (pos != nullptr) pe = __ldg(reinterpret_cast<const float4*>(pos + static_cast<int64_t>(l) * d) + g);
    const float a = e.x + pe.x, b = e.y + pe.y, c = e.z + pe.z, dd = e.w + pe.w;
    if (out_dt == DT_BF16) {
      uint2 q;
      q.x = pack_bf16(a, b); q.y = pack_bf16(c, dd);
      *reinterpret_cast<uint2*>(reinterpret_cast<bf16*>(out) + tok * d + g * 4) = q;
    } else {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + tok * d + g * 4) = make_float4(a, b, c, dd);
    }
  }
}

// dtable[ids[b,l],:] += dy[b,l,:]   (scatter-add; duplicates resolved by fp32 atomics)
__global__ void embed_bwd_table_kernel(const int32_t* __restrict__ ids, const void* __restrict__ dy,
                                       int dy_dt, float* __restrict__ dtable, int64_t n, int L,
                                       int d, int vocab) {
  const int64_t total = n * L * d;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % d);
    const int64_t tok = idx / d;
    int id = ids[tok];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    atomicAdd(dtable + static_cast<int64_t>(id) * d + c, ld_as_float(dy, dy_dt, idx));
  }
}
// dpos[l,c] += sum_b dy[b,l,c]
__global__ void embed_bwd_pos_kernel(const void* __restrict__ dy, int dy_dt,
                                     float* __restrict__ dpos, int64_t n, int L, int d) {
  const int64_t total = static_cast<int64_t>(L) * d;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float acc = 0.f;
    for (int64_t b = 0; b < n; ++b) acc += ld_as_float(dy, dy_dt, b * total + idx);
    dpos[idx] += acc;
  }
}

// ---------------------------------------------------------------------------
// column sums: out[c] += sum_r x[r, c]      (bias gradients)
// block = 32 column-groups (8 cols each) x 8 row lanes
// ---------------------------------------------------------------------------
constexpr int CS_ROWS_PER_BLOCK = 512;
__global__ void __launch_bounds__(256)
colsum_kernel(const void* __restrict__ x, int dt, float* __restrict__ out, int64_t rows,
              int64_t cols, int64_t ld) {
  __shared__ float red[8][32][8];
  const int cg = blockIdx.x * 32 + threadIdx.x;       // 8-column group
  const int64_t c0 = static_cast<int64_t>(cg) * 8;
  const int64_t r0 = static_cast<int64_t>(blockIdx.y) * CS_ROWS_PER_BLOCK;
  int64_t r1 = r0 + CS_ROWS_PER_BLOCK;
  if (r1 > rows) r1 = rows;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c0 < cols && dt == DT_BF16) {
    // 4 independent 16-byte loads in flight per thread
    const bf16* xb = reinterpret_cast<const bf16*>(x);
    int64_t r = r0 + threadIdx.y;
    for (; r + 24 < r1; r += 32) {
      uint4 q[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) q[u] = *reinterpret_cast<const uint4*>(xb + (r + 8 * u) * ld + c0);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        acc[0] += bf16_lo(q[u].x); acc[1] += bf16_hi(q[u].x); acc[2] += bf16_lo(q[u].y); acc[3] += bf16_hi(q[u].y);
        acc[4] += bf16_lo(q[u].z); acc[5] += bf16_hi(q[u].z); acc[6] += bf16_lo(q[u].w); acc[7] += bf16_hi(q[u].w);
      }
    }
    for (; r < r1; r += 8) {
      const uint4 q = *reinterpret_cast<const uint4*>(xb + r * ld + c0);
      acc[0] += bf16_lo(q.x); acc[1] += bf16_hi(q.x); acc[2] += bf16_lo(q.y); acc[3] += bf16_hi(q.y);
      acc[4] += bf16_lo(q.z); acc[5] += bf16_hi(q.z); acc[6] += bf16_lo(q.w); acc[7] += bf16_hi(q.w);
    }
  } else if (c0 < cols) {
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      if (dt == DT_BF16) {
        const uint4 q = *reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(x) + r * ld + c0);
        acc[0] += bf16_lo(q.x); acc[1] += bf16_hi(q.x); acc[2] += bf16_lo(q.y); acc[3] += bf16_hi(q.y);
        acc[4] += bf16_lo(q.z); acc[5] += bf16_hi(q.z); acc[6] += bf16_lo(q.w); acc[7] += bf16_hi(q.w);
      } else {
        const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x) + r * ld + c0);
        const float4 a = p[0], b = p[1];
        acc[0] += a.x; acc[1] += a.y; acc[2] += a.z; acc[3] += a.w;
        acc[4] += b.x; acc[5] += b.y; acc[6] += b.z; acc[7] += b.w;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[threadIdx.y][threadIdx.x][j] = acc[j];
  __syncthreads();
  if (threadIdx.y == 0 && c0 < cols) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float s = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) s += red[y][threadIdx.x][j];
      if (c0 + j < cols) atomicAdd(out + c0 + j, s);
    }
  }
}

// ---------------------------------------------------------------------------
// casts / simple maps
// ---------------------------------------------------------------------------
__global__ void cast_kernel(const void* __restrict__ src, int sdt, void* __restrict__ dst, int ddt,
                            int64_t n) {
  const int64_t n4 = n / 4;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float v[4];
    if (sdt == DT_BF16) {
      const uint2 q = reinterpret_cast<const uint2*>(src)[i];
      v[0] = bf16_lo(q.x); v[1] = bf16_hi(q.x); v[2] = bf16_lo(q.y); v[3] = bf16_hi(q.y);
    } else {
      const float4 q = reinterpret_cast<const float4*>(src)[i];
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    }
    if (ddt == DT_BF16) {
      uint2 q;
      q.x = pack_bf16(v[0], v[1]); q.y = pack_bf16(v[2], v[3]);
      reinterpret_cast<uint2*>(dst)[i] = q;
    } else {
      reinterpret_cast<float4*>(dst)[i] = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = n4 * 4 + threadIdx.x;
    st_from_float(dst, ddt, i, ld_as_float(src, sdt, i));
  }
}

enum : int { MAP_TANH = 0, MAP_TANH_BWD = 1, MAP_GELU = 2, MAP_AXPBY = 3 };
template <int OP>
__global__ void map_kernel(const void* __restrict__ a, const void* __restrict__ b,
                           void* __restrict__ out, int dt, float fa, float fb, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float x = ld_as_float(a, dt, i);
    float r;
    if (OP == MAP_TANH) r = tanhf(x);
    else if (OP == MAP_TANH_BWD) { const float y = ld_as_float(b, dt, i); r = x * (1.f - y * y); }
    else if (OP == MAP_GELU) r = gelu_tanh(x);
    else r = fa * x + fb * ld_as_float(b, dt, i);
    st_from_float(out, dt, i, r);
  }
}

// ---------------------------------------------------------------------------
// L2 normalise: z = x / (||x|| + eps)   (models/proj/image_text/two_towers.py:60-61,73-74)
// ---------------------------------------------------------------------------
__global__ void l2norm_fwd_kernel(const void* __restrict__ x, int dt, float* __restrict__ z,
                                  float* __restrict__ norm, int64_t n, int d, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  float s = 0.f;
  for (int c = lane; c < d; c += 32) { const float v = ld_as_float(x, dt, row * d + c); s += v * v; }
  s = warp_sum(s);
  const float r = sqrtf(s);
  const float inv = 1.f / (r + eps);
  if (lane == 0 && norm) norm[row] = r;
  for (int c = lane; c < d; c += 32) z[row * d + c] = ld_as_float(x, dt, row * d + c) * inv;
}
// dx = (dz - z (z.dz) (r+eps)/r) / (r+eps)
__global__ void l2norm_bwd_kernel(const float* __restrict__ dz, const float* __restrict__ z,
                                  const float* __restrict__ norm, void* __restrict__ dx, int dt,
                                  int64_t n, int d, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  float s = 0.f;
  for (int c = lane; c < d; c += 32) s += dz[row * d + c] * z[row * d + c];
  s = warp_sum(s);
  const float r = norm[row];
  const float inv = 1.f / (r + eps);
  const float k = r > 0.f ? s * (r + eps) / r : 0.f;
  for (int c = lane; c < d; c += 32)
    st_from_float(dx, dt, row * d + c, (dz[row * d + c] - z[row * d + c] * k) * inv);
}

// ---------------------------------------------------------------------------
// pooling over tokens: mode 0 = mean (gap), mode 1 = select token `tok`, mode 2 = max (gmp)
// (models/vit.py:245-253, text_transformer.py:82-90)
// ---------------------------------------------------------------------------
__global__ void pool_fwd_kernel(const void* __restrict__ x, int xdt, void* __restrict__ y, int ydt,
                                int64_t n, int N, int d, int mode, int tok) {
  const int64_t total = n * d;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % d);
    const int64_t b = idx / d;
    float r;
    if (mode == 0) {
      float s = 0.f;
      for (int t = 0; t < N; ++t) s += ld_as_float(x, xdt, (b * N + t) * d + c);
      r = s / static_cast<float>(N);
    } else if (mode == 2) {
      r = ld_as_float(x, xdt, b * N * d + c);
      for (int t = 1; t < N; ++t) r = fmaxf(r, ld_as_float(x, xdt, (b * N + t) * d + c));
    } else {
      r = ld_as_float(x, xdt, (b * N + tok) * d + c);
    }
    st_from_float(y, ydt, idx, r);
  }
}
// d max / d x: the cotangent goes to the positions that hold the maximum, split evenly between
// ties (the rule jnp.max differentiates with); one thread per (item, channel) column
__global__ void pool_max_bwd_kernel(const void* __restrict__ dy, int ydt, const void* __restrict__ x,
                                    int xdt, void* __restrict__ dx, int dxdt, int64_t n, int N, int d) {
  const int64_t total = n * d;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % d);
    const int64_t b = idx / d;
    float m = ld_as_float(x, xdt, b * N * d + c);
    int ties = 1;
    for (int t = 1; t < N; ++t) {
      const float v = ld_as_float(x, xdt, (b * N + t) * d + c);
      if (v > m) { m = v; ties = 1; } else if (v == m) { ++ties; }
    }
    const float g = ld_as_float(dy, ydt, idx) / static_cast<float>(ties);
    for (int t = 0; t < N; ++t) {
      const int64_t at = (b * N + t) * d + c;
      st_from_float(dx, dxdt, at, ld_as_float(x, xdt, at) == m ? g : 0.f);
    }
  }
}
__global__ void pool_bwd_kernel(const void* __restrict__ dy, int ydt, void* __restrict__ dx,
                                int xdt, int64_t n, int N, int d, int mode, int tok) {
  const int64_t total = n * N * d;
  const float invN = 1.f / static_cast<float>(N);
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % d);
    const int64_t bt = idx / d;
    const int t = static_cast<int>(bt % N);
    const int64_t b = bt / N;
    float g = ld_as_float(dy, ydt, b * d + c);
    g = (mode == 0) ? g * invN : (t == tok ? g : 0.f);
    st_from_float(dx, xdt, idx, g);
  }
}

// y[r, :] = x[r % src_rows, :] (+ row[:]) : broadcast / bias add over rows
__global__ void add_rows_kernel(const void* __restrict__ x, int xdt, const float* __restrict__ row,
                                void* __restrict__ y, int ydt, int64_t rows, int d,
                                int64_t src_rows) {
  const int64_t total = rows * d;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % d);
    const int64_t r = idx / d;
    float v = ld_as_float(x, xdt, (r % src_rows) * d + c);
    if (row) v += row[c];
    st_from_float(y, ydt, idx, v);
  }
}

// bf16 [n, N, d] -> [n, d, Np] (Np >= N, pad zero) : Mixer token-mixing transpose
//
// 64 x 64 tiles, 16-byte global accesses on both sides (eight lanes per 128-byte row).  The tile is
// written to shared memory already transposed, two bytes at a time, and read back as 16-byte rows;
// the 8-element column group of row r is XOR-ed with (r / 8) % 8, which spreads the eight row groups a
// warp writes over distinct banks (an unpadded or 16-byte-padded pitch would put them all on one).
constexpr int TT = 64;
__device__ __forceinline__ int tt_swz(int row, int col) { return col ^ (((row >> 3) & 7) << 3); }

__global__ void __launch_bounds__(256)
transpose_tokens_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int N, int d, int Np) {
  __shared__ __align__(16) bf16 tile[TT][TT];          // [channel][token], swizzled
  const int64_t b = blockIdx.z;
  const int t0 = blockIdx.x * TT, c0 = blockIdx.y * TT;
  const int sub = threadIdx.x & 7, row = threadIdx.x >> 3;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const int tl = pass * 32 + row, t = t0 + tl, c = c0 + sub * 8;
    uint4 q = make_uint4(0u, 0u, 0u, 0u);
    if (t < N && c < d) q = *reinterpret_cast<const uint4*>(x + (b * N + t) * d + c);
    const bf16* e = reinterpret_cast<const bf16*>(&q);
#pragma unroll
    for (int i = 0; i < 8; ++i) tile[sub * 8 + i][tt_swz(sub * 8 + i, tl)] = e[i];
  }
  __syncthreads();
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const int cl = pass * 32 + row, c = c0 + cl, t = t0 + sub * 8;
    if (c < d && t < Np)
      *reinterpret_cast<uint4*>(y + (b * d + c) * Np + t) =
          *reinterpret_cast<const uint4*>(&tile[cl][tt_swz(cl, sub * 8)]);
  }
}

// out[b,0,:] = cls[:], out[b,1+t,:] = x[b,t,:]   (models/vit.py:223-225, cls prepended AFTER posemb)
__global__ void concat_cls_kernel(const bf16* __restrict__ x, const float* __restrict__ cls,
                                  bf16* __restrict__ out, int64_t n, int N0, int d) {
  const int groups = d / 8;
  const int64_t total = n * (N0 + 1) * groups;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(idx % groups);
    const int64_t row = idx / groups;
    const int t = static_cast<int>(row % (N0 + 1));
    const int64_t b = row / (N0 + 1);
    uint4 q;
    if (t == 0) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(cls + g * 8));
      const float4 c = __ldg(reinterpret_cast<const float4*>(cls + g * 8) + 1);
      q.x = pack_bf16(a.x, a.y); q.y = pack_bf16(a.z, a.w);
      q.z = pack_bf16(c.x, c.y); q.w = pack_bf16(c.z, c.w);
    } else {
      q = *reinterpret_cast<const uint4*>(x + (b * N0 + (t - 1)) * d + g * 8);
    }
    *reinterpret_cast<uint4*>(out + row * d + g * 8) = q;
  }
}
// out[b,t,:] = x[b,1+t,:]  : drops the cls row (backward of the concat for the patch rows)
__global__ void drop_cls_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int64_t n,
                                int N0, int d) {
  const int groups = d / 8;
  const int64_t total = n * N0 * groups;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(idx % groups);
    const int64_t row = idx / groups;
    const int t = static_cast<int>(row % N0);
    const int64_t b = row / N0;
    *reinterpret_cast<uint4*>(out + row * d + g * 8) =
        *reinterpret_cast<const uint4*>(x + (b * (N0 + 1) + t + 1) * d + g * 8);
  }
}

// Per-sample residual gate of stochastic depth (models/mlp_mixer.py:52,55 with the mask of :173-177):
//   out[b,t,:] = mask[b] != 0 ? a[b,t,:] : (b_or_null ? b_or_null[b,t,:] : 0)        (bf16, d % 8 == 0)
// forward:  a = x + branch(x) (the fused residual epilogue), b = x   ->  x + mask * branch(x), exactly
// backward: a = d out, b = null                                       ->  mask * d out (into the branch)
__global__ void row_select_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b,
                                  const float* __restrict__ mask, bf16* __restrict__ out,
                                  int64_t n, int64_t per_sample_vec) {
  const int64_t total = n * per_sample_vec;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t smp = idx / per_sample_vec;
    uint4 q;
    if (mask[smp] != 0.f) q = reinterpret_cast<const uint4*>(a)[idx];
    else if (b != nullptr) q = reinterpret_cast<const uint4*>(b)[idx];
    else q = make_uint4(0u, 0u, 0u, 0u);
    reinterpret_cast<uint4*>(out)[idx] = q;
  }
}

// out[b,t,c] = (res ? res[b,t,c] : 0) + y[b,c,t]   with y stored [n, d, Np]: inverse of
// transpose_tokens fused with the residual add (models/mlp_mixer.py:51-52)
__global__ void __launch_bounds__(256)
untranspose_add_kernel(const bf16* __restrict__ y, const bf16* __restrict__ res,
                       bf16* __restrict__ out, int N, int d, int Np) {
  __shared__ __align__(16) bf16 tile[TT][TT];          // [token][channel], swizzled
  const int64_t b = blockIdx.z;
  const int t0 = blockIdx.x * TT, c0 = blockIdx.y * TT;
  const int sub = threadIdx.x & 7, row = threadIdx.x >> 3;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const int cl = pass * 32 + row, c = c0 + cl, t = t0 + sub * 8;
    uint4 q = make_uint4(0u, 0u, 0u, 0u);
    if (c < d && t < Np) q = *reinterpret_cast<const uint4*>(y + (b * d + c) * Np + t);
    const bf16* e = reinterpret_cast<const bf16*>(&q);
#pragma unroll
    for (int i = 0; i < 8; ++i) tile[sub * 8 + i][tt_swz(sub * 8 + i, cl)] = e[i];
  }
  __syncthreads();
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const int tl = pass * 32 + row, t = t0 + tl, c = c0 + sub * 8;
    if (t < N && c < d) {
      uint4 q = *reinterpret_cast<const uint4*>(&tile[tl][tt_swz(tl, sub * 8)]);
      if (res != nullptr) {
        const uint4 r = *reinterpret_cast<const uint4*>(res + (b * N + t) * d + c);
        bf16* a = reinterpret_cast<bf16*>(&q);
        const bf16* rr = reinterpret_cast<const bf16*>(&r);
#pragma unroll
        for (int i = 0; i < 8; ++i)
          a[i] = __float2bfloat16_rn(__bfloat162float(a[i]) + __bfloat162float(rr[i]));
      }
      *reinterpret_cast<uint4*>(out + (b * N + t) * d + c) = q;
    }
  }
}

int check_launch(const char* what) { return check_cuda(cudaGetLastError(), what); }

}  // namespace
}  // namespace bv

extern "C" {

int bv_patchify(const float* img, void* out, int64_t n, int32_t H, int32_t W, int32_t C, int32_t P,
                void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0 || P <= 0 || H % P || W % P || C <= 0) {
    set_error("bv_patchify: bad geometry n=%lld H=%d W=%d C=%d P=%d", (long long)n, H, W, C, P);
    return BV_ERR_INVALID;
  }
  const int Kp = (P * P * C + 7) / 8 * 8;
  const int64_t total = n * (H / P) * (W / P) * (Kp / 8);
  patchify_kernel<<<grid_for(total, 256, num_sms() * 16), 256, 0, s>>>(img, reinterpret_cast<bf16*>(out),
                                                                n, H, W, C, P, Kp);
  return check_launch("patchify_kernel");
}

int bv_patchify_u8(const uint8_t* img, void* out, int64_t n, int32_t H, int32_t W, int32_t C, int32_t P,
                   float vmin, float vmax, float in_min, float in_max, int32_t clip, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0 || P <= 0 || H % P || W % P || C <= 0 || !(in_max > in_min)) {
    set_error("bv_patchify_u8: need n > 0, H,W multiples of P, in_max > in_min");
    return BV_ERR_INVALID;
  }
  const int Kp = (P * P * C + 7) / 8 * 8;
  const int64_t total = n * (H / P) * (W / P) * (Kp / 8);
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = static_cast<int64_t>(num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  // (vmax - vmin) is evaluated in double and rounded once, like the Python constant of the reference
  const float vrange = static_cast<float>(static_cast<double>(vmax) - static_cast<double>(vmin));
  patchify_u8_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(
      img, reinterpret_cast<bf16*>(out), n, H, W, C, P, Kp, vmin, vrange, in_min, in_max - in_min, clip, vmax);
  return check_cuda(cudaGetLastError(), "patchify_u8_kernel launch");
}

int bv_embed_fwd(const int32_t* ids, const float* table, const float* pos, void* out, int out_dtype,
                 int64_t n, int32_t L, int32_t d, int32_t vocab, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (d % 4) { set_error("bv_embed_fwd: d %% 4 != 0"); return BV_ERR_INVALID; }
  embed_fwd_kernel<<<grid_for(n * L * (d / 4), 256, num_sms() * 16), 256, 0, s>>>(ids, table, pos, out,
                                                                         out_dtype, n, L, d, vocab);
  return check_launch("embed_fwd_kernel");
}
int bv_embed_bwd(const int32_t* ids, const void* dy, int dy_dtype, float* dtable, float* dpos, int64_t n,
                 int32_t L, int32_t d, int32_t vocab, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtable) {
    embed_bwd_table_kernel<<<grid_for(n * L * d, 256, num_sms() * 16), 256, 0, s>>>(ids, dy, dy_dtype,
                                                                           dtable, n, L, d, vocab);
    int rc = check_launch("embed_bwd_table_kernel");
    if (rc) return rc;
  }
  if (dpos) {
    embed_bwd_pos_kernel<<<grid_for(static_cast<int64_t>(L) * d, 128, num_sms() * 16), 128, 0, s>>>(
        dy, dy_dtype, dpos, n, L, d);
    return check_launch("embed_bwd_pos_kernel");
  }
  return BV_OK;
}

int bv_colsum(const void* x, int x_dtype, float* out, int64_t rows, int64_t cols, int64_t ld, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (cols % 8 || ld % 8 || (reinterpret_cast<uintptr_t>(x) & 15)) {
    set_error("bv_colsum: cols, ld must be multiples of 8 and x 16B aligned");
    return BV_ERR_INVALID;
  }
  if (rows <= 0) return BV_OK;
  dim3 grid(static_cast<unsigned>((cols / 8 + 31) / 32),
            static_cast<unsigned>((rows + CS_ROWS_PER_BLOCK - 1) / CS_ROWS_PER_BLOCK));
  colsum_kernel<<<grid, dim3(32, 8), 0, s>>>(x, x_dtype, out, rows, cols, ld);
  return check_launch("colsum_kernel");
}

int bv_cast(const void* src, int sdt, void* dst, int ddt, int64_t n, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return BV_OK;
  cast_kernel<<<grid_for(n / 4 + 1, 256, num_sms() * 16), 256, 0, s>>>(src, sdt, dst, ddt, n);
  return check_launch("cast_kernel");
}

int bv_l2norm_fwd(const void* x, int dt, float* z, float* norm, int64_t n, int32_t d, float eps,
                  void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return BV_OK;
  l2norm_fwd_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(x, dt, z, norm, n, d, eps);
  return check_launch("l2norm_fwd_kernel");
}
int bv_l2norm_bwd(const float* dz, const float* z, const float* norm, void* dx, int dt, int64_t n, int32_t d,
                  float eps, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0) return BV_OK;
  l2norm_bwd_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(dz, z, norm, dx, dt, n, d, eps);
  return check_launch("l2norm_bwd_kernel");
}

int bv_pool_fwd(const void* x, int xdt, void* y, int ydt, int64_t n, int32_t N, int32_t d, int32_t mode,
                int32_t tok, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (mode < 0 || mode > 2) { set_error("bv_pool: mode must be 0 (mean), 1 (token) or 2 (max)"); return BV_ERR_INVALID; }
  if (mode == 1 && (tok < 0 || tok >= N)) { set_error("bv_pool: token index out of range"); return BV_ERR_INVALID; }
  pool_fwd_kernel<<<grid_for(n * d, 256, num_sms() * 16), 256, 0, s>>>(x, xdt, y, ydt, n, N, d, mode, tok);
  return check_launch("pool_fwd_kernel");
}
int bv_pool_bwd(const void* dy, int ydt, void* dx, int xdt, int64_t n, int32_t N, int32_t d, int32_t mode,
                int32_t tok, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (mode == 2) { set_error("bv_pool_bwd: the max pool needs its input, use bv_pool_max_bwd"); return BV_ERR_INVALID; }
  if (mode != 0 && (tok < 0 || tok >= N)) { set_error("bv_pool_bwd: token index out of range"); return BV_ERR_INVALID; }
  pool_bwd_kernel<<<grid_for(n * N * d, 256, num_sms() * 16), 256, 0, s>>>(dy, ydt, dx, xdt, n, N, d, mode, tok);
  return check_launch("pool_bwd_kernel");
}
int bv_pool_max_bwd(const void* dy, int ydt, const void* x, int xdt, void* dx, int dxdt, int64_t n, int32_t N,
                    int32_t d, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0 || N <= 0 || d <= 0) { set_error("bv_pool_max_bwd: empty problem"); return BV_ERR_INVALID; }
  pool_max_bwd_kernel<<<grid_for(n * d, 256, num_sms() * 16), 256, 0, s>>>(dy, ydt, x, xdt, dx, dxdt, n, N, d);
  return check_launch("pool_max_bwd_kernel");
}

int bv_broadcast_row(const void* x, int xdt, const float* row, void* y, int ydt, int64_t rows, int32_t d,
                     void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  // x holds a single row that is broadcast to `rows` rows (src_rows = 1)
  add_rows_kernel<<<grid_for(rows * d, 256, num_sms() * 16), 256, 0, s>>>(x, xdt, row, y, ydt, rows, d, 1);
  return check_launch("add_rows_kernel");
}

int bv_tanh_fwd(const void* x, void* y, int dt, int64_t n, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  map_kernel<MAP_TANH><<<grid_for(n, 256, num_sms() * 16), 256, 0, s>>>(x, nullptr, y, dt, 0.f, 0.f, n);
  return check_launch("tanh_fwd");
}
int bv_tanh_bwd(const void* dy, const void* y, void* dx, int dt, int64_t n, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  map_kernel<MAP_TANH_BWD><<<grid_for(n, 256, num_sms() * 16), 256, 0, s>>>(dy, y, dx, dt, 0.f, 0.f, n);
  return check_launch("tanh_bwd");
}
int bv_gelu_fwd(const void* x, void* y, int dt, int64_t n, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  map_kernel<MAP_GELU><<<grid_for(n, 256, num_sms() * 16), 256, 0, s>>>(x, nullptr, y, dt, 0.f, 0.f, n);
  return check_launch("gelu_fwd");
}
int bv_axpby(const void* x, const void* y, void* out, int dt, float a, float b, int64_t n, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  map_kernel<MAP_AXPBY><<<grid_for(n, 256, num_sms() * 16), 256, 0, s>>>(x, y, out, dt, a, b, n);
  return check_launch("axpby");
}
int bv_transpose_tokens(const void* x, void* y, int64_t n, int32_t N, int32_t d, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0 || N <= 0 || d <= 0 || d % 8) { set_error("bv_transpose_tokens: need n,N,d > 0, d %% 8 == 0"); return BV_ERR_INVALID; }
  const int Np = (N + 7) / 8 * 8;
  dim3 grid((Np + TT - 1) / TT, (d + TT - 1) / TT, static_cast<unsigned>(n));
  transpose_tokens_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const bf16*>(x),
                                                      reinterpret_cast<bf16*>(y), N, d, Np);
  return check_launch("transpose_tokens_kernel");
}
int bv_untranspose_add(const void* y, const void* res, void* out, int64_t n, int32_t N, int32_t d,
                       void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0 || N <= 0 || d <= 0 || d % 8) { set_error("bv_untranspose_add: need n,N,d > 0, d %% 8 == 0"); return BV_ERR_INVALID; }
  const int Np = (N + 7) / 8 * 8;
  dim3 grid((N + TT - 1) / TT, (d + TT - 1) / TT, static_cast<unsigned>(n));
  untranspose_add_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const bf16*>(y),
                                                     reinterpret_cast<const bf16*>(res),
                                                     reinterpret_cast<bf16*>(out), N, d, Np);
  return check_launch("untranspose_add_kernel");
}
int bv_row_select(const void* a, const void* b, const float* mask, void* out, int64_t n, int32_t N, int32_t d,
                  void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0 || N <= 0 || d <= 0 || d % 8) { set_error("bv_row_select: need n,N,d > 0, d %% 8 == 0"); return BV_ERR_INVALID; }
  const int64_t per = static_cast<int64_t>(N) * d / 8;
  row_select_kernel<<<grid_for(n * per, 256, num_sms() * 16), 256, 0, s>>>(
      reinterpret_cast<const bf16*>(a), reinterpret_cast<const bf16*>(b), mask,
      reinterpret_cast<bf16*>(out), n, per);
  return check_cuda(cudaGetLastError(), "row_select_kernel launch");
}
int bv_concat_cls(const void* x, const float* cls, void* out, int64_t n, int32_t N0, int32_t d,
                  void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (d % 8) { set_error("bv_concat_cls: d %% 8 != 0"); return BV_ERR_INVALID; }
  concat_cls_kernel<<<grid_for(n * (N0 + 1) * (d / 8), 256, num_sms() * 16), 256, 0, s>>>(
      reinterpret_cast<const bf16*>(x), cls, reinterpret_cast<bf16*>(out), n, N0, d);
  return check_launch("concat_cls_kernel");
}
int bv_drop_cls(const void* x, void* out, int64_t n, int32_t N0, int32_t d, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (d % 8) { set_error("bv_drop_cls: d %% 8 != 0"); return BV_ERR_INVALID; }
  drop_cls_kernel<<<grid_for(n * N0 * (d / 8), 256, num_sms() * 16), 256, 0, s>>>(
      reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(out), n, N0, d);
  return check_launch("drop_cls_kernel");
}

}  // extern "C"


// ---- mixup (K16): utils.py:1146-1158 ---------------------------------------------------------
//   out[i] = a * x[i] + (1 - a) * x[(i - 1) mod n]      (jnp.roll(x, shift=1, axis=0))
// One pass, 16-byte vectors when every row is a whole number of them (a scalar pass otherwise, e.g. the
// [n, 21843] labels of ImageNet-21k); the rolled operand is the row the neighbouring block has just read,
// so it is served by L2.  Products and the sum are rounded separately (no FMA contraction): the
// result is bit-identical to the fp32 expression evaluated left to right.
namespace bv {
namespace {
__device__ __forceinline__ float mix1(float a, float b, float u, float v) {
  return __fadd_rn(__fmul_rn(a, u), __fmul_rn(b, v));
}

__global__ void __launch_bounds__(256)
mixup_kernel(const float4* __restrict__ x, float4* __restrict__ out, int64_t n, int64_t row_vec, float a) {
  const float b = __fsub_rn(1.0f, a);
  const int64_t total = n * row_vec;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = idx / row_vec, c = idx - i * row_vec;
    const int64_t ip = (i == 0) ? n - 1 : i - 1;
    const float4 u = x[idx], v = x[ip * row_vec + c];
    float4 o;
    o.x = mix1(a, b, u.x, v.x);
    o.y = mix1(a, b, u.y, v.y);
    o.z = mix1(a, b, u.z, v.z);
    o.w = mix1(a, b, u.w, v.w);
    out[idx] = o;
  }
}

__global__ void __launch_bounds__(256)
mixup_scalar_kernel(const float* __restrict__ x, float* __restrict__ out, int64_t n, int64_t row_elems, float a) {
  const float b = __fsub_rn(1.0f, a);
  const int64_t total = n * row_elems;
  for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = idx / row_elems, c = idx - i * row_elems;
    const int64_t ip = (i == 0) ? n - 1 : i - 1;
    out[idx] = mix1(a, b, x[idx], x[ip * row_elems + c]);
  }
}
}  // namespace
}  // namespace bv

extern "C" {

int bv_mixup(const float* x, float* out, int64_t n, int64_t row_elems, float a, void* stream) {
  using namespace bv;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n <= 0 || row_elems <= 0 || x == out ||
      (reinterpret_cast<uintptr_t>(x) & 3) || (reinterpret_cast<uintptr_t>(out) & 3)) {
    set_error("bv_mixup: need n, row_elems >= 1, 4B-aligned distinct buffers");
    return BV_ERR_INVALID;
  }
  const bool vec = row_elems % 4 == 0 && !(reinterpret_cast<uintptr_t>(x) & 15) &&
                   !(reinterpret_cast<uintptr_t>(out) & 15);
  const unsigned blocks = grid_for(vec ? n * (row_elems / 4) : n * row_elems, 256, num_sms() * 8);
  if (vec) {
    mixup_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(out), n,
                                        row_elems / 4, a);
  } else {
    mixup_scalar_kernel<<<blocks, 256, 0, s>>>(x, out, n, row_elems, a);
  }
  return check_cuda(cudaGetLastError(), "mixup_kernel launch");
}

}  // extern "C"
