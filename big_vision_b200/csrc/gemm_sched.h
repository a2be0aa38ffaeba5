// Work decomposition of the persistent GEMM (csrc/gemm.cu), shared by the host launcher, the
// kernel's producer and consumers, and the CPU tests that check it (tests/test_gemm_sched.py,
// tests/test_gemm_pingpong_sched.py).
//
// A work unit is one 128 x BN output tile times one K split.  Units are numbered n-tile fastest,
// then m-tile, then split (so the CTAs that run at the same time share the A row-panel in L2), and
// CTA b of a grid of G runs units b, b + G, b + 2G, ...  The producer loads every unit of its CTA and
// keeps one running k-block counter across them; its (stage, phase) is a PipeState.  The consumer
// warpgroups walk the same units (ConsumerWalk) and keep the same counter.
#pragma once

#ifdef __CUDACC__
#define BV_HD __host__ __device__ __forceinline__
#else
#define BV_HD inline
#endif

namespace bv {

struct GemmSched {
  int num_m, num_n;          // output tiles along M and N
  int kblocks_total;         // 64-deep k blocks of the whole K
  int kblocks_per_split;     // k blocks per split (the last split may have fewer)
  int splits;
  int units;                 // num_m * num_n * splits
};

struct WorkUnit {
  int m0, n0;                // first output row / column of the tile
  int kb0, kb1;              // k-block range [kb0, kb1), never empty
};

// splits_req <= 0 selects the split count automatically for reduce-add outputs (the weight
// gradients): the count whose units fill whole waves of `slots` persistent CTAs best.  Each extra
// split costs one more fp32 reduce-add of the output tile, negligible against a K of 10^5.  Returns
// false when the request needs split-K without a reduce-add output.
inline bool gemm_make_sched(long long M, long long N, long long K, int bm, int bn, int bk, int splits_req,
                            bool reduce_out, int slots, GemmSched* s) {
  s->num_m = static_cast<int>((M + bm - 1) / bm);
  s->num_n = static_cast<int>((N + bn - 1) / bn);
  s->kblocks_total = static_cast<int>((K + bk - 1) / bk);
  int splits = splits_req;
  if (splits <= 0) {
    splits = 1;
    if (reduce_out) {
      const int tiles = s->num_m * s->num_n;
      int smax = s->kblocks_total / 16;
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
  if (splits > s->kblocks_total) splits = s->kblocks_total;
  if (splits < 1) splits = 1;
  if (splits > 1 && !reduce_out) return false;
  s->kblocks_per_split = (s->kblocks_total + splits - 1) / splits;
  s->splits = (s->kblocks_total + s->kblocks_per_split - 1) / s->kblocks_per_split;
  s->units = s->num_m * s->num_n * s->splits;
  return true;
}

BV_HD WorkUnit gemm_work_unit(const GemmSched& s, int u, int bm, int bn) {
  const int tiles = s.num_m * s.num_n;
  const int split = u / tiles, t = u - split * tiles;
  const int mt = t / s.num_n, nt = t - mt * s.num_n;
  WorkUnit w;
  w.m0 = mt * bm;
  w.n0 = nt * bn;
  w.kb0 = split * s.kblocks_per_split;
  w.kb1 = w.kb0 + s.kblocks_per_split < s.kblocks_total ? w.kb0 + s.kblocks_per_split : s.kblocks_total;
  return w;
}

// position in the STAGES-deep ring of the running k-block counter
struct PipeState {
  int stage = 0;
  unsigned phase = 0;
  BV_HD void advance(int stages) {
    if (++stage == stages) { stage = 0; phase ^= 1u; }
  }
  // n k blocks at once
  BV_HD void advance(int stages, int n) {
    const int t = stage + n;
    phase ^= static_cast<unsigned>(t / stages) & 1u;
    stage = t % stages;
  }
};

// The units of CTA `cta` (of `grid`) that one consumer warpgroup runs.  Ping-pong (`cw` = 0 or 1): the
// CTA's i-th unit is warpgroup i % 2's, so the two warpgroups alternate.  Cooperative (`cw` < 0): the
// warpgroup runs every unit.  next() returns the warpgroup's next unit in `w` (its index in `unit`) and
// moves `ps` past the k blocks of the other warpgroup's units on the way, without waiting on them, so
// that at every k block the warpgroup runs, its (stage, phase) is the producer's.
struct ConsumerWalk {
  int unit, i, grid, cw;
  BV_HD ConsumerWalk(int cta, int grid_, int cw_) : unit(cta - grid_), i(-1), grid(grid_), cw(cw_) {}
  BV_HD bool next(const GemmSched& s, int bm, int bn, int stages, PipeState& ps, WorkUnit& w) {
    for (unit += grid, ++i; unit < s.units; unit += grid, ++i) {
      w = gemm_work_unit(s, unit, bm, bn);
      if (cw < 0 || (i & 1) == cw) return true;
      ps.advance(stages, w.kb1 - w.kb0);
    }
    return false;
  }
};

}  // namespace bv
