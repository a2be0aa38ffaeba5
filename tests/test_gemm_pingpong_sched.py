"""The ping-pong consumers of the persistent GEMM (csrc/gemm_sched.h, ConsumerWalk), compiled for the
host: the two consumer warpgroups of a CTA take its units alternately, each exactly once, and at every
k block a warpgroup runs, its ring position (stage, phase) is the one the producer loaded it at, though
it stepped over the other warpgroup's units without waiting on them."""
import ctypes
import shutil
import subprocess

import numpy as np
import pytest

from test_gemm_sched import CSRC, M_IMG, M_TXT, SHAPES

DRIVER = r"""
#include "gemm_sched.h"
using namespace bv;

extern "C" int units(int M, int N, int K, int splits, int reduce, int slots) {
  GemmSched s;
  gemm_make_sched(M, N, K, 128, 128, 64, splits, reduce != 0, slots, &s);
  return s.units;
}

// Records (unit, kb, stage, phase) per k block of CTA `cta` of `grid` at 128 x 128 units.  cw = -2 is
// the producer's loop (recording the phase it loads at, i.e. its "empty" parity flipped), cw = 0 / 1 a
// ping-pong consumer and cw = -1 a cooperative one, each through ConsumerWalk.
extern "C" int walk(int M, int N, int K, int splits, int reduce, int slots, int stages, int cta, int grid, int cw,
                    int* out) {
  GemmSched s;
  gemm_make_sched(M, N, K, 128, 128, 64, splits, reduce != 0, slots, &s);
  PipeState ps;
  int n = 0;
  auto rec = [&](int u, int kb) {
    out[4 * n] = u; out[4 * n + 1] = kb; out[4 * n + 2] = ps.stage; out[4 * n + 3] = static_cast<int>(ps.phase);
    ++n;
    ps.advance(stages);
  };
  if (cw == -2) {
    for (int u = cta; u < s.units; u += grid) {
      const WorkUnit w = gemm_work_unit(s, u, 128, 128);
      for (int kb = w.kb0; kb < w.kb1; ++kb) rec(u, kb);
    }
    return n;
  }
  ConsumerWalk walk(cta, grid, cw);
  WorkUnit w;
  while (walk.next(s, 128, 128, stages, ps, w))
    for (int kb = w.kb0; kb < w.kb1; ++kb) rec(walk.unit, kb);
  return n;
}
"""


@pytest.fixture(scope="module")
def sched(tmp_path_factory):
  cxx = shutil.which("c++") or shutil.which("g++") or shutil.which("clang++")
  if cxx is None:
    pytest.skip("no host C++ compiler")
  d = tmp_path_factory.mktemp("gemm_pingpong")
  src, so = d / "driver.cc", d / "driver.so"
  src.write_text(DRIVER)
  subprocess.run([cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, str(src), "-o", str(so)], check=True)
  return ctypes.CDLL(str(so))


def _walk(lib, M, N, K, splits, reduce, stages, cta, grid, cw, cap):
  out = np.zeros(4 * cap, dtype=np.int32)
  n = lib.walk(M, N, K, splits, reduce, 132, stages, cta, grid, cw, out.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
  assert n <= cap
  return out[:4 * n].reshape(n, 4)


def _check_cta(lib, M, N, K, splits, reduce, stages, cta, grid, cap):
  prod = _walk(lib, M, N, K, splits, reduce, stages, cta, grid, -2, cap)
  cons = [_walk(lib, M, N, K, splits, reduce, stages, cta, grid, cw, cap) for cw in (0, 1)]
  # the CTA's i-th unit belongs to warpgroup i % 2, and each runs its units in the producer's order
  cta_units = list(dict.fromkeys(prod[:, 0].tolist()))
  for cw in (0, 1):
    assert list(dict.fromkeys(cons[cw][:, 0].tolist())) == cta_units[cw::2]
  # together they run every (unit, k block) of the CTA exactly once, each at the producer's (stage,
  # phase): joined on (unit, kb), the records are the producer's
  both = np.concatenate(cons)
  both = both[np.lexsort((both[:, 1], both[:, 0]))]
  assert both.shape == prod.shape
  assert (both == prod[np.lexsort((prod[:, 1], prod[:, 0]))]).all()
  # the cooperative walk is the producer's
  assert (_walk(lib, M, N, K, splits, reduce, stages, cta, grid, -1, cap) == prod).all()
  return len(cta_units)


# the step's shapes (SHAPES of test_gemm_sched.py: forward / dgrad, split-K weight gradients, ragged ones)
@pytest.mark.parametrize("stages", [5, 6, 7])
@pytest.mark.parametrize("M,N,K,reduce", SHAPES)
def test_pingpong_walk_matches_the_producer(sched, M, N, K, reduce, stages):
  units = sched.units(M, N, K, 0, reduce, 132)
  kbt = (K + 63) // 64
  seen = set()
  # the persistent grid; a grid that leaves some CTAs an odd unit count; one unit per CTA
  for grid in sorted({min(units, 132), min(units, 7), units}):
    cap = kbt * (-(-units // grid)) + 1
    ctas = range(grid) if grid <= 132 else (0, grid // 2, grid - 1)
    counts = [_check_cta(sched, M, N, K, 0, reduce, stages, cta, grid, cap) for cta in ctas]
    seen.update(c % 2 for c in counts)
    if grid == units:
      assert set(counts) == {1}      # warpgroup 1 runs nothing (the walk above found no unit for it)
  assert 1 in seen                   # an odd unit count per CTA occurred


@pytest.mark.parametrize("M,N,K,splits,reduce", [(M_TXT, 768, 768, 1, 0), (3000, 700, 64, 1, 0),
                                                 (768, 768, M_IMG, 5, 1), (200, 40, 192, 3, 1)])
@pytest.mark.parametrize("grid", [1, 2, 3, 132])
def test_pingpong_walk_small_grids(sched, M, N, K, splits, reduce, grid):
  """Units with fewer k blocks than stages (K = 64) and many units per CTA on tiny grids."""
  units = sched.units(M, N, K, splits, reduce, 132)
  grid = min(grid, units)
  cap = (K + 63) // 64 * (-(-units // grid)) + 1
  for cta in range(grid):
    _check_cta(sched, M, N, K, splits, reduce, 3, cta, grid, cap)
