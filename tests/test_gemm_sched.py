"""The persistent GEMM's work decomposition (csrc/gemm_sched.h), compiled for the host: every output
element of every K split is covered by exactly one work unit, the splits partition K, and the
producer and the consumers of each CTA walk the same (unit, k block) -> (stage, phase) sequence."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "big_vision_b200", "csrc")

DRIVER = r"""
#include "gemm_sched.h"
using namespace bv;

extern "C" int plan(long long M, long long N, long long K, int bn, int splits, int reduce, int slots, int* out) {
  GemmSched s;
  if (!gemm_make_sched(M, N, K, 128, bn, 64, splits, reduce != 0, slots, &s)) return -1;
  out[0] = s.num_m; out[1] = s.num_n; out[2] = s.kblocks_total; out[3] = s.kblocks_per_split;
  out[4] = s.splits; out[5] = s.units;
  return 0;
}

extern "C" void units(int M, int N, int K, int bn, int splits, int reduce, int slots, int* out) {
  GemmSched s;
  gemm_make_sched(M, N, K, 128, bn, 64, splits, reduce != 0, slots, &s);
  for (int u = 0; u < s.units; ++u) {
    const WorkUnit w = gemm_work_unit(s, u, 128, bn);
    out[4 * u] = w.m0; out[4 * u + 1] = w.n0; out[4 * u + 2] = w.kb0; out[4 * u + 3] = w.kb1;
  }
}

// The kernel's two loops for CTA `cta` of `grid`, recording (unit, kb, stage, phase) per k block.
// role 0 is the producer, role 1 a consumer warpgroup; returns the number of records.
extern "C" int walk(int M, int N, int K, int bn, int splits, int reduce, int slots, int stages, int cta, int grid,
                    int role, int* out) {
  GemmSched s;
  gemm_make_sched(M, N, K, 128, bn, 64, splits, reduce != 0, slots, &s);
  PipeState ps;
  int n = 0;
  for (int u = cta; u < s.units; u += grid) {
    const WorkUnit w = gemm_work_unit(s, u, 128, bn);
    for (int kb = w.kb0; kb < w.kb1; ++kb) {
      out[4 * n] = u; out[4 * n + 1] = kb; out[4 * n + 2] = ps.stage;
      out[4 * n + 3] = static_cast<int>(role == 0 ? ps.phase ^ 1u : ps.phase);   // producer waits on "empty"
      ++n;
      ps.advance(stages);
    }
  }
  return n;
}
"""


@pytest.fixture(scope="module")
def sched(tmp_path_factory):
  cxx = shutil.which("c++") or shutil.which("g++") or shutil.which("clang++")
  if cxx is None:
    pytest.skip("no host C++ compiler")
  d = tmp_path_factory.mktemp("gemm_sched")
  src, so = d / "driver.cc", d / "driver.so"
  src.write_text(DRIVER)
  subprocess.run([cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, str(src), "-o", str(so)], check=True)
  return ctypes.CDLL(str(so))


def _plan(lib, M, N, K, bn, splits=0, reduce=0, slots=132):
  out = (ctypes.c_int * 6)()
  rc = lib.plan(ctypes.c_longlong(M), ctypes.c_longlong(N), ctypes.c_longlong(K), bn, splits, reduce, slots, out)
  return None if rc else dict(zip(("num_m", "num_n", "kbt", "kbps", "splits", "units"), list(out)))


def _units(lib, M, N, K, bn, splits, reduce, slots, n):
  out = np.zeros(4 * n, dtype=np.int32)
  lib.units(M, N, K, bn, splits, reduce, slots, out.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
  return out.reshape(n, 4)


M_IMG, M_TXT = 768 * 196, 768 * 64
# (M, N, K, reduce): the step's forward / dgrad shapes and its split-K weight gradients, then ragged ones
SHAPES = [
    (M_IMG, 3072, 768, 0), (M_IMG, 768, 3072, 0), (M_IMG, 2304, 768, 0), (M_IMG, 768, 2304, 0),
    (M_TXT, 3072, 768, 0), (M_TXT, 768, 768, 0),
    (768, 3072, M_IMG, 1), (3072, 768, M_IMG, 1), (768, 2304, M_TXT, 1), (768, 768, M_TXT, 1),
    (1, 768, 768, 0), (3, 1000, 64, 0), (130, 1000, 768, 0), (200, 40, 192, 0), (1, 768, 768, 1),
    (1000, 1000, 100, 1),
]


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("M,N,K,reduce", SHAPES)
def test_units_cover_every_element_once(sched, M, N, K, reduce, bn):
  p = _plan(sched, M, N, K, bn, reduce=reduce)
  assert p["units"] == p["num_m"] * p["num_n"] * p["splits"]
  if not reduce:
    assert p["splits"] == 1
  u = _units(sched, M, N, K, bn, 0, reduce, 132, p["units"])
  m0, n0, kb0, kb1 = u.T
  assert (kb1 > kb0).all()
  assert (m0 % 128 == 0).all() and (n0 % bn == 0).all() and (m0 < M).all() and (n0 < N).all()
  # raster order: n-tile fastest, then m-tile, then split
  tiles = p["num_m"] * p["num_n"]
  idx = np.arange(p["units"])
  assert (n0 // bn == idx % p["num_n"]).all() and (m0 // 128 == (idx % tiles) // p["num_n"]).all()
  # per split, the tiles cover [0, M) x [0, N) exactly once (tile-level: tiles are disjoint 128 x bn
  # blocks, so covering each (m-tile, n-tile) once covers each element once)
  kb_per_split = {}
  for s in range(p["splits"]):
    sel = slice(s * tiles, (s + 1) * tiles)
    cover = np.zeros((p["num_m"], p["num_n"]), dtype=np.int32)
    np.add.at(cover, (m0[sel] // 128, n0[sel] // bn), 1)
    assert (cover == 1).all()
    ranges = set(zip(kb0[sel].tolist(), kb1[sel].tolist()))
    assert len(ranges) == 1
    kb_per_split[s] = ranges.pop()
  # the splits partition the k blocks of K
  edges = sorted(kb_per_split.values())
  assert edges[0][0] == 0 and edges[-1][1] == (K + 63) // 64
  assert all(a[1] == b[0] for a, b in zip(edges, edges[1:]))


def test_wgrad_split_selection(sched):
  """Split-K still fills whole waves of persistent CTAs at the step's weight-gradient shapes."""
  for M, N, K in ((768, 3072, M_IMG), (3072, 768, M_IMG), (768, 768, M_IMG), (768, 2304, M_TXT)):
    p = _plan(sched, M, N, K, 256, reduce=1)
    assert p["splits"] > 1 and p["units"] > 132
    assert p["units"] / (-(-p["units"] // 132) * 132) >= 0.9
  assert _plan(sched, 1000, 1000, 6400, 256, splits=2, reduce=0) is None


@pytest.mark.parametrize("stages", [3, 4, 6])
@pytest.mark.parametrize("M,N,K,reduce", [(M_IMG, 3072, 768, 0), (768, 3072, M_IMG, 1), (130, 1000, 768, 0)])
def test_producer_and_consumers_agree(sched, M, N, K, reduce, stages):
  p = _plan(sched, M, N, K, 256, reduce=reduce)
  grid = min(p["units"], 132)
  total = 0
  for cta in range(grid):
    n_max = 4 * (p["kbps"] * (-(-p["units"] // grid)) + 1)
    recs = []
    for role in (0, 1):
      out = np.zeros(n_max, dtype=np.int32)
      n = sched.walk(M, N, K, 256, 0, reduce, 132, stages, cta, grid, role,
                     out.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
      recs.append(out[:4 * n].reshape(n, 4))
    prod, cons = recs
    assert prod.shape == cons.shape
    assert (prod[:, :3] == cons[:, :3]).all()            # same units, k blocks and stages
    assert (prod[:, 3] == cons[:, 3] ^ 1).all()          # producer waits "empty" at the flipped parity
    # the running counter: stage = i mod STAGES, phase flips on every wrap
    i = np.arange(len(cons))
    assert (cons[:, 2] == i % stages).all() and (cons[:, 3] == (i // stages) % 2).all()
    total += len(cons)
  assert total == p["kbt"] * p["num_m"] * p["num_n"]     # every tile's k blocks, once over all CTAs
