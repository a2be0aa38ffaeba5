"""CPU: the bounds of test_gemm_elementwise_gpu.py and test_attention_elementwise_gpu.py checked against
numpy simulations of the arithmetic they model, before any GPU runs them.  Each simulation is a small
instance of the kernel's own order of operations: fp32 accumulation with one truncating addition per
k16 group, fp32 epilogues, bf16 rounding of P and dS, and split-K partials added one by one.  The
bound must cover the simulation, and the same simulation with one defect (a bias added by every split,
alpha applied after the bias, eight columns missing from delta, the last query's delta read as 0) must
break it."""
import math

import numpy as np
import pytest
import torch

import test_attention_elementwise_gpu as AT
import test_gemm_elementwise_gpu as GM

F32 = np.float32


def _trunc32(x):
  """fp64 -> fp32, rounded toward zero (the truncating alignment the bound allows for)."""
  f = x.astype(F32)
  over = np.abs(f.astype(np.float64)) > np.abs(x)
  f[over] = np.nextafter(f[over], F32(0))
  return f


def _bf16(x):
  return torch.from_numpy(np.asarray(x, dtype=F32)).to(torch.bfloat16).float().numpy()


def _mma(a, b, acc=None):
  """sum_k a[:, k] b[:, k] over k16 groups: each group's exact sum added to the fp32 accumulator with
  one truncation (a [M, K], b [N, K], fp64 holding bf16 values)."""
  out = np.zeros((a.shape[0], b.shape[0]), F32) if acc is None else acc
  for g0 in range(0, a.shape[1], 16):
    out = _trunc32(out.astype(np.float64) + a[:, g0:g0 + 16] @ b[:, g0:g0 + 16].T)
  return out


def _rand_bf16(rng, *shape, binades=4):
  x = rng.standard_normal(shape) * np.exp2(rng.integers(-binades, binades + 1, (shape[0], 1)))
  return _bf16(x).astype(np.float64)


# ---------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------
def _sim_gemm(A, B, ranges, alpha, bias, d0, mode, mutation=None, order=None):
  """One output tile: per split the accumulator over its k range, the fp32 epilogue, then the
  reduce-add (fp32 atomics, or bf16 rounding of the partial and a bf16 atomic) in `order`."""
  vs = []
  for s, (k0, k1) in enumerate(ranges):
    acc = _mma(A[:, k0:k1], B[:, k0:k1])
    b = bias if (s == 0 or mutation == "bias_per_split") else F32(0)
    if mutation == "alpha_after_bias":
      vs.append(((acc + b) * F32(alpha)).astype(F32))
    else:
      vs.append((acc * F32(alpha) + b).astype(F32))
  out = d0.astype(F32)
  for s in (order or range(len(vs))):
    if mode == "f32add":
      out = (out + vs[s]).astype(F32)
    else:
      out = _bf16(out + _bf16(vs[s]))
  return out


def _gemm_case(seed, mode):
  rng = np.random.default_rng(seed)
  M, N, K = 6, 5, 300
  A, B = _rand_bf16(rng, M, K), _rand_bf16(rng, N, K)
  bias = rng.standard_normal(N).astype(F32)
  d0 = rng.standard_normal((M, N)).astype(F32)
  if mode == "bf16add":
    d0 = _bf16(d0)
  ranges = GM.splits_of(M, N, K, 128, 3, True, 132)
  assert len(ranges) == 3 and ranges[-1][1] == K
  t = lambda x: torch.from_numpy(np.asarray(x, dtype=np.float64))   # noqa: E731
  parts, errs = GM.split_partials(t(A), t(B), ranges)
  ref, bound = GM.gemm_bound(parts, errs, -3.0, t(bias), mode, d0=t(d0))
  return A, B, ranges, bias, d0, ref.numpy(), bound.numpy()


@pytest.mark.parametrize("mode", ["f32add", "bf16add"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gemm_bound_covers_the_simulation(mode, seed):
  A, B, ranges, bias, d0, ref, bound = _gemm_case(seed, mode)
  for order in ([0, 1, 2], [2, 0, 1]):
    got = _sim_gemm(A, B, ranges, -3.0, bias, d0, mode, order=order)
    err = np.abs(got - ref)
    assert (err <= bound).all(), float((err / bound).max())
  assert float((err / bound).max()) > 1e-3                  # the bound is not vacuous


@pytest.mark.parametrize("mutation", ["bias_per_split", "alpha_after_bias"])
def test_gemm_bound_catches_the_mutations(mutation):
  A, B, ranges, bias, d0, ref, bound = _gemm_case(5, "f32add")
  got = _sim_gemm(A, B, ranges, -3.0, bias, d0, "f32add", mutation=mutation)
  assert (np.abs(got - ref) > bound).any()


def test_splits_of_matches_the_issue_example():
  """M = N = 128, K = 4096 on 132 SMs: 4 splits of 16 k blocks; a request above the k-block count is
  clamped; 49 k blocks in 5 requested splits give 5 splits of 10, 10, 10, 10, 9."""
  assert GM.splits_of(128, 128, 4096, 128, 0, True, 132) == [(0, 1024), (1024, 2048), (2048, 3072), (3072, 4096)]
  assert GM.splits_of(1, 8, 63, 256, 7, True, 132) == [(0, 63)]
  r = GM.splits_of(63, 127, 3096, 128, 5, True, 132)
  assert [(b - a + 63) // 64 for a, b in r] == [10, 10, 10, 10, 9]


# ---------------------------------------------------------------------------------------------------
# attention, one head
# ---------------------------------------------------------------------------------------------------
def _ex2(x):
  """ex2.approx within its 2-ulp bound: the exact value rounded to fp32 (0 below 2^-126)."""
  y = np.exp2(x.astype(np.float64)).astype(F32)
  y[y < 2.0 ** -126] = 0
  return y


def _sim_fwd(q, k, v, scale):
  """attn_fwd_kernel on one head of one batch entry: 64-key blocks, online max / l, bf16 P."""
  Nq, Nk = q.shape[0], k.shape[0]
  sl2 = F32(F32(scale) * F32(AT.LOG2E))
  m = np.full(Nq, -np.inf, F32)
  l = np.zeros(Nq, F32)
  o = np.zeros((Nq, v.shape[1]), F32)
  for j0 in range(0, Nk, AT.T):
    s = (_mma(q, k[j0:j0 + AT.T]) * sl2).astype(F32)
    mx = np.maximum(m, s.max(1))
    corr = _ex2((m - mx).astype(F32))
    m = mx
    p = _ex2((s - m[:, None]).astype(F32))
    l = (l * corr + p.sum(1, dtype=F32)).astype(F32)
    o = (o * corr[:, None]).astype(F32)
    o = _mma(_bf16(p).astype(np.float64), v[j0:j0 + AT.T].T, o)
  out = _bf16(o * (F32(1) / l)[:, None])
  lse = ((m + np.log2(l).astype(F32)) * F32(AT.LN2)).astype(F32)
  return out.astype(np.float64), lse


def _sim_bwd(q, k, v, o, do, lse, scale, mutation=None):
  """The delta pre-kernel, attn_bwd_dq_kernel and attn_bwd_dkdv_kernel on one head."""
  Nq = q.shape[0]
  dh = q.shape[1]
  cols = dh - 8 if mutation == "delta_drops_8_columns" else dh
  delta = (o[:, :cols] * do[:, :cols]).astype(F32).sum(1, dtype=F32)
  sl2 = F32(F32(scale) * F32(AT.LOG2E))
  lse2 = (lse * F32(AT.LOG2E)).astype(F32)
  s = (_mma(q, k) * sl2).astype(F32)
  P = _ex2((s - lse2[:, None]).astype(F32))
  dP = _mma(do, v)
  dl = delta.copy()
  if mutation == "last_query_delta_zero":
    dl[Nq - 1] = 0
  dS = (P * (dP - dl[:, None]).astype(F32)).astype(F32)
  dSb = _bf16(dS).astype(np.float64)
  dq = _bf16(_mma(dSb, k.T) * F32(scale))
  dk = _bf16(_mma(dSb.T, q.T) * F32(scale))
  dv = _bf16(_mma(_bf16(P).astype(np.float64).T, do.T))
  return dq, dk, dv


def _attn_case(seed, dh=72, Nq=5, Nk=70):
  rng = np.random.default_rng(seed)
  q, k, v, do = (_rand_bf16(rng, n, dh, binades=1) for n in (Nq, Nk, Nk, Nq))
  scale = float(F32(1 / math.sqrt(dh)))
  t = lambda x: torch.from_numpy(np.asarray(x, dtype=np.float64))[None]   # noqa: E731
  f = AT.fwd_bound(t(q), t(k), t(v), scale)
  b = AT.bwd_bound(t(q), t(k), t(v), t(do), scale, f)
  return q, k, v, do, scale, f, b


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_attention_bounds_cover_the_simulation(seed):
  q, k, v, do, scale, f, b = _attn_case(seed)
  o, lse = _sim_fwd(q, k, v, scale)
  assert (np.abs(o - f["O"][0].numpy()) <= f["bO"][0].numpy()).all()
  assert (np.abs(lse - f["lse"][0].numpy()) <= f["blse"][0].numpy()).all()
  dq, dk, dv = _sim_bwd(q, k, v, o, do, lse, scale)
  for got, name in ((dq, "dQ"), (dk, "dK"), (dv, "dV")):
    err = np.abs(got - b[name][0].numpy())
    assert (err <= b["b" + name][0].numpy()).all(), name


@pytest.mark.parametrize("mutation", ["delta_drops_8_columns", "last_query_delta_zero"])
def test_attention_bounds_catch_the_mutations(mutation):
  q, k, v, do, scale, f, b = _attn_case(7)
  o, lse = _sim_fwd(q, k, v, scale)
  dq, dk, _ = _sim_bwd(q, k, v, o, do, lse, scale, mutation=mutation)
  bad = (np.abs(dq - b["dQ"][0].numpy()) > b["bdQ"][0].numpy()).any() or \
      (np.abs(dk - b["dK"][0].numpy()) > b["bdK"][0].numpy()).any()
  assert bad
