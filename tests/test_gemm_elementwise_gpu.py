"""Element-wise fp64 parity of bv_gemm over its instantiations: the four operand layouts, block_n 128 /
256 / auto, fp32 and bf16 outputs, plain and reduce-add, every split-K schedule, every epilogue, alpha
other than 1, and ragged M, N and K.  Every operand is a strided view into a wider buffer whose
padding (columns past the extent, rows past it) holds NaN, and every output is a view into a buffer
whose surroundings hold a sentinel: a read outside the logical extent reaches an output as NaN, and a
write outside it changes the sentinel.  References are fp64 matrix products on the GPU.

Tier 1, exact arithmetic.  Integer-valued bf16 operands and dyadic bias, aux, initial D and alpha,
with alpha * sum_k |a_k b_k| + |bias| + |aux| + |D| < 2^21 for every element (asserted): every value
is a multiple of 1/8 below 2^21, so every partial sum the kernel can form, in any order, split or
tensor-core grouping, is exact in fp32.  fp32 outputs then equal the fp64 value bit for bit, bf16
outputs equal its round-to-nearest-even, BIAS_RESID gives bf16(bf16(exact + bias) + aux) with the
aux_row_mod wrap, BIAS_GELU's D2 is bf16(exact + bias).  A wrong tile, k block, split boundary, a bias
or residual added per split, alpha applied in the wrong place or a wrong residual row changes bits.
The exceptions are bounded: GELU / gelu' through tanh.approx (the bounds stated in common.cuh and
swept in test_kernel_edges_gpu.py) and bf16 reduce-adds with more than one split, which round each
split's partial and add them in no fixed order.

Tier 2, random data, a derived bound (`gemm_bound`).  Gaussian operands with rows and columns scaled
over several binades and a few outlier rows.  The accumulation is modelled as one fp32 addition per
k16 wgmma, in the kernel's own split boundaries (gemm_make_sched restated in `splits_of`), whose
error is at most 2^-23 (|running accumulator| + sum of the group's |a b|): 2^-23 rather than the
unit roundoff 2^-24 because the tensor core's internal alignment may truncate instead of round.
That rounding behaviour is not documented by NVIDIA and was not measured for this model: the bound
is an assumption the test holds the hardware to.  Then fp32 roundings of the epilogue (2^-24 of each
operand of alpha * acc + bias), one output ulp, and for reduce-adds one rounding per atomic
addition.  No constant is fitted to observed errors; the largest err / bound ratio of each test is
printed by test_print_error_bound_ratios.
"""
import json
import zlib

import pytest
import torch

from test_kernel_edges_gpu import _TANH_APPROX, _check, _dgelu64, _gelu64, _same, _ulp

pytestmark = pytest.mark.gpu
F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
U32 = 2.0 ** -24          # fp32 unit roundoff
U_MMA = 2.0 ** -23        # per-k16-wgmma accumulation error (module docstring)
U_BF = 2.0 ** -8          # bf16 unit roundoff (8 significant bits)
BM, BK = 128, 64
DEV = "cuda"
NAN = float("nan")
SENT = {F32: 1234.5, BF16: -8192.0}
RATIOS = {}


@pytest.fixture(scope="module")
def ops():
  from big_vision_b200 import lib, ops as _ops
  assert lib.load().bv_device_supported() == 1, "needs a compute-capability 9.x GPU"
  return _ops


# ---------------------------------------------------------------------------------------------------
# the kernel's schedule and the bound (importable without a device: test_elementwise_bounds.py)
# ---------------------------------------------------------------------------------------------------
def splits_of(M, N, K, bn, splits_req, reduce_out, slots):
  """gemm_make_sched (csrc/gemm_sched.h) restated: the [k0, k1) element ranges of the K splits."""
  num_m, num_n = -(-M // BM), -(-N // bn)
  kbt = -(-K // BK)
  splits = splits_req
  if splits <= 0:
    splits = 1
    if reduce_out:
      tiles, best = num_m * num_n, -1.0
      for sp in range(1, min(kbt // 16, 32) + 1):
        units = tiles * sp
        eff = units / (-(-units // slots) * slots) - 0.002 * sp
        if eff > best + 1e-9:
          best, splits = eff, sp
  splits = max(1, min(splits, kbt))
  kps = -(-kbt // splits)
  return [(kb * BK, min((kb + kps) * BK, K)) for kb in range(0, kbt, kps)]


def split_partials(A, B, ranges, model_error=True, elems=2 ** 25):
  """A [M, K], B [N, K] fp64 (the logical operands).  Per split: the exact partial sum_k A B^T over
  its k range and, with model_error, the accumulation bound 2^-23 sum_g (|S before g| + sum_{k in g}
  |a_k b_k|) over the split's k16 groups g (the accumulator restarts at each split).  Chunked over
  rows and groups so that no temporary exceeds `elems` elements."""
  M, N = A.shape[0], B.shape[0]
  parts, errs = [], []
  for k0, k1 in ranges:
    a, b = A[:, k0:k1], B[:, k0:k1]
    parts.append(a @ b.T)
    if not model_error:
      continue
    err = a.abs() @ b.abs().T
    pad = -(k1 - k0) % 16
    if pad:
      a = torch.nn.functional.pad(a, (0, pad))
      b = torch.nn.functional.pad(b, (0, pad))
    ng = a.shape[1] // 16
    mc = max(1, min(M, elems // max(1, N * min(ng, 64))))
    gc = max(1, min(ng, elems // max(1, mc * N)))
    bg = b.reshape(N, ng, 16).permute(1, 2, 0)                    # [ng, 16, N]
    for m0 in range(0, M, mc):
      ag = a[m0:m0 + mc].reshape(-1, ng, 16).transpose(0, 1)      # [ng, mc, 16]
      run = torch.zeros(ag.shape[1], N, dtype=F64, device=A.device)
      for g0 in range(0, ng, gc):
        gs = torch.bmm(ag[g0:g0 + gc], bg[g0:g0 + gc])            # group sums [gc, mc, N]
        cs = torch.cumsum(gs, 0)
        err[m0:m0 + mc] += (run + cs - gs).abs().sum(0)            # |S before g|
        run += cs[-1]
    errs.append(err * U_MMA)
  return parts, errs


def gemm_bound(parts, errs, alpha, bias, mode, d0=None, aux=None, resid=False, dgelu=None):
  """Bound on |D - ref| per element, ref = d0 + sum_s v_s with v_s = alpha p_s (+ bias + aux on split
  0) (times gelu'(aux) for dgelu, whose fp64 value and tanh.approx error are passed as (g, dg)).
    fp32 epilogue: 2^-24 (|alpha p_s| + |alpha p_s + b|), + 2^-24 |v| for the residual add;
    accumulation: |alpha| * err_s (split_partials);
    mode 'f32': nothing more; 'f32add': (splits + 1) fp32 additions of the atomics onto d0,
    each at most 2^-24 (|d0| + sum_s |v_s|); 'bf16': one bf16 ulp of the reference (and of the
    pre-residual value for the residual, which is rounded to bf16 before aux is added); 'bf16add':
    each split's bf16 rounding 2^-8 |v_s| and each atomic's 2^-8 (|d0| + sum_s |v_s|), with (1 + 2^-6)
    for the second-order terms."""
  b = torch.zeros_like(parts[0][0]) if bias is None else bias
  S = len(parts)
  tot = torch.zeros_like(parts[0])
  vabs = torch.zeros_like(parts[0])
  ref = torch.zeros_like(parts[0]) if d0 is None else d0.clone()
  for s, (p, e) in enumerate(zip(parts, errs)):
    ap = alpha * p
    pre = ap + (b if s == 0 else 0.0)
    eps = abs(alpha) * e + U32 * (ap.abs() + pre.abs())
    v = pre
    if resid and s == 0:
      v = pre + aux
      eps = eps + U32 * v.abs()
      if mode in ("bf16", "bf16add"):
        eps = eps + _ulp(pre, BF16)
    if dgelu is not None:
      g, dg = dgelu
      v = pre * g
      eps = eps * g.abs() + pre.abs() * dg + U32 * v.abs() + 2.0 ** -20 * v.abs()
    if mode == "bf16add":
      eps = eps + U_BF * v.abs() * (1 + 2.0 ** -6)
    tot = tot + eps
    vabs = vabs + v.abs()
    ref = ref + v
  d0a = 0.0 if d0 is None else d0.abs()
  if mode == "f32add":
    tot = tot + (S + 1) * U32 * (d0a + vabs)
  elif mode == "bf16add":
    tot = tot + S * U_BF * (d0a + vabs) * (1 + 2.0 ** -6)
  elif mode == "bf16":
    tot = tot + _ulp(ref, BF16)
  return ref, tot


def colsum_chain(M):
  """Longest fp32 addition chain of the fused colsum: two rows per thread, three shuffle levels, one
  atomic per warp (8 per 128-row tile) onto the initial value."""
  return 2 + 3 + 8 * -(-M // BM) + 1


# ---------------------------------------------------------------------------------------------------
# buffers
# ---------------------------------------------------------------------------------------------------
def _nan_view(data, extra_rows=3, extra_cols=5, dtype=BF16):
  """`data` [R, C] inside a NaN buffer with row stride round_up(C, 8) + 8 and `extra_rows` NaN rows;
  returns the stored view [R + extra_rows - 1, C + extra_cols] (larger than the logical operand)."""
  R, C = data.shape
  ld = -(-C // 8) * 8 + 8
  buf = torch.full((R + extra_rows, ld), NAN, dtype=dtype, device=DEV)
  buf[:R, :C] = data.to(dtype)
  return buf[:R + extra_rows - 1, :min(ld, C + extra_cols)]


def _out_buf(M, N, dtype, init=None):
  """(buffer, view): the view [M, N] holds `init` (NaN if None), the rest of the buffer a sentinel."""
  ld = -(-N // 8) * 8 + 8
  buf = torch.full((M + 2, ld), SENT[dtype], dtype=dtype, device=DEV)
  view = buf[:M, :N]
  view.fill_(NAN) if init is None else view.copy_(init)
  return buf, view


def _sentinel_intact(buf, M, N, what):
  mask = torch.ones(buf.shape, dtype=torch.bool, device=DEV)
  mask[:M, :N] = False
  outside = buf[mask]
  assert bool((outside == SENT[buf.dtype]).all()), f"{what}: {int((outside != SENT[buf.dtype]).sum())} " \
                                                   "elements outside the output view were written"


def _bias_buf(b):
  n = b.numel()
  buf = torch.full((-(-n // 8) * 8 + 8,), NAN, dtype=F32, device=DEV)
  buf[:n] = b
  return buf[:n]


def _record(key, got, ref, bound):
  err = (got.double() - ref).abs()
  r = float((err / bound.clamp_min(1e-300)).max())
  RATIOS[key] = max(RATIOS.get(key, 0.0), r)


def _check_r(key, got, ref, bound, what):
  _check(got, ref, bound, what)
  _record(key, got, ref, bound)


# ---------------------------------------------------------------------------------------------------
# the configuration matrix (sampled, not enumerated)
# (a_mn, b_mn, block_n, mode, epilogue, alpha, M, N, K, splits, aux_row_mod); alpha -4 is -3 in tier 2
# ---------------------------------------------------------------------------------------------------
M_IMG = 768 * 196           # ViT-B/16 at 224, 768 images per GPU: the training step's token rows
CASES = [
    (0, 1, 0, "bf16", "bias", 1.0, M_IMG, 768, 768, 0, 0),         # step forward (the MLP's fc2 shape)
    (1, 1, 0, "f32add", "bias", 1.0, 768, 768, M_IMG, 0, 0),       # step wgrad, auto split
    (0, 0, 128, "bf16", "none", 0.125, 65, 1000, 65, 0, 0),
    (1, 1, 256, "f32add", "bias", 1.0, 64, 255, 3096, 2, 0),
    (1, 0, 0, "f32add", "bias", -4.0, 128, 128, 4096, 0, 0),       # auto: 4 splits on 132 SMs
    (1, 1, 128, "f32add", "none", 0.125, 63, 127, 3096, 5, 0),     # 49 k blocks in 5 splits
    (0, 1, 256, "f32add", "bias", 1.0, 1, 8, 63, 7, 0),            # 7 splits of 1 k block: clamped
    (0, 0, 256, "f32add", "none", -4.0, 64, 1000, 776, 1, 0),
    (0, 0, 0, "f32", "bias", -4.0, 1, 1, 1, 0, 0),
    (1, 1, 0, "f32", "resid", 1.0, 4097, 65, 64, 0, 196),
    (0, 1, 128, "f32", "resid", 0.125, 129, 7, 8, 0, 0),
    (0, 1, 256, "f32", "none", 1.0, 127, 21843, 8, 0, 0),
    (0, 1, 256, "f32add", "resid", 1.0, 65, 129, 3096, 3, 0),
    (0, 1, 0, "bf16", "resid", 1.0, 4097, 255, 64, 0, 0),
    (1, 0, 256, "bf16", "resid", -4.0, 129, 257, 776, 0, 49),
    (0, 1, 128, "bf16", "resid", 0.125, 63, 21843, 65, 0, 257),
    (0, 1, 0, "bf16add", "resid", 1.0, 65, 9, 776, 0, 0),
    (1, 1, 0, "bf16add", "resid", 1.0, 128, 65, 3096, 2, 196),
    (0, 0, 0, "bf16add", "bias", -4.0, 64, 1, 63, 0, 0),
    (1, 0, 0, "bf16add", "bias", 0.125, 127, 129, 4096, 0, 0),
    (0, 1, 256, "bf16", "gelu", 1.0, 129, 1000, 776, 0, 0),
    (1, 1, 128, "bf16", "gelu_act", -4.0, 64, 129, 64, 0, 0),
    (0, 0, 0, "bf16", "dgelu", 0.125, 4097, 127, 63, 0, 0),
    (0, 1, 0, "bf16add", "dgelu", 1.0, 65, 257, 3096, 2, 0),
    (1, 0, 128, "bf16", "bias", 1.0, 128, 8, 1, 0, 0),
]


def _cid(c):
  return f"{'NT'[c[0]]}{'NT'[c[1]]}-bn{c[2]}-{c[3]}-{c[4]}-a{c[5]}-{c[6]}x{c[7]}x{c[8]}-s{c[9]}-mod{c[10]}"


def _epi(L, name):
  return {"none": L.EPI_NONE, "bias": L.EPI_BIAS, "resid": L.EPI_BIAS_RESID, "gelu": L.EPI_BIAS_GELU,
          "gelu_act": L.EPI_BIAS_GELU_ACT, "dgelu": L.EPI_DGELU}[name]


def _operands(g, tier, M, N, K):
  """Logical A [M, K], B [N, K] as fp64 (bf16-representable)."""
  if tier == 1:
    r = 8 if K <= 4096 else 2
    A = torch.randint(-r, r + 1, (M, K), generator=g, device=DEV).double()
    B = torch.randint(-r, r + 1, (N, K), generator=g, device=DEV).double()
    return A, B

  def scaled(R):
    x = torch.randn(R, K, generator=g, device=DEV, dtype=F64)
    x *= torch.exp2(torch.randint(-6, 5, (R, 1), generator=g, device=DEV).double())
    x *= torch.exp2(torch.randint(-3, 4, (1, K), generator=g, device=DEV).double())
    x[::97] *= 256.0                                                   # outlier rows
    return x.to(BF16).double()
  return scaled(M), scaled(N)


def _run_case(ops, c, tier, seed):
  from big_vision_b200 import lib as L
  a_mn, b_mn, bn, mode, epi, alpha, M, N, K, splits, mod = c
  if tier == 2 and alpha == -4.0:
    alpha = -3.0
  g = torch.Generator(device=DEV)
  g.manual_seed(seed)
  A, B = _operands(g, tier, M, N, K)
  if tier == 1:
    bias = torch.randint(-16, 17, (N,), generator=g, device=DEV).double() / 4
    aux = torch.randint(-32, 33, (mod or M, N), generator=g, device=DEV).double() / 4
    d0 = torch.randint(-16, 17, (M, N), generator=g, device=DEV).double() / 4
  else:
    bias = torch.randn(N, generator=g, device=DEV, dtype=F64).float().double()
    aux = torch.randn(mod or M, N, generator=g, device=DEV, dtype=F64).to(BF16).double()
    d0 = torch.randn(M, N, generator=g, device=DEV, dtype=F64)
  if epi == "dgelu":
    aux = (torch.randn(M, N, generator=g, device=DEV, dtype=F64) * 3).to(BF16).double()
  out_dt = F32 if mode.startswith("f32") else BF16
  reduce_out = mode.endswith("add")
  d0 = d0.to(out_dt).double() if reduce_out else None
  eff_bn = 128 if mode == "bf16add" else (bn or (256 if N > 128 else 128))
  ranges = splits_of(M, N, K, eff_bn, splits, reduce_out, torch.cuda.get_device_properties(0).multi_processor_count)
  a_st = _nan_view(A.T if a_mn else A)
  b_st = _nan_view(B.T if b_mn else B)
  use_bias = epi in ("none", "bias", "resid", "gelu", "gelu_act")    # EPI_NONE gets one and must ignore it
  bias_v = _bias_buf(bias.float()) if use_bias else None
  aux_v = _nan_view(aux, extra_cols=0)[:aux.shape[0], :N] if epi in ("resid", "dgelu") else None
  buf, out = _out_buf(M, N, out_dt, None if d0 is None else d0.to(out_dt))
  buf2 = out2 = None
  if epi == "gelu":
    buf2, out2 = _out_buf(M, N, BF16)
  ops.gemm(a_st, b_st, a_mn=bool(a_mn), b_mn=bool(b_mn), out=out, bias=bias_v, aux=aux_v, aux_row_mod=mod,
           epilogue=_epi(L, epi), out2=out2, reduce_out=reduce_out, splits=splits, block_n=bn, alpha=alpha,
           M=M, N=N, K=K)
  torch.cuda.synchronize()
  _sentinel_intact(buf, M, N, "D")
  if buf2 is not None:
    _sentinel_intact(buf2, M, N, "D2")
  parts, errs = split_partials(A, B, ranges, model_error=tier == 2)
  if tier == 1:
    errs = [torch.zeros_like(p) for p in parts]
  eb = bias if epi in ("bias", "resid", "gelu", "gelu_act") else None
  aux_rows = aux[torch.arange(M, device=DEV) % mod] if mod else aux
  return dict(A=A, B=B, parts=parts, errs=errs, alpha=alpha, bias=eb, aux=aux_rows, d0=d0, out=out, out2=out2,
              mode=mode, epi=epi, ranges=ranges)


def _exact_precondition(r):
  """alpha sum|ab| + |bias| + |aux| + |D0| < 2^21: every value a multiple of 1/8 is exact in fp32."""
  mag = abs(r["alpha"]) * (r["A"].abs() @ r["B"].abs().T)
  if r["bias"] is not None:
    mag = mag + r["bias"].abs()
  if r["epi"] == "resid":
    mag = mag + r["aux"].abs()
  if r["d0"] is not None:
    mag = mag + r["d0"].abs()
  assert float(mag.max()) < 2.0 ** 21, "tier-1 data would not be exact in fp32"


@pytest.mark.parametrize("c", CASES, ids=_cid)
def test_tier1_exact(ops, c):
  """Integer operands: bit-exact outputs (bf16 multi-split reduce-adds and the GELU family bounded)."""
  r = _run_case(ops, c, 1, seed=zlib.crc32(_cid(c).encode()))
  _exact_precondition(r)
  mode, epi, alpha, out = r["mode"], r["epi"], r["alpha"], r["out"]
  exact = alpha * sum(r["parts"])                         # alpha * A B^T, exact
  pre = exact + (r["bias"] if r["bias"] is not None else 0.0)
  key = f"tier1::{_cid(c)}"
  if epi == "gelu":
    _same(r["out2"], pre.float().to(BF16), "D2 = bf16(exact + bias)")
  if epi in ("gelu", "gelu_act"):
    x = pre.float().to(BF16).double()
    ref = _gelu64(x)
    _check_r(key, out, ref, _ulp(ref, BF16) + 0.5 * x.abs() * _TANH_APPROX + 2.0 ** -20 * ref.abs(), "gelu")
    return
  if epi == "dgelu":
    dg, du = _dgelu64(r["aux"])
    dprop = (0.5 + r["aux"].abs() * du) * _TANH_APPROX
    ref, bound = gemm_bound(r["parts"], r["errs"], alpha, None, mode, d0=r["d0"], dgelu=(dg, dprop))
    _check_r(key, out, ref, bound, f"dgelu {mode}")
    return
  if epi == "resid":
    val = pre.float()
    if mode in ("bf16", "bf16add"):
      val = val.to(BF16).float()
    val = val + r["aux"].float()                           # the same fp32 addition as the kernel
  else:
    val = pre.float()
  if mode == "f32":
    _same(out, val, f"fp32 {epi}")
  elif mode == "bf16":
    _same(out, val.to(BF16), f"bf16 {epi}")
  elif mode == "f32add":
    _same(out, (r["d0"] + pre + (r["aux"] if epi == "resid" else 0.0)).float(), f"fp32 reduce-add {epi}")
  else:
    if len(r["ranges"]) == 1:
      _same(out, (r["d0"].float() + val.to(BF16).float()).to(BF16), f"bf16 reduce-add {epi}")
    else:
      ref, bound = gemm_bound(r["parts"], r["errs"], alpha, r["bias"], mode, d0=r["d0"], aux=r["aux"],
                              resid=epi == "resid")
      _check_r(key, out, ref, bound, f"bf16 reduce-add {epi}, {len(r['ranges'])} splits")


@pytest.mark.parametrize("c", CASES, ids=_cid)
def test_tier2_bound(ops, c):
  """Gaussian operands over several binades: |D - ref| within gemm_bound per element."""
  r = _run_case(ops, c, 2, seed=zlib.crc32(_cid(c).encode()) + 1)
  mode, epi, alpha, out = r["mode"], r["epi"], r["alpha"], r["out"]
  key = f"tier2::{_cid(c)}"
  if epi in ("gelu", "gelu_act"):
    ref, bound = gemm_bound(r["parts"], r["errs"], alpha, r["bias"], "bf16")
    if epi == "gelu":
      _check_r(key + "::D2", r["out2"], ref, bound, "D2")
      x = r["out2"].double()
      gref = _gelu64(x)
      _check(out, gref, _ulp(gref, BF16) + 0.5 * x.abs() * _TANH_APPROX + 2.0 ** -20 * gref.abs(), "gelu(D2)")
    else:
      # D = gelu(bf16(pre)): the pre-activation's error propagated by |gelu'| <= 1.13, then the tanh bound
      gref = _gelu64(ref)
      bnd = 1.13 * bound + _ulp(gref, BF16) + 0.5 * (ref.abs() + bound) * _TANH_APPROX + 2.0 ** -20 * gref.abs()
      _check_r(key, out, gref, bnd, "gelu_act")
    return
  if epi == "dgelu":
    dg, du = _dgelu64(r["aux"])
    dprop = (0.5 + r["aux"].abs() * du) * _TANH_APPROX
    ref, bound = gemm_bound(r["parts"], r["errs"], alpha, None, mode, d0=r["d0"], dgelu=(dg, dprop))
    _check_r(key, out, ref, bound, f"dgelu {mode}")
    return
  ref, bound = gemm_bound(r["parts"], r["errs"], alpha, r["bias"], mode, d0=r["d0"], aux=r["aux"],
                          resid=epi == "resid")
  if mode == "f32":
    bound = bound + _ulp(ref, F32)
  _check_r(key, out, ref, bound, f"{mode} {epi}")


COLSUM_EPIS = [("none", 0), ("bias", 0), ("gelu", 0), ("gelu_act", 0), ("resid", 0), ("resid", 49), ("dgelu", 0)]


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("epi,mod", COLSUM_EPIS)
def test_colsum_of_the_stored_output(ops, epi, mod, block_n):
  """colsum += column sums of the stored bf16 D, into a non-zero initial value, within the chain
  bound of colsum_add (two rows, three shuffles, 8 atomics per 128-row tile, the initial value).
  The values sit in [128, 256) with a fraction of 3/8 (bias 192.375 + 4 j, |j| <= 2, |acc| <= 32), so every bf16
  rounding of D goes the same way: a sum of unrounded values misses by 3/8 per row."""
  from big_vision_b200 import lib as L
  g = torch.Generator(device=DEV)
  g.manual_seed(block_n + mod + len(epi))
  M, N, K = 4097, 257, 8
  A = torch.randint(-2, 3, (M, K), generator=g, device=DEV).double()
  B = torch.randint(-2, 3, (N, K), generator=g, device=DEV).double()
  bias = torch.full((N,), 192.375, device=DEV) + torch.randint(-2, 3, (N,), generator=g, device=DEV) * 4.0
  aux = torch.randint(-32, 33, (mod or M, N), generator=g, device=DEV).to(BF16) / 4
  if epi == "dgelu":
    aux = (torch.randn(M, N, generator=g, device=DEV) * 3).to(BF16)
  init = torch.randn(N, generator=g, device=DEV) * 100
  cs_buf = torch.full((N + 8,), SENT[F32], device=DEV)
  cs_buf[:N] = init
  buf, out = _out_buf(M, N, BF16)
  out2 = _out_buf(M, N, BF16)[1] if epi == "gelu" else None
  ops.gemm(_nan_view(A), _nan_view(B), out=out, bias=None if epi == "dgelu" else _bias_buf(bias),
           aux=_nan_view(aux, extra_cols=0)[:aux.shape[0], :N] if epi in ("resid", "dgelu") else None,
           aux_row_mod=mod, epilogue=_epi(L, epi), out2=out2, block_n=block_n, M=M, N=N, K=K,
           colsum=cs_buf[:N])
  torch.cuda.synchronize()
  _sentinel_intact(buf, M, N, "D")
  assert bool((cs_buf[N:] == SENT[F32]).all()), "colsum written past N"
  D = out.double()
  assert not torch.isnan(D).any()
  ref = init.double() + D.sum(0)
  bound = colsum_chain(M) * U32 * (init.double().abs() + D.abs().sum(0))
  _check_r(f"colsum::{epi}-mod{mod}-bn{block_n}", cs_buf[:N], ref, bound, f"colsum {epi}")


def test_split_k_adds_bias_once(ops):
  """D += x w + bias with splits = 2 and with the automatic split count at M = N = 128, K = 4096:
  bias enters once, bit for bit (integer data)."""
  for splits in (2, 0):
    c = (0, 1, 0, "f32add", "bias", 1.0, 128, 128, 4096, splits, 0)
    r = _run_case(ops, c, 1, seed=7 + splits)
    _exact_precondition(r)
    assert len(r["ranges"]) > 1
    want = (r["d0"] + r["alpha"] * sum(r["parts"]) + r["bias"]).float()
    got = r["out"]
    if not torch.equal(got.view(torch.int32), want.view(torch.int32)):
      excess = (got.double() - want.double()) / r["bias"]
      ok = r["bias"].abs() > 0
      raise AssertionError(f"splits={len(r['ranges'])}: (got - want) / bias over nonzero bias: "
                           f"min {float(excess[:, ok].min()):.4f} max {float(excess[:, ok].max()):.4f}")


def test_print_error_bound_ratios():
  """One JSON line: the largest err / bound per test above (run after them, in file order)."""
  if RATIOS:
    print("GEMM_ERR_BOUND_RATIOS " + json.dumps({k: round(v, 4) for k, v in sorted(RATIOS.items())}))
