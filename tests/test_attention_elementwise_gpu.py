"""Element-wise fp64 parity of the attention kernels at every head dim (64, 72, 80, 96, 104) through
bv_attention_fwd_hd / bv_attention_bwd_hd.

q, k, v and dO are views into buffers holding NaN in the rows past N, the columns past H * dh and the
gap of a batch stride larger than N * ld; delta is NaN-filled before the backward; o, dq, dk and dv
are written into views whose surroundings hold a sentinel.  A read outside a logical extent reaches
an output as NaN, a write outside one changes the sentinel.  References are fp64 on the GPU, one head
at a time.

Exact and structural cases: q = 0 (every probability exactly 1 / Nk), one dominant key per row (the
output equals that key's v to bf16) in the first key block, at the last key of a ragged tail block,
and moving to a later block on every block (so every block rescales the whole accumulator by `corr`).

Bound cases (`fwd_bound`, `bwd_bound`): per element, built from fp64 products of absolute values.
  * Scores: S accumulates over dh in k16 wgmma steps, each modelled as one fp32 addition with error
    at most 2^-23 (|running sum| + sum |q k| of the step) (the tensor core's alignment may truncate;
    not documented), so |dS| <= (ksteps + 1) 2^-23 sum_d |q k|.  x = S * fl(scale * log2 e) in
    log2 units is off by scale log2e |dS| + 2 * 2^-24 |x|, and x - m by a further 2^-24 |x - m|; the
    row maximum m is a common shift whose error cancels between numerator and l.
  * ex2.approx.ftz.f32 is within 2 ulp (relative 2^-22) over its range, and lg2.approx.f32 within an
    absolute 2^-22.6 on the log of the mantissa: PTX ISA, section 9.7.3 (floating-point
    instructions), `ex2` and `lg2`.  Results below 2^-126 flush to zero (relative error 1).
  * O = sum_j bf16(p_j) v_j / l: eps_ij = 2^-8 (bf16 P: 8 significant bits, so the unit roundoff
    is 2^-8) + 2^-22 + ln2 * (error of x_ij); l is an fp32 sum of 16 NB + NB + 2 terms (NB key blocks); the P V accumulation adds (4 NB + 1) 2^-23, the corr
    and 1 / l scalings (NB + 2) 2^-24; then one bf16 ulp of O.
  * lse = (m + lg2 l) ln2: the P-weighted error of x, ex2's 2^-22 and l's chain in log2 units,
    lg2's 2^-22.6, two fp32 roundings.
  * Backward: P = ex2(x - fl(lse log2e)), so the lse bound enters P's relative error; dV like O with
    (4 QT + 1) 2^-23; dS = P (dP - delta) with dP's accumulation error, delta's error (computed from
    the stored bf16 O: the forward bound of O against |dO|, plus its 12-term fp32 chain), P's error,
    two fp32 roundings and the bf16 rounding 2^-8 |dS| before the dQ / dK products; dQ = scale dS K
    and dK = scale dS^T Q with (4 KT + 1) resp. (4 QT + 1) 2^-23 of accumulation and one bf16 ulp.
No constant is fitted to observed errors; test_print_error_bound_ratios prints the largest err / bound
of each test.
"""
import ctypes
import json
import math
import zlib

import numpy as np
import pytest
import torch

from test_kernel_edges_gpu import _check, _same, _ulp

pytestmark = pytest.mark.gpu
F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
U32, U_MMA, U_BF = 2.0 ** -24, 2.0 ** -23, 2.0 ** -8   # U_BF: bf16 has 8 significant bits
EX2_REL = 2.0 ** -22          # ex2.approx.ftz.f32: 2 ulp
LG2_ABS = 2.0 ** -22.6        # lg2.approx.f32: absolute, on the log2 of the mantissa
LOG2E, LN2 = 1.0 / math.log(2.0), math.log(2.0)
T = 64
DEV = "cuda"
NAN = float("nan")
SENT = -8192.0
HEAD_DIMS = (64, 72, 80, 96, 104)
RATIOS = {}


@pytest.fixture(scope="module")
def ops():
  from big_vision_b200 import lib, ops as _ops
  assert lib.load().bv_device_supported() == 1, "needs a compute-capability 9.x GPU"
  return _ops


def _f32(x):
  return float(np.float32(x))


# ---------------------------------------------------------------------------------------------------
# bounds (one head; q [B, Nq, dh], k / v [B, Nk, dh], do [B, Nq, dh] fp64; any device)
# ---------------------------------------------------------------------------------------------------
def fwd_bound(q, k, v, scale):
  """Reference O, lse and their bounds; also what the backward bound needs."""
  dh, Nk = q.shape[-1], k.shape[1]
  NB = -(-Nk // T)
  s = q @ k.transpose(1, 2)
  sabs = q.abs() @ k.abs().transpose(1, 2)
  sl2 = scale * LOG2E
  x = s * sl2
  m = x.max(-1, keepdim=True).values
  p = torch.exp2(x - m)
  l = p.sum(-1, keepdim=True)
  P = p / l
  O = P @ v
  lse = (m + torch.log2(l)) * LN2
  dS = (-(-dh // 16) + 1) * U_MMA * sabs
  dx = abs(sl2) * dS + 2 * U32 * x.abs()                       # error of x, before the shift
  eps = EX2_REL + LN2 * (dx + U32 * (x - m).abs())
  eps = torch.where(p * l.clamp_max(1.0) < 2.0 ** -125, torch.ones_like(eps), eps)   # flushed to zero
  ebar = (P * eps).sum(-1, keepdim=True)                        # relative error of l from its terms
  chain_l = 16 * NB + NB + 2
  vabs = v.abs()
  PV = P @ vabs
  bO = _ulp(O, BF16) + (P * (eps + U_BF)) @ vabs + (ebar + chain_l * U32 + (4 * NB + 1) * U_MMA
                                                    + (NB + 2) * U32) * PV
  dlog2 = (P * (dx + LOG2E * EX2_REL)).sum(-1) + LOG2E * (chain_l * U32 + ebar[..., 0]) + LG2_ABS \
      + U32 * (m[..., 0] + torch.log2(l[..., 0])).abs()
  blse = LN2 * dlog2 + 2 * U32 * lse[..., 0].abs()
  return dict(O=O, lse=lse[..., 0], bO=bO, blse=blse, P=P, x=x, dx=dx)


def bwd_bound(q, k, v, do, scale, f):
  """Reference dQ, dK, dV and their bounds from the forward's dict `f` (fwd_bound)."""
  dh, Nq, Nk = q.shape[-1], q.shape[1], k.shape[1]
  QT, KT = -(-Nq // T), -(-Nk // T)
  P, O, lse = f["P"], f["O"], f["lse"]
  dP = do @ v.transpose(1, 2)
  dPabs = do.abs() @ v.abs().transpose(1, 2)
  delta = (O * do).sum(-1, keepdim=True)
  dSr = P * (dP - delta)
  dQ = scale * dSr @ k
  dK = scale * dSr.transpose(1, 2) @ q
  dV = P.transpose(1, 2) @ do
  lse2 = lse[..., None] * LOG2E
  # P's relative error: x, lse (in log2 units, plus the rounding of lse * log2e), the subtraction, ex2
  xl = f["x"] - lse2
  eP = EX2_REL + LN2 * (f["dx"] + LOG2E * f["blse"][..., None] + 2 * U32 * lse2.abs() + U32 * xl.abs())
  eP = torch.where(torch.exp2(xl) < 2.0 ** -125, torch.ones_like(eP), eP)
  # dV = sum_i bf16(P_ij) dO_id
  doabs = do.abs()
  PtdO = P.transpose(1, 2) @ doabs
  bdV = _ulp(dV, BF16) + (P * (eP + U_BF)).transpose(1, 2) @ doabs + (4 * QT + 1) * U_MMA * PtdO
  # delta from the stored O: the forward bound against |dO| and a 12-term fp32 chain
  ddelta = (f["bO"] * doabs).sum(-1, keepdim=True) + 12 * U32 * ((O.abs() + f["bO"]) * doabs).sum(-1, keepdim=True)
  ddP = (-(-dh // 16) + 1) * U_MMA * dPabs
  r = (dP - delta).abs()
  edS = (P * eP * (r + ddP + ddelta) + P * (ddP + ddelta) + 2 * U32 * P * r) * (1 + 2.0 ** -6) \
      + U_BF * dSr.abs()
  dSabs = dSr.abs()
  sc = abs(scale)
  bdQ = _ulp(dQ, BF16) + sc * (edS @ k.abs()) + sc * ((4 * KT + 1) * U_MMA + U32) * (dSabs @ k.abs())
  bdK = _ulp(dK, BF16) + sc * (edS.transpose(1, 2) @ q.abs()) + \
      sc * ((4 * QT + 1) * U_MMA + U32) * (dSabs.transpose(1, 2) @ q.abs())
  return dict(dQ=dQ, dK=dK, dV=dV, bdQ=bdQ, bdK=bdK, bdV=bdV)


def colsum_chain(blocks_total):
  """tile_colsum: two rows per thread, three shuffles, one atomic per warp (4 per 64-row tile), the
  initial value."""
  return 2 + 3 + 4 * blocks_total + 1


# ---------------------------------------------------------------------------------------------------
# buffers and calls
# ---------------------------------------------------------------------------------------------------
def _layout(B, N, C, pad_rows=2, pad_cols=8, gap=64):
  ld = C + pad_cols
  return ld, (N + pad_rows) * ld + gap


def _poisoned(data):
  """`data` [B, N, C] as a view into a NaN buffer (rows past N, columns past C, a batch-stride gap)."""
  B, N, C = data.shape
  ld, bs = _layout(B, N, C)
  buf = torch.full((B * bs,), NAN, dtype=BF16, device=DEV)
  view = buf.as_strided((B, N, C), (bs, ld, 1))
  view.copy_(data)
  return view


def _sentinel_out(B, N, C):
  """(buffer, view): NaN inside the view, the sentinel everywhere else."""
  ld, bs = _layout(B, N, C, pad_rows=1, pad_cols=16, gap=8)
  buf = torch.full((B * bs,), SENT, dtype=BF16, device=DEV)
  view = buf.as_strided((B, N, C), (bs, ld, 1))
  view.fill_(NAN)
  return buf, view


def _sentinel_intact(buf, view, what):
  mask = torch.ones(buf.shape, dtype=torch.bool, device=DEV)
  mask.as_strided(view.shape, view.stride()).fill_(False)
  assert bool((buf[mask] == SENT).all()), f"{what}: written outside its view"


def _fwd(ops, q, k, v, H, dh, scale):
  from big_vision_b200 import lib as L
  B, Nq, C = q.shape
  obuf, o = _sentinel_out(B, Nq, C)
  lse = torch.full((B, H, Nq), NAN, dtype=F32, device=DEV)
  args = ops._attn_args(q, k, v, o, lse, H, scale)
  L.call("bv_attention_fwd_hd", ctypes.byref(args), dh, ops._stream())
  torch.cuda.synchronize()
  _sentinel_intact(obuf, o, "o")
  return o, lse


def _bwd(ops, do, q, k, v, o, lse, H, dh, scale, colsums=None):
  from big_vision_b200 import lib as L
  B, Nq, C = q.shape
  Nk = k.shape[1]
  f = ops._attn_args(q, k, v, o, lse, H, scale)
  outs = [_sentinel_out(B, Nq, C), _sentinel_out(B, Nk, C), _sentinel_out(B, Nk, C)]
  delta = torch.full((B, H, Nq), NAN, dtype=F32, device=DEV)
  dop, lddo, bsdo = ops._attn_view(do)
  views = [ops._attn_view(t[1]) for t in outs]
  cs = colsums or (None, None, None)
  args = L.AttnBwdArgs(fwd=f, d_o=dop, lddo=lddo, bsdo=bsdo, dq=views[0][0], dk=views[1][0], dv=views[2][0],
                       lddq=views[0][1], lddk=views[1][1], lddv=views[2][1],
                       bsdq=views[0][2], bsdk=views[1][2], bsdv=views[2][2],
                       dq_colsum=cs[0].data_ptr() if cs[0] is not None else None,
                       dk_colsum=cs[1].data_ptr() if cs[1] is not None else None,
                       dv_colsum=cs[2].data_ptr() if cs[2] is not None else None,
                       delta=delta.data_ptr())
  L.call("bv_attention_bwd_hd", ctypes.byref(args), dh, ops._stream())
  torch.cuda.synchronize()
  for (buf, view), name in zip(outs, ("dq", "dk", "dv")):
    _sentinel_intact(buf, view, name)
  return outs[0][1], outs[1][1], outs[2][1]


def _heads(t, H):
  B, N, C = t.shape
  return [t[:, :, h * (C // H):(h + 1) * (C // H)] for h in range(H)]


def _record(key, got, ref, bound):
  r = float(((got.double() - ref).abs() / bound.clamp_min(1e-300)).max())
  RATIOS[key] = max(RATIOS.get(key, 0.0), r)


def _check_r(key, got, ref, bound, what):
  _check(got, ref, bound, what)
  _record(key, got, ref, bound)


def _gen(seed):
  g = torch.Generator(device=DEV)
  g.manual_seed(seed)
  return g


def _ints_nonzero(g, *shape):
  """integers in +-[1, 8]"""
  mag = torch.randint(1, 9, shape, generator=g, device=DEV)
  sgn = torch.randint(0, 2, shape, generator=g, device=DEV) * 2 - 1
  return (mag * sgn).to(BF16)


# ---------------------------------------------------------------------------------------------------
# exact and structural cases
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dh", HEAD_DIMS)
@pytest.mark.parametrize("Nk", [1, 64, 197, 2048])
def test_zero_queries_average_every_key_once(ops, dh, Nk):
  """q = 0: every probability is 1 / Nk.  With integer v, O = fl(fl(sum v) * fl(1 / Nk)) rounded to
  bf16 (exact for a power-of-two Nk); a key past Nk that leaks in, or a key inside it that is
  masked, changes the sum.  lse = ln Nk within lg2's error."""
  g = _gen(dh * 7 + Nk)
  B, H, Nq = 2, 2, 65
  C = H * dh
  q = torch.zeros(B, Nq, C, dtype=BF16, device=DEV)
  k = torch.randn(B, Nk, C, generator=g, device=DEV).to(BF16)
  v = _ints_nonzero(g, B, Nk, C)
  scale = _f32(1 / math.sqrt(dh))
  o, lse = _fwd(ops, _poisoned(q), _poisoned(k), _poisoned(v), H, dh, scale)
  sv = v.double().sum(1, keepdim=True).float()                      # exact in fp32
  want = (sv * (torch.ones(1, device=DEV) / Nk)).expand(B, Nq, C)
  if Nk & (Nk - 1) == 0:
    _same(o, want.to(BF16), "O = mean of v")
  else:
    ref = v.double().mean(1, keepdim=True).expand(B, Nq, C)
    _check(o, ref, _ulp(ref, BF16) + 2 * U32 * ref.abs(), "O = mean of v")
  lref = torch.full_like(lse, math.log(Nk), dtype=F64)
  _check_r(f"zero_q::dh{dh}-Nk{Nk}::lse", lse, lref, LN2 * LG2_ABS + 3 * U32 * lref.abs() + 1e-30, "lse")


def _peak_scores(Nk, placement):
  """Integer scores t_j (exact in bf16) of every key: one dominant key per row."""
  t = torch.zeros(Nk, dtype=F64)
  if placement == "first":
    t[min(5, Nk - 1)] = 48.0
  elif placement == "last":
    t[Nk - 1] = 48.0
  else:                                # 24 per block, +48 at a block-dependent position
    nb = -(-Nk // T)
    t = torch.tensor([24.0 * (j // T) for j in range(Nk)], dtype=F64)
    for b in range(nb):
      width = min(T, Nk - b * T)
      t[b * T + (7 * b + 3) % width] += 48.0
  return t


@pytest.mark.parametrize("dh", HEAD_DIMS)
@pytest.mark.parametrize("placement,Nk", [("first", 197), ("last", 197), ("last", 577), ("moving", 2048),
                                          ("moving", 577), ("moving", 65)])
def test_dominant_key_gives_its_value(ops, dh, placement, Nk):
  """scale = 1, q = e_0, k_j = t_j e_0: scores t_j with the peak at least 24 above every other key
  (34.6 in log2 units; 69 for the within-block gap), so O equals the peak's integer v exactly.
  'moving': the row maximum grows on every key block, so every block rescales the whole
  accumulator (registers 32 .. R - 1 included at dh > 64) by corr; the last block may be ragged."""
  g = _gen(dh + Nk + len(placement))
  B, H, Nq = 2, 2, 63
  C = H * dh
  t = _peak_scores(Nk, placement).to(DEV)
  q = torch.zeros(B, Nq, C, dtype=BF16, device=DEV)
  k = torch.randn(B, Nk, C, generator=g, device=DEV).to(BF16)
  for h in range(H):
    q[:, :, h * dh] = 1.0
    k[:, :, h * dh] = t.to(BF16)
    k[:, :, h * dh + 1:(h + 1) * dh] = 0.0
  v = _ints_nonzero(g, B, Nk, C)
  o, lse = _fwd(ops, _poisoned(q), _poisoned(k), _poisoned(v), H, dh, 1.0)
  jstar = int(t.argmax())
  _same(o, v[:, jstar:jstar + 1].expand(B, Nq, C).contiguous(), f"O = v[{jstar}]")
  lref = torch.logsumexp(t, 0).expand_as(lse)
  f_b = fwd_bound(q[:, :, :dh].double(), k[:, :, :dh].double(), v[:, :, :dh].double(), 1.0)
  _check_r(f"peak::dh{dh}-{placement}-Nk{Nk}::lse", lse, lref, f_b["blse"].max() + 0 * lref, "lse")


# ---------------------------------------------------------------------------------------------------
# bound cases
# ---------------------------------------------------------------------------------------------------
# (B, H, Nq, Nk); Nq, Nk from {1, 63, 64, 65, 197, 577, 2048}, the So400m and text geometries
SHAPES = {"s1": (2, 2, 1, 197), "s2": (1, 3, 65, 63), "s3": (2, 2, 577, 64), "s4": (1, 2, 63, 2048),
          "s5": (1, 1, 2048, 65), "s6": (2, 3, 197, 65), "so400m": (2, 16, 729, 729), "text": (4, 12, 64, 64)}
BOUND_CASES = [(dh, s, sc) for dh in HEAD_DIMS for s, sc in (("s1", None), ("s2", 1.0), ("s4", None),
                                                            ("s5", 0.05))]
BOUND_CASES += [(64, "s3", None), (64, "s6", None), (104, "s3", 1.0), (72, "so400m", None), (64, "text", None),
                (96, "s3", 0.05)]


def _random_qkv(g, B, H, Nq, Nk, dh):
  C = H * dh
  q = torch.randn(B, Nq, C, generator=g, device=DEV)
  q[:, ::37] *= 4.0                                                  # a few peaky rows
  k = torch.randn(B, Nk, C, generator=g, device=DEV)
  k *= torch.exp2(torch.randint(-2, 2, (1, Nk, 1), generator=g, device=DEV).float())
  v = torch.randn(B, Nk, C, generator=g, device=DEV)
  v *= torch.exp2(torch.randint(-3, 4, (1, 1, C), generator=g, device=DEV).float())   # columns over binades
  do = torch.randn(B, Nq, C, generator=g, device=DEV)
  return q.to(BF16), k.to(BF16), v.to(BF16), do.to(BF16)


def _bid(c):
  return f"dh{c[0]}-{c[1]}-scale{c[2]}"


@pytest.mark.parametrize("c", BOUND_CASES, ids=_bid)
def test_forward_and_backward_within_bound(ops, c):
  """Random q, k, v, dO: O, lse, dQ, dK, dV within fwd_bound / bwd_bound per element; the fused column
  sums of dq / dk / dv against the stored outputs within the tile_colsum chain."""
  dh, sname, scale = c
  B, H, Nq, Nk = SHAPES[sname]
  scale = _f32(1 / math.sqrt(dh) if scale is None else scale)
  g = _gen(zlib.crc32(_bid(c).encode()))
  q, k, v, do = _random_qkv(g, B, H, Nq, Nk, dh)
  qp, kp, vp, dop = (_poisoned(t) for t in (q, k, v, do))
  o, lse = _fwd(ops, qp, kp, vp, H, dh, scale)
  C = H * dh
  inits = [torch.randn(C, generator=g, device=DEV) * 10 for _ in range(3)]
  cs = [t.clone() for t in inits]
  dq, dk, dv = _bwd(ops, dop, qp, kp, vp, o, lse, H, dh, scale, colsums=cs)
  key = _bid(c)
  for h, (qh, kh, vh, doh) in enumerate(zip(*(_heads(t.double(), H) for t in (q, k, v, do)))):
    sl = slice(h * dh, (h + 1) * dh)
    f = fwd_bound(qh, kh, vh, scale)
    _check_r(key + "::O", o[:, :, sl], f["O"], f["bO"], f"O head {h}")
    _check_r(key + "::lse", lse[:, h], f["lse"], f["blse"], f"lse head {h}")
    b = bwd_bound(qh, kh, vh, doh, scale, f)
    _check_r(key + "::dV", dv[:, :, sl], b["dV"], b["bdV"], f"dV head {h}")
    _check_r(key + "::dQ", dq[:, :, sl], b["dQ"], b["bdQ"], f"dQ head {h}")
    _check_r(key + "::dK", dk[:, :, sl], b["dK"], b["bdK"], f"dK head {h}")
  for name, got, init, out, n in (("dq_colsum", cs[0], inits[0], dq, Nq), ("dk_colsum", cs[1], inits[1], dk, Nk),
                                  ("dv_colsum", cs[2], inits[2], dv, Nk)):
    D = out.double().reshape(-1, C)
    ref = init.double() + D.sum(0)
    bound = colsum_chain(B * -(-n // T)) * U32 * (init.double().abs() + D.abs().sum(0))
    _check_r(key + "::" + name, got, ref, bound, name)


def test_print_error_bound_ratios():
  """One JSON line: the largest err / bound per test above (run after them, in file order)."""
  if RATIOS:
    print("ATTN_ERR_BOUND_RATIOS " + json.dumps({k: round(v, 4) for k, v in sorted(RATIOS.items())}))
