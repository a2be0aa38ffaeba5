"""Element-wise fp64 parity for the small kernels of the C ABI, at the shapes, dtypes and edges where
they go wrong: scalar tails, ragged blocks, strided views, aliased outputs, zero rows, every bf16 input
of GELU and tanh, and the losses at their operating point.

Every comparison is per element (`_check`) against a float64 reference computed in the test, never
against the tensor maximum, so an error confined to small-magnitude elements fails.  Three kinds of
bound are used:
  * bit-exact: data movement and single roundings whose result torch computes the same way;
  * `ulp(ref)`: one unit in the last place of the output dtype at the fp64 value, i.e. the result is
    one of the two representable neighbours of the exact value (plus, where stated, the propagated
    error of an fp32 intermediate the kernel rounds on the way);
  * the summation bound c * 2^-24 * sum|terms| of each output element, c the length of the longest
    chain of fp32 additions in the kernel's summation order (the standard first-order bound of
    recursive summation), stated where it is used.
"""
import json
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
F64 = torch.float64
BF16 = torch.bfloat16
U32 = 2.0 ** -24            # unit roundoff of fp32
DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
  from big_vision_b200 import lib, ops as _ops
  assert lib.load().bv_device_supported() == 1, "needs a compute-capability 9.x GPU"
  return _ops


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _ulp(ref, dtype):
  """Spacing of `dtype` at |ref| (fp64), floored at the spacing of the smallest normal number."""
  mant = 7 if dtype == BF16 else 23
  e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126)))
  return torch.exp2(e - mant)


def _check(got, ref, bound, what):
  """|got - ref| <= bound element by element (equal infinities and equal values always pass)."""
  got = got.detach().to(F64)
  ref = ref.detach().to(device=got.device, dtype=F64)
  bound = torch.as_tensor(bound, dtype=F64, device=got.device).expand_as(ref)
  assert got.shape == ref.shape, (what, got.shape, ref.shape)
  assert not torch.isnan(got[~torch.isnan(ref)]).any(), f"{what}: NaN where the reference is finite"
  err = (got - ref).abs()
  ok = (got == ref) | (err <= bound)
  if not bool(ok.all()):
    bad = (~ok).nonzero()[0].tolist()
    i = tuple(bad)
    raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements out of bound; first at {i}: "
                         f"got {got[i].item()!r} ref {ref[i].item()!r} err {err[i].item():.3e} "
                         f"bound {bound[i].item():.3e}")


def _same(got, want, what):
  """Bit-identical, except that any NaN matches any NaN."""
  assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape)
  it = torch.int16 if got.dtype == BF16 else torch.int32
  same = (got.view(it) == want.view(it)) | (torch.isnan(got) & torch.isnan(want))
  assert bool(same.all()), f"{what}: {int((~same).sum())} elements differ, first at {(~same).nonzero()[0].tolist()}"


def _gen(seed):
  g = torch.Generator(device=DEV)
  g.manual_seed(seed)
  return g


def _randn(g, *shape, scale=1.0, dtype=torch.float32):
  return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def _grid_chain(work, cap, per_item):
  """Longest fp32 addition chain of a grid-stride kernel (256 threads, min(ceil(work/256), cap)
  blocks) that adds `per_item` terms per item into a thread partial, reduces the block with two
  5-level warp trees and adds the block partials into the output with one atomic each."""
  blocks = max(1, min((work + 255) // 256, cap))
  iters = (work + blocks * 256 - 1) // (blocks * 256)
  return iters * per_item + 1 + 10 + blocks + 1


# ---------------------------------------------------------------------------------------------------
# bit-exact data movement and single roundings
# ---------------------------------------------------------------------------------------------------
_SPECIAL = [0.0, -0.0, 1.0, -1.0, float("inf"), float("-inf"), float("nan"), 3.0e38, -3.4e38,
            1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -8 + 2.0 ** -20,     # ties to even, above a tie
            2.0 ** -130, -2.0 ** -133, 2.0 ** -126, 1.5 * 2.0 ** -127, 2.0 ** -149]  # bf16 subnormals


@pytest.mark.parametrize("n", [1, 2, 3, 5, 4 * 1001 + 3, 17])
def test_cast_both_directions_bit_exact(ops, n):
  """fp32 -> bf16 rounds to nearest even (ties, +-inf, NaN, overflow to inf, subnormals) exactly like
  torch.Tensor.to; bf16 -> fp32 is exact.  n % 4 != 0 runs the scalar tail after the 4-wide body."""
  g = _gen(n)
  x = _randn(g, n, scale=3.0)
  sp = torch.tensor(_SPECIAL, device=DEV)
  x[:min(n, len(sp))] = sp[:min(n, len(sp))]
  x[-1] = sp[(n * 7) % len(sp)]                 # a special value in the scalar tail too
  y = ops.cast(x, torch.empty(n, dtype=BF16, device=DEV))
  _same(y, x.to(BF16), "fp32->bf16")
  z = ops.cast(y, torch.empty(n, device=DEV))
  _same(z, y.float(), "bf16->fp32")
  z = ops.cast(x, torch.empty(n, device=DEV))
  _same(z, x, "fp32->fp32")


@pytest.mark.parametrize("n,N0,d", [(3, 196, 64), (2, 49, 1024), (1, 1, 8)])
def test_concat_and_drop_cls_bit_exact(ops, n, N0, d):
  g = _gen(N0 + d)
  x = _randn(g, n * N0, d, dtype=BF16)
  cls = _randn(g, d)
  out = ops.concat_cls(x, cls, n, N0).view(n, N0 + 1, d)
  _same(out[:, 0], cls.to(BF16).expand(n, d), "cls row")
  _same(out[:, 1:], x.view(n, N0, d), "patch rows")
  back = ops.drop_cls(out.view(n * (N0 + 1), d), n, N0)
  _same(back, x, "drop_cls")


@pytest.mark.parametrize("with_b", [False, True])
def test_row_select_bit_exact(ops, with_b):
  g = _gen(3)
  n, N, d = 6, 50, 72
  a = _randn(g, n * N, d, dtype=BF16)
  b = _randn(g, n * N, d, dtype=BF16) if with_b else None
  mask = torch.tensor([1.0, 0.0, 0.0, 1.0, 1.0, 0.0], device=DEV)
  out = ops.row_select(a, b, mask, n, N).view(n, N, d)
  other = b.view(n, N, d) if with_b else torch.zeros(n, N, d, dtype=BF16, device=DEV)
  want = torch.where(mask.view(n, 1, 1) != 0, a.view(n, N, d), other)
  _same(out, want, "row_select")


@pytest.mark.parametrize("xdt,ydt", [(BF16, BF16), (torch.float32, torch.float32), (BF16, torch.float32),
                                     (torch.float32, BF16)])
def test_broadcast_row(ops, xdt, ydt):
  """Without `row` the copy is one rounding that torch does the same way (bit-exact); with `row` the
  fp32 sum x + row is rounded once (fp32 out) or rounded again to bf16: within 1 ulp of the fp64 sum."""
  g = _gen(5)
  d, rows = 200, 37
  x = _randn(g, 1, d, dtype=xdt)
  row = _randn(g, d, scale=0.3)
  _same(ops.broadcast_row(x, rows, out_dtype=ydt), x.to(ydt).expand(rows, d).contiguous(), "broadcast")
  ref = (x.double() + row.double()).expand(rows, d)
  _check(ops.broadcast_row(x, rows, row=row, out_dtype=ydt), ref, _ulp(ref, ydt), "broadcast + row")


@pytest.mark.parametrize("xdt,ydt", [(BF16, BF16), (torch.float32, torch.float32), (BF16, torch.float32)])
def test_pool_token_mode_and_pool_bwd(ops, xdt, ydt):
  """Token pooling and its backward are data movement (bit-exact).  The mean-pool backward is
  dy * fl(1/N): within 1 ulp of dy / N in the output dtype."""
  g = _gen(9)
  n, N, d = 5, 197, 96
  x = _randn(g, n * N, d, dtype=xdt)
  _same(ops.pool_fwd(x, n, N, 1, tok=196, out_dtype=ydt), x.view(n, N, d)[:, 196].to(ydt), "token pool")
  _same(ops.pool_fwd(x, n, N, 1, tok=0, out_dtype=ydt), x.view(n, N, d)[:, 0].to(ydt), "token pool 0")
  dy = _randn(g, n, d, dtype=xdt)
  dx = ops.pool_bwd(dy, n, N, 1, tok=7, dx_dtype=ydt).view(n, N, d)
  want = torch.zeros(n, N, d, dtype=ydt, device=DEV)
  want[:, 7] = dy.to(ydt)
  _same(dx, want, "token pool bwd")
  dx = ops.pool_bwd(dy, n, N, 0, dx_dtype=ydt).view(n, N, d)
  ref = (dy.double() / N).view(n, 1, d).expand(n, N, d)
  _check(dx, ref, _ulp(ref, ydt) + U32 * ref.abs(), "mean pool bwd")      # + the rounding of 1/N


@pytest.mark.parametrize("P,C", [(14, 3), (14, 1), (32, 3), (32, 1)])
def test_patchify_layout_and_zero_pad(ops, P, C):
  """Patch extraction in the (ph, pw, c) order of the HWIO conv kernel, rounded once to bf16; the
  round_up(P*P*C, 8) - P*P*C pad columns (4 of 592 at P = 14, C = 3) are written as exact zeros."""
  from big_vision_b200 import lib as L
  g = _gen(P * 10 + C)
  n, H, W = 2, 2 * P, 3 * P
  img = _randn(g, n, H, W, C)
  K = P * P * C
  Kp = (K + 7) // 8 * 8
  out = torch.full((n * 2 * 3, Kp), float("nan"), dtype=BF16, device=DEV)   # NaN: unwritten shows up
  L.call("bv_patchify", ops._p(img), ops._p(out), n, H, W, C, P, ops._stream())
  ref = img.reshape(n, 2, P, 3, P, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, K)
  _same(out[:, :K], ref.to(BF16), "patches")
  _same(out[:, K:], torch.zeros(out.shape[0], Kp - K, dtype=BF16, device=DEV), "pad columns")
  if P == 14:
    u8 = torch.randint(0, 256, (n, H, W, C), generator=g, device=DEV, dtype=torch.uint8)
    out8 = torch.full_like(out, float("nan"))
    L.call("bv_patchify_u8", ops._p(u8), ops._p(out8), n, H, W, C, P, -1.0, 1.0, 0.0, 255.0, 0, ops._stream())
    # fp32, each operation rounded separately (numpy; torch divides by a scalar as a reciprocal product)
    f = np.float32
    vr = f(-1.0) + (u8.cpu().numpy().astype(f) - f(0.0)) / f(255.0) * f(2.0)
    assert vr.dtype == np.float32
    want = torch.full_like(out, float("nan"))
    L.call("bv_patchify", ops._p(torch.from_numpy(vr).to(DEV)), ops._p(want), n, H, W, C, P, ops._stream())
    _same(out8, want, "patchify_u8")


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
@pytest.mark.parametrize("aliased", [False, True])
def test_axpby(ops, dtype, aliased):
  """out = a x + b y.  With a = b = 1 (every call in the models: gradient accumulation, often with
  `out` aliasing `x`) the sum is rounded once: within 1 ulp of the fp64 value.  With general a, b the
  compiler contracts one product into an FMA, so the other product's fp32 rounding (2^-24 of it) is
  added to the bound."""
  g = _gen(11)
  n = 4 * 1000 + 3
  x = _randn(g, n, dtype=dtype)
  y = _randn(g, n, scale=1e-3, dtype=dtype)
  y[:16] = -x[:16]                                  # exact cancellation to zero
  for a, b in ((1.0, 1.0), (0.75, -3.0)):
    xd, yd = x.double(), y.double()
    ref = a * xd + b * yd
    bound = _ulp(ref, dtype)
    if (a, b) != (1.0, 1.0):
      bound = bound + U32 * torch.maximum((a * xd).abs(), (b * yd).abs())
    if aliased:
      xx = x.clone()
      out = ops.axpby(xx, y, a, b, out=xx)
      assert out.data_ptr() == xx.data_ptr()
    else:
      out = ops.axpby(x, y, a, b)
    _check(out, ref, bound, f"axpby a={a} b={b}")


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_embed_fwd_and_bwd(ops, dtype):
  """Forward: table[id] + pos rounded once to fp32, then (bf16 out) to bf16: within 1 ulp.  Backward
  with a `dtype` cotangent: dtable by fp32 atomics (chain = number of occurrences of the id + 1),
  dpos by a sequential sum over the batch (chain = n + 1)."""
  g = _gen(13)
  n, Ln, d, vocab = 9, 16, 72, 40
  ids = torch.randint(0, vocab, (n, Ln), generator=g, device=DEV, dtype=torch.int32)
  ids[:, -3:] = 1                                     # the pad id, many duplicates
  table, pos = _randn(g, vocab, d), _randn(g, Ln, d)
  e = ops.embed_fwd(ids, table, pos, out_dtype=dtype)
  ref = (table.double()[ids.long()] + pos.double()[None]).reshape(-1, d)
  _check(e, ref, _ulp(ref, dtype), "embed_fwd")
  dy = _randn(g, n * Ln, d, dtype=dtype)
  dt = _randn(g, vocab, d)
  dp = _randn(g, Ln, d)
  dt0, dp0 = dt.clone(), dp.clone()
  ops.embed_bwd(ids, dy, dt, dp)
  oh = torch.nn.functional.one_hot(ids.flatten().long(), vocab).double()           # [n*Ln, vocab]
  ref_t = dt0.double() + oh.T @ dy.double()
  cnt = oh.sum(0)[:, None]
  _check(dt, ref_t, (cnt + 2) * U32 * (dt0.double().abs() + oh.T @ dy.double().abs()), "embed_bwd dtable")
  ref_p = dp0.double() + dy.double().view(n, Ln, d).sum(0)
  _check(dp, ref_p, (n + 2) * U32 * (dp0.double().abs() + dy.double().abs().view(n, Ln, d).sum(0)),
         "embed_bwd dpos")


# ---------------------------------------------------------------------------------------------------
# reductions: the summation bound
# ---------------------------------------------------------------------------------------------------
def _colsum_chain(rows):
  """colsum_kernel: each of 8 row lanes sums every 8th row of a 512-row block (<= 64 terms), the 8
  lane partials are added in sequence, then one atomic per 512-row block onto the initial value."""
  return -(-min(rows, 512) // 8) + 8 + -(-rows // 512) + 2


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
@pytest.mark.parametrize("rows", [1, 7, 511, 512, 513, 4 * 512 + 25])
def test_colsum(ops, dtype, rows):
  """out[c] += sum_r x[r, c] over a strided view (ld > cols, cols not a multiple of 256) into a
  non-zero initial `out`."""
  g = _gen(rows)
  cols, ld = 1000, 1032
  buf = _randn(g, rows, ld, dtype=dtype)
  buf[:, cols:] = float("nan")                        # read past the view: NaN in the result
  x = buf[:, :cols]
  x[rows // 2, :cols // 2] = 0.0
  out = _randn(g, cols)
  out0 = out.double().clone()
  ops.colsum(x, out)
  xd = x.double()
  _check(out, out0 + xd.sum(0), _colsum_chain(rows) * U32 * (out0.abs() + xd.abs().sum(0)), "colsum")


def test_colsum_of_the_patch_embedding_view(ops):
  """PatchEmbedding.bwd: the column sums of dx [n, N, d] viewed as [n, N*d] (cls and pos-embedding
  gradients), bf16, n = 256 images, N = 197 tokens, d = 64."""
  g = _gen(21)
  n, N, d = 256, 197, 64
  dx = _randn(g, n * N, d, dtype=BF16)
  out = torch.zeros(N * d, device=DEV)
  ops.colsum(dx.view(n, N * d), out)
  xd = dx.double().view(n, N * d)
  _check(out, xd.sum(0), _colsum_chain(n) * U32 * xd.abs().sum(0), "colsum [n, N*d]")


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_pool_fwd_mean(ops, dtype):
  """Mean over N tokens: a sequential fp32 sum (chain N) divided by N, rounded to the output
  dtype (bf16 input -> fp32 output as the ViT gap head calls it, and bf16 -> bf16)."""
  g = _gen(23)
  n, N, d = 4, 257, 136
  x = _randn(g, n * N, d, dtype=BF16)
  x.view(n, N, d)[:, :, :8] += 30.0                   # a large common offset: cancellation-free sums
  y = ops.pool_fwd(x, n, N, 0, out_dtype=dtype)
  xd = x.double().view(n, N, d)
  ref = xd.mean(1)
  _check(y, ref, _ulp(ref, dtype) + (N + 2) * U32 * xd.abs().sum(1) / N, "mean pool")


@pytest.mark.parametrize("n", [1, 2, 3, 4 * 37 + 1, 4 * 37 + 2, 4 * 37 + 3, 4 * 2 ** 20 + 3])
def test_sumsq(ops, n):
  """out[0] += sum x^2, into a non-zero initial value; n % 4 != 0 takes the scalar tail, the last
  size spans every block of the grid."""
  g = _gen(n)
  x = _randn(g, n)
  out = torch.tensor([2.5], device=DEV)
  ops.sumsq(x, out)
  xd = x.double()
  s = (xd * xd).sum()
  chain = _grid_chain(n // 4, _sms() * 8, 4)
  _check(out, (2.5 + s).view(1), (chain + 1) * U32 * (2.5 + s).view(1), "sumsq")


def _f32(v):
  return float(np.float32(v))


def _clip_scale(gsq, grad_mult, clip):
  gs = grad_mult
  if clip > 0:
    gn = math.sqrt(gsq) * grad_mult
    if not gn < clip:
      gs *= clip / gn
  return gs


@pytest.mark.parametrize("mu_dtype", [torch.float32, BF16])
@pytest.mark.parametrize("clip", [0.0, 1e4, 0.5])             # off, enabled but inactive, active
def test_adam_step_state_and_norms(ops, mu_dtype, clip):
  """Four Adam steps on random gradients with grad_mult != 1.  Each step is checked element-wise
  against an fp64 step from the kernel's own previous state (fp32 hyperparameters): params, nu, mu
  (1 ulp of its dtype) plus an fp32 term of 64 * 2^-24 of the update's parts; the bf16 shadow equals
  bf16(params); upd_sq and param_sq against fp64 sums of the applied update and the new params."""
  g = _gen(31)
  n = 4 * 30011
  p = _randn(g, n)
  mu = torch.zeros(n, dtype=mu_dtype, device=DEV)
  nu = torch.zeros(n, device=DEV)
  p16 = torch.empty(n, dtype=BF16, device=DEV)
  lr, b1, b2, eps, wd, gm = 1e-3, 0.9, 0.95, 1e-8, 1e-4, 0.37
  f = {k: _f32(v) for k, v in dict(lr=lr, b1=b1, b2=b2, eps=eps, wd=wd, gm=gm).items()}
  chain = _grid_chain(n // 4, _sms() * 8, 4)
  for step in range(1, 5):
    gr = _randn(g, n, scale=2.0)
    gsq = (gr.double() ** 2).sum()
    gsq_t = torch.tensor([gsq], dtype=torch.float32, device=DEV)
    P, M, V = p.double(), mu.double(), nu.double()
    us, ps = torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
    ops.adam_step(p, gr, mu, nu, p16, lr_eff=lr, b1=b1, b2=b2, eps=eps, wd_eff=wd, step=step, grad_mult=gm,
                  clip_norm=clip, gnorm_sq=gsq_t, upd_sq=us, param_sq=ps)
    gs = _clip_scale(float(gsq_t), f["gm"], clip)
    grs = gr.double() * gs
    m1 = f["b1"] * M + (1 - f["b1"]) * grs
    v1 = f["b2"] * V + (1 - f["b2"]) * grs * grs
    bc1, bc2 = 1 - f["b1"] ** step, 1 - f["b2"] ** step
    den = torch.sqrt(v1 / bc2) + f["eps"]
    step_dir = (m1 / bc1) / den
    upd = -(f["lr"] * step_dir + f["wd"] * P)
    p1 = P + upd
    dm1 = 8 * U32 * (f["b1"] * M.abs() + grs.abs())      # m1 may cancel: its absolute error
    # the division chain and the fp32 powf in the bias corrections: 128 * 2^-24 relative
    noise = 128 * U32 * (f["lr"] * step_dir.abs() + f["wd"] * P.abs()) + f["lr"] * dm1 / bc1 / den
    _check(p, p1, _ulp(p1, torch.float32) + noise, f"params step {step}")
    _check(nu, v1, _ulp(v1, torch.float32) + 16 * U32 * v1, f"nu step {step}")
    _check(mu, m1, _ulp(m1, mu_dtype) + dm1, f"mu step {step}")
    _same(p16, p.to(BF16), "bf16 shadow")
    applied = p.double() - P
    ref_us = (applied * applied).sum()
    # the kernel sums the unrounded update: |upd - applied| <= ulp(p) / 2 per element
    slack = (applied.abs() * _ulp(p.double(), torch.float32)).sum()
    _check(us, ref_us.view(1), ((chain + 1) * U32 * ref_us + 2 * slack).view(1), f"upd_sq step {step}")
    ref_ps = (p.double() ** 2).sum()
    _check(ps, ref_ps.view(1), ((chain + 1) * U32 * ref_ps).view(1), f"param_sq step {step}")


@pytest.mark.parametrize("clip", [0.0, 1e4, 0.5])
def test_scale_step_state_and_norms(ops, clip):
  """The SGD chain: p += -(lr * g * gscale + wd * p) with grad_mult != 1, checked like the Adam step."""
  g = _gen(37)
  n = 50001                                              # the scale step takes any n
  p = _randn(g, n)
  p16 = torch.empty(n, dtype=BF16, device=DEV)
  lr, wd, gm = _f32(0.05), _f32(1e-3), _f32(1.7)
  chain = _grid_chain(n, _sms() * 8, 1)
  for step in range(3):
    gr = _randn(g, n)
    gsq_t = torch.tensor([(gr.double() ** 2).sum()], dtype=torch.float32, device=DEV)
    P = p.double()
    us, ps = torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
    ops.scale_step(p, gr, p16, lr_eff=lr, wd_eff=wd, grad_mult=gm, clip_norm=clip, gnorm_sq=gsq_t,
                   upd_sq=us, param_sq=ps)
    gs = _clip_scale(float(gsq_t), gm, clip)
    upd = -(lr * gr.double() * gs + wd * P)
    p1 = P + upd
    _check(p, p1, _ulp(p1, torch.float32) + 8 * U32 * (lr * (gr.double() * gs).abs() + wd * P.abs()),
           f"params step {step}")
    _same(p16, p.to(BF16), "bf16 shadow")
    applied = p.double() - P
    ref_us = (applied * applied).sum()
    slack = (applied.abs() * _ulp(p.double(), torch.float32)).sum()
    _check(us, ref_us.view(1), ((chain + 1) * U32 * ref_us + 2 * slack).view(1), f"upd_sq step {step}")
    ref_ps = (p.double() ** 2).sum()
    _check(ps, ref_ps.view(1), ((chain + 1) * U32 * ref_ps).view(1), f"param_sq step {step}")


@pytest.mark.parametrize("xdt", [torch.float32, BF16])
@pytest.mark.parametrize("d", [40, 200, 768])
def test_l2norm(ops, xdt, d):
  """z = x / (||x|| + eps) with one warp per row (chain ceil(d/32) + 5).  norm and z within the
  summation bound propagated through sqrt and the division; the backward, from the kernel's own z and
  norm, within 1 ulp of the output dtype plus the propagated error of the dot product z.dz.  An
  all-zero row gives z = 0, norm = 0 and the finite gradient dz / eps."""
  g = _gen(d)
  n, eps = 19, _f32(1e-8)
  x = _randn(g, n, d, dtype=xdt)
  x[3] = 0
  z, nrm = ops.l2norm_fwd(x, eps=eps)
  xd = x.double()
  chain = -(-d // 32) + 5 + 1
  r = xd.norm(dim=1)
  _check(nrm, r, (chain / 2 + 2) * U32 * r, "norm")
  zref = xd / (r[:, None] + eps)
  _check(z, zref, (chain / 2 + 4) * U32 * zref.abs(), "z")
  assert float(z[3].abs().max()) == 0.0 and float(nrm[3]) == 0.0
  dz = _randn(g, n, d)
  for dxdt in (torch.float32, BF16):
    dx = ops.l2norm_bwd(dz, z, nrm, dx_dtype=dxdt, eps=eps)
    Z, R, DZ = z.double(), nrm.double()[:, None], dz.double()
    s = (DZ * Z).sum(1, keepdim=True)
    k = torch.where(R > 0, s * (R + eps) / R.clamp_min(1e-300), torch.zeros_like(R))
    ref = (DZ - Z * k) / (R + eps)
    dk = torch.where(R > 0, (R + eps) / R.clamp_min(1e-300), torch.zeros_like(R)) * chain * U32 * \
        (DZ * Z).abs().sum(1, keepdim=True)
    noise = (8 * U32 * (DZ.abs() + (Z * k).abs()) + Z.abs() * dk) / (R + eps)
    _check(dx, ref, _ulp(ref, dxdt) + noise, f"l2norm_bwd {dxdt}")
    assert torch.isfinite(dx.float()).all()


# ---------------------------------------------------------------------------------------------------
# GELU, GELU' and tanh over every bf16 input with |x| <= 16
# ---------------------------------------------------------------------------------------------------
def _bf16_sweep():
  """Every finite bf16 value with |x| <= 16 (no -0: the GEMM's accumulator cannot produce it), as fp32."""
  bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
  v = bits.view(BF16).float()
  keep = torch.isfinite(v) & (v.abs() <= 16) & ~((v == 0) & torch.signbit(v))
  return v[keep].sort().values.to(DEV)


def _gelu64(x):
  """0.5 x (1 + tanh u) written as x / (1 + exp(-2u)): no cancellation in the negative tail, where
  1 + tanh u rounds to 0 in fp64 below x = -8."""
  u = math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)
  return x / (1 + torch.exp(-2 * u))


def _dgelu64(x):
  """gelu'(x) = (1 + t) / 2 + x (1 - t) (1 + t) du / 2 with 1 +- t = 2 / (1 + exp(-+2u))."""
  k0 = math.sqrt(2 / math.pi)
  u = k0 * (x + 0.044715 * x ** 3)
  one_p, one_m = 2 / (1 + torch.exp(-2 * u)), 2 / (1 + torch.exp(2 * u))
  du = k0 * (1 + 3 * 0.044715 * x * x)
  return 0.5 * one_p + 0.5 * x * one_m * one_p * du, du


_TANH_APPROX = 2.0 ** -11        # documented max relative error of tanh.approx.f32
_SWEEP_STATS = {}


def _onehot_gemm_operands(v):
  """A [128, 64] with A[m, m % 64] = 1 and B [N, 64] holding the values: the fp32 accumulator of
  D[m, n] is exactly B[n, m % 64] = v[n * 64 + m % 64] (one product with 1, the rest with 0)."""
  N = -(-v.numel() // 64)
  N = -(-N // 8) * 8
  B = torch.zeros(N * 64, device=DEV)
  B[:v.numel()] = v
  B = B.view(N, 64).to(BF16)
  A = torch.zeros(128, 64, device=DEV)
  A[torch.arange(128), torch.arange(128) % 64] = 1
  return A.to(BF16), B, N


def _as_sweep(D, count):
  """D [128, N] -> the value at each sweep index, from the first 64 rows; rows 64..127 must repeat them."""
  assert torch.equal(D[:64].view(torch.int16), D[64:].view(torch.int16))
  return D[:64].T.reshape(-1)[:count]


def _units(got, ref, scale):
  return float(((got.double() - ref).abs() / scale).max())


def _max_rel(got, ref, x, lo=-8.0, hi=-2.0):
  sel = (x >= lo) & (x <= hi)
  return float(((got.double() - ref).abs() / ref.abs())[sel].max())


@pytest.mark.parametrize("block_n", [128, 256])
def test_gemm_gelu_epilogues_over_every_bf16_input(ops, block_n):
  """EPI_BIAS_GELU (D and D2), EPI_BIAS_GELU_ACT and EPI_DGELU over the sweep.  D2 equals x bit for
  bit.  The tanh.approx epilogues stay within 1 bf16 ulp plus the documented 2^-11 tanh error
  propagated through each formula: |x|/2 * 2^-11 for gelu, (1/2 + |x| du(x)) * 2^-11 for gelu', with
  du = sqrt(2/pi) (1 + 3 * 0.044715 x^2), plus 2^-20 relative fp32 noise."""
  from big_vision_b200 import lib as L
  x = _bf16_sweep()
  A, B, N = _onehot_gemm_operands(x)
  xd = x.double()
  act, pre = ops.gemm(A, B, bias=torch.zeros(N, device=DEV), epilogue=L.EPI_BIAS_GELU, block_n=block_n)
  _same(_as_sweep(pre, x.numel()), x.to(BF16), "D2 = x")
  act = _as_sweep(act, x.numel())
  ref = _gelu64(xd)
  prop = 0.5 * xd.abs() * _TANH_APPROX
  _check(act, ref, _ulp(ref, BF16) + prop + 2.0 ** -20 * ref.abs(), "EPI_BIAS_GELU")
  act_only = ops.gemm(A, B, bias=torch.zeros(N, device=DEV), epilogue=L.EPI_BIAS_GELU_ACT, block_n=block_n)
  _same(_as_sweep(act_only, x.numel()), act, "EPI_BIAS_GELU_ACT = D of EPI_BIAS_GELU")
  # gelu': aux is the sweep laid out as D, acc = 1 (A[:, 0] = 1, B[:, 0] = 1)
  aux = _as_sweep_layout(x, N)
  A1 = torch.zeros(128, 64, device=DEV, dtype=BF16)
  A1[:, 0] = 1
  B1 = torch.zeros(N, 64, device=DEV, dtype=BF16)
  B1[:, 0] = 1
  dg = _as_sweep(ops.gemm(A1, B1, aux=aux, epilogue=L.EPI_DGELU, block_n=block_n), x.numel())
  dref, du = _dgelu64(xd)
  dprop = (0.5 + xd.abs() * du) * _TANH_APPROX
  _check(dg, dref, _ulp(dref, BF16) + dprop + 2.0 ** -20 * dref.abs(), "EPI_DGELU")
  _SWEEP_STATS[f"epilogue_bn{block_n}"] = {
      "gelu_max_err_in_bound_units": _units(act, ref, _ulp(ref, BF16) + prop),
      "dgelu_max_err_in_bound_units": _units(dg, dref, _ulp(dref, BF16) + dprop),
      "gelu_max_err_in_bf16_ulps": _units(act, ref, _ulp(ref, BF16)),
      "dgelu_max_err_in_bf16_ulps": _units(dg, dref, _ulp(dref, BF16)),
      "gelu_max_rel_err_x_in_-8_-2": _max_rel(act, ref, xd),
      "dgelu_max_rel_err_x_in_-8_-2": _max_rel(dg, dref, xd)}


def _as_sweep_layout(v, N):
  """The sweep laid out like D of _onehot_gemm_operands: aux[m, n] = v[n * 64 + m % 64]."""
  flat = torch.zeros(N * 64, device=DEV)
  flat[:v.numel()] = v
  t = flat.view(N, 64).T
  return torch.cat([t, t], 0).contiguous().to(BF16)


def test_standalone_gelu_and_tanh_over_every_bf16_input(ops):
  """bv_gelu_fwd (exp-based tanh) and bv_tanh_fwd / bv_tanh_bwd over the sweep in fp32 and bf16.
  gelu: 1 ulp plus |x|/2 * 2^-21 (the absolute error of 1 - 2 / (1 + exp(2u)), a few fp32 ulps of 1)
  plus 2^-21 relative.  tanh: tanhf is within 2 fp32 ulps (CUDA's documented bound), so 1 bf16 ulp
  or 2 fp32 ulps.  tanh_bwd dy (1 - y^2), from the kernel's own y: 2 ulps plus the fp32 rounding of
  y^2 scaled by |dy|."""
  x = _bf16_sweep()
  xd = x.double()
  ref = _gelu64(xd)
  for dt in (torch.float32, BF16):
    got = ops.gelu_fwd(x.to(dt))
    noise = 0.5 * xd.abs() * 2.0 ** -21 + 2.0 ** -21 * ref.abs()
    _check(got, ref, _ulp(ref, dt) + noise, f"gelu_fwd {dt}")
    _SWEEP_STATS[f"gelu_fwd_{'bf16' if dt == BF16 else 'fp32'}"] = {
        "max_err_in_bound_units": _units(got, ref, _ulp(ref, dt) + noise),
        "max_rel_err_x_in_-8_-2": _max_rel(got, ref, xd)}
  tref = torch.tanh(xd)
  y32 = ops.tanh_fwd(x)
  _check(y32, tref, 2 * _ulp(tref, torch.float32), "tanh_fwd fp32")
  y16 = ops.tanh_fwd(x.to(BF16))
  _check(y16, tref, _ulp(tref, BF16) + 2.0 ** -22 * tref.abs(), "tanh_fwd bf16")
  g = _gen(41)
  for dt, y in ((torch.float32, y32), (BF16, y16)):
    dy = _randn(g, x.numel(), dtype=dt)
    dx = ops.tanh_bwd(dy, y)
    Y, DY = y.double(), dy.double()
    ref = DY * (1 - Y * Y)
    _check(dx, ref, 2 * _ulp(ref, dt) + 2 * U32 * DY.abs() * Y * Y, f"tanh_bwd {dt}")


def test_print_gelu_sweep_summary():
  """One JSON line with the measured errors of the sweeps above (run after them, in file order)."""
  if _SWEEP_STATS:
    print("GELU_SWEEP " + json.dumps(_SWEEP_STATS, sort_keys=True))


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("mod", [49, 256, 576, 729])
def test_resid_epilogue_position_embedding_periods(ops, mod, block_n):
  """EPI_BIAS_RESID with aux_row_mod at the position-embedding periods of B/32, /14 at 224, L/14 at
  336 and So400m at 384: D[m] = bf16(x w + bias) + aux[m % mod], bit for bit against the fp32-output
  GEMM of the same accumulators.  At 49 a 128-row tile wraps the period more than twice."""
  from big_vision_b200 import lib as L
  g = _gen(mod)
  M, N, K = 3 * mod + 77, 768, 256
  x, w = _randn(g, M, K, dtype=BF16), _randn(g, K, N, scale=0.05, dtype=BF16)
  bias, aux = _randn(g, N), _randn(g, mod, N, dtype=BF16)
  f = ops.gemm(x, w, b_mn=True, bias=bias, out_dtype=torch.float32, block_n=block_n)
  ref = (f.to(BF16).float() + aux.float()[torch.arange(M, device=DEV) % mod]).to(BF16)
  got = ops.gemm(x, w, b_mn=True, bias=bias, aux=aux, aux_row_mod=mod, epilogue=L.EPI_BIAS_RESID,
                 block_n=block_n)
  _same(got, ref, f"resid mod {mod}")


# ---------------------------------------------------------------------------------------------------
# losses at the operating point
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,B,off", [(768, 6144, 768 * 3), (768, 768, -768), (100, 1036, 37)])
@pytest.mark.parametrize("tp,bp", [(math.log(10.0), -10.0), (math.log(117.0), -16.0), (math.log(117.0), 0.0),
                                   (math.log(10.0), None)])
def test_siglip_loss_elementwise(ops, n, B, off, tp, bp):
  """The [768, 6144] slab of an 8-GPU siglip_b16 step, an all-negative chunked round (row_offset = -n)
  and a ragged slab, with correlated positives so that x = dot * t + b spans about -130 .. +30.
  Each G element within 1 bf16 ulp plus an fp32 term 2^-20 (1 + |x|) relative (the rounding of x and
  of exp(t') propagated through the sigmoid); the loss, dt and db within the summation bound
  (per-thread strips, two 5-level trees, a fixed-order pass over <= 1056 block partials)."""
  g = _gen(n + B + int(tp))
  zt = torch.nn.functional.normalize(_randn(g, B, 64).double(), dim=1)
  rows = torch.arange(n, device=DEV)
  partner = (rows + off) % B if off >= 0 else rows % B
  zi = torch.nn.functional.normalize(zt[partner] * 3 + _randn(g, n, 64).double(), dim=1)
  if off < 0:
    zi = torch.nn.functional.normalize(_randn(g, n, 64).double(), dim=1)
  dots = (zi @ zt.T).float()
  dots[:, 0] = -1.0
  dots[:, 1] = 1.0
  t_param = torch.tensor([tp], device=DEV)
  b_param = torch.tensor([bp], device=DEV) if bp is not None else None
  loss, dt, db = (torch.zeros(1, device=DEV) for _ in range(3))
  G = ops.siglip_loss(dots, off, t_param, b_param, B, loss, dt, db)
  t = math.exp(float(t_param))
  b = float(b_param) if bp is not None else 0.0
  D = dots.double()
  x = D * t + b
  sgn = -torch.ones_like(x)
  cols = rows + off
  valid = (cols >= 0) & (cols < B)
  sgn[rows[valid], cols[valid]] = 1.0
  gx = -sgn * torch.sigmoid(-sgn * x) / B
  Gref = gx * t
  _check(G, Gref, _ulp(Gref, BF16) + 2.0 ** -20 * (1 + x.abs()) * Gref.abs(), "G")
  terms = -torch.nn.functional.logsigmoid(sgn * x) / B
  blocks = min((n * (B // 4) + 255) // 256, _sms() * 8)
  per_thread = -(-(n * (B // 4)) // (blocks * 256)) * 4
  chain = per_thread + 10 + blocks + 8 + 2
  _check(loss, terms.sum().view(1), (chain * U32 * terms.abs().sum() + 2.0 ** -20 * terms.abs().sum()).view(1),
         "loss")
  # each term's own fp32 error (x rounded, exp(t') approximated) is ~2^-20 (1 + |x|) of it
  tt = gx * D * t
  _check(dt, tt.sum().view(1), ((chain * U32 + 2.0 ** -20) * ((1 + x.abs()) * tt.abs()).sum()).view(1), "dt")
  _check(db, gx.sum().view(1), ((chain * U32 + 2.0 ** -20) * ((1 + x.abs()) * gx.abs()).sum()).view(1), "db")


def test_softmax_contrastive_at_batch_6144(ops):
  """B = 6144 with t = 100: peaky rows (x spans hundreds), some rows whose argmax ties exactly with
  another column (the first index wins), G within 1 bf16 ulp plus fp32 terms, loss and dt within the
  summation bound, the argmax count exact."""
  g = _gen(61)
  n, B, off = 256, 6144, 1024
  dots = _randn(g, n, B, scale=0.1)
  rows = torch.arange(n, device=DEV)
  dots[rows, off + rows] += 0.3 * (rows % 2 == 0)                      # half the rows retrieve correctly
  dots[rows[::4], 5] = dots[rows[::4], off + rows[::4]]                 # exact ties: column 5 is earlier
  dots[rows[1::4], B - 1] = dots[rows[1::4], off + rows[1::4]]          # a tie after the positive
  dots = dots.contiguous()
  tp = torch.tensor([math.log(100.0)], device=DEV)
  sc = torch.zeros(3, device=DEV)
  G = ops.softmax_contrastive_loss(dots, off, tp, B, 0.5, sc[0:1], sc[1:2], sc[2:3])
  t = math.exp(float(tp))
  x = dots.double() * t
  lse = torch.logsumexp(x, 1, keepdim=True)
  p = torch.exp(x - lse)
  onehot = torch.zeros_like(x)
  onehot[rows, off + rows] = 1
  w = 0.5 / B
  gref = (p - onehot) * w * t
  mx = x.max(1, keepdim=True).values
  chain = -(-B // 32) + 5 + -(-n // 256) + 8 + 2
  # relative error of p = exp(x - lse): the sum under lse (chain * 2^-24), and the rounding of
  # x = dot * exp(t') and of mx + log(sum), ~2^-22 (1 + |x| + |mx|) in the exponent
  dp = chain * U32 + 2.0 ** -20 * (1 + x.abs() + mx.abs())
  _check(G, gref, _ulp(gref, BF16) + w * t * (dp * p + U32 * onehot), "G")
  li = (lse[:, 0] - x[rows, off + rows]) * w
  err_row = (chain * U32 + 2.0 ** -20 * (1 + mx.abs()[:, 0])) * w       # lse of each row: mx + log(sum)
  _check(sc[0:1], li.sum().view(1), (chain * U32 * li.abs().sum() + err_row.sum()).view(1), "loss")
  dtt = ((p - onehot) * w * x).sum(1)
  dt_bound = (chain * U32 + 2.0 ** -20) * ((p + onehot) * w * x.abs() * (1 + x.abs() + mx.abs())).sum()
  _check(sc[1:2], dtt.sum().view(1), dt_bound.view(1), "dt")
  first = x.argmax(1)                                               # torch: first maximal index
  assert int(sc[2]) == int((first == off + rows).sum())
  assert int((x[rows[::4], 5] == x[rows[::4], off + rows[::4]]).sum()) == len(rows[::4])


@pytest.mark.parametrize("C", [1000, 21843])
def test_classification_losses_wide_logits(ops, C):
  """sigmoid_xent / softmax_xent with |logits| up to 60 (the min(y, 0) branch of log_sigmoid and
  exp underflow) and C = 21843 (ImageNet-21k).  dlogits within 1 fp32 ulp plus 2^-20 (1 + |x|) of
  its exponential part; the loss within the summation bound of its terms (per-lane strips of
  ceil(C / 32), a 5-level tree, the fixed-order pass over the rows)."""
  g = _gen(C)
  n = 24
  lg = _randn(g, n, C, scale=20.0).clamp(-60, 60)
  lg[:, :4] = torch.tensor([60.0, -60.0, 59.5, -59.5], device=DEV)
  lab = torch.zeros(n, C, device=DEV)
  lab[torch.arange(n), torch.randint(0, C, (n,), generator=g, device=DEV)] = 0.9
  lab[:, 1] += 0.1
  X, Y = lg.double(), lab.double()
  chain = -(-C // 32) + 5 + -(-n // 256) + 8 + 2
  # sigmoid
  loss = torch.zeros(1, device=DEV)
  dl = ops.sigmoid_xent(lg, lab, loss)
  s = torch.sigmoid(X)
  ref = (s - Y) / n
  _check(dl, ref, _ulp(ref, torch.float32) + 2 * U32 * ref.abs() + (2.0 ** -20 * (1 + X.abs()) * s + 2 * U32 * Y) / n,
         "sigmoid dlogits")
  terms = -(Y * torch.nn.functional.logsigmoid(X) + (1 - Y) * torch.nn.functional.logsigmoid(-X)) / n
  tb = ((chain * U32 + 2.0 ** -20 * (1 + X.abs())) * terms.abs()).sum()
  _check(loss, terms.sum().view(1), tb.view(1), "sigmoid loss")
  # softmax
  loss = torch.zeros(1, device=DEV)
  dl = ops.softmax_xent(lg, lab, loss)
  lse = torch.logsumexp(X, 1, keepdim=True)
  p = torch.exp(X - lse)
  sy = Y.sum(1, keepdim=True)
  ref = (p * sy - Y) / n
  mx = X.max(1, keepdim=True).values
  dp = chain * U32 + 2.0 ** -20 * (1 + X.abs() + mx.abs())
  _check(dl, ref, _ulp(ref, torch.float32) + 2 * U32 * ref.abs() + (dp * p * sy + 2 * U32 * Y) / n,
         "softmax dlogits")
  li = (lse[:, 0] * sy[:, 0] - (Y * X).sum(1)) / n
  # the kernel sums the shifted values: log sum exp(x - mx) and sum y (x - mx)
  tb = (chain * U32 + 2.0 ** -20) * (((lse.abs() + 2 * mx.abs() + 1) * sy)[:, 0] + (Y * X).abs().sum(1)) / n
  _check(loss, li.sum().view(1), tb.sum().view(1), "softmax loss")
