"""GPU parity tests, kernel by kernel, through the C ABI, against the CPU oracle
(oracle/bv_oracle.py) on the same seeded inputs.  Tolerances: bf16 outputs 2^-8 relative to
the tensor scale (one bf16 rounding of O(1) data after an fp32-accumulated contraction);
fp32 reductions 1e-5."""
import math

import numpy as np
import pytest
import torch

from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu
F64 = torch.float64


def _close(got, ref, tol):
  got = got.detach().double().cpu()
  ref = ref.detach().double().cpu()
  scale = ref.abs().max().item() + 1e-12
  err = (got - ref).abs().max().item() / scale
  assert not torch.isnan(got).any()
  assert err <= tol, f"rel err {err:.3e} > {tol}"


@pytest.fixture(scope="module")
def ops():
  from big_vision_b200 import lib, ops as _ops
  assert lib.load().bv_device_supported() == 1, "needs a compute-capability 9.x GPU"
  return _ops


def _bf(x):
  return x.to(torch.bfloat16)


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (200, 768, 320), (1030, 2304, 768), (64, 1000, 776)])
def test_dense_forward_epilogues(ops, M, N, K):
  from big_vision_b200 import lib as L
  g = torch.Generator().manual_seed(M + N + K)
  x = _bf(torch.randn(M, K, generator=g) * 0.5)
  w = _bf(torch.randn(K, N, generator=g) * 0.5)
  b = torch.randn(N, generator=g)
  r = _bf(torch.randn(M, N, generator=g))
  ref = O.dense(x.double(), w.double(), b.double(), "bfloat16")
  out = ops.gemm(x.cuda(), w.cuda(), b_mn=True, bias=b.cuda())
  _close(out, ref, 2 ** -7)
  out = ops.gemm(x.cuda(), w.cuda(), b_mn=True, bias=b.cuda(), aux=r.cuda(), epilogue=L.EPI_BIAS_RESID)
  _close(out, O.rnd(O.rnd(ref, "bfloat16") + r.double(), "bfloat16"), 2 ** -7)
  act, pre = ops.gemm(x.cuda(), w.cuda(), b_mn=True, bias=b.cuda(), epilogue=L.EPI_BIAS_GELU)
  _close(pre, ref, 2 ** -7)
  _close(act, O.gelu_tanh(pre.double().cpu()), 2 ** -7)
  out32 = ops.gemm(x.cuda(), w.cuda(), b_mn=True, bias=b.cuda(), out_dtype=torch.float32)
  _close(out32, ref, 1e-4)


@pytest.mark.parametrize("M,N,K", [(256, 128, 256), (777, 768, 3072), (1000, 3072, 768)])
def test_dense_backward_contractions(ops, M, N, K):
  """dgrad (K,K) with gelu' epilogue and split-K wgrad (MN,MN) with fp32 reduce-add."""
  from big_vision_b200 import lib as L
  g = torch.Generator().manual_seed(7)
  x = _bf(torch.randn(M, K, generator=g) * 0.5)        # activations
  w = _bf(torch.randn(K, N, generator=g) * 0.1)        # kernel [K, N]
  dy = _bf(torch.randn(M, N, generator=g) * 0.5)
  pre = _bf(torch.randn(M, K, generator=g))
  dx_ref = dy.double() @ w.double().T
  dx = ops.gemm(dy.cuda(), w.cuda())                   # B = W as stored [K, N] = [N'=K rows, K'=N]
  _close(dx, dx_ref, 2 ** -7)
  pr = pre.double().requires_grad_(True)
  O.gelu_tanh(pr).sum().backward()
  db = torch.full((K,), 0.5, device="cuda")             # fused bias gradient: += column sums of dxg
  dxg = ops.gemm(dy.cuda(), w.cuda(), aux=pre.cuda(), epilogue=L.EPI_DGELU, colsum=db)
  _close(dxg, dx_ref * pr.grad, 2 ** -7)
  _close(db, 0.5 + dxg.double().sum(0), 1e-5)           # exactly the stored (bf16) values, fp32 sums
  dw = torch.zeros(K, N, device="cuda")
  ops.gemm(x.cuda(), dy.cuda(), a_mn=True, b_mn=True, out=dw, reduce_out=True)
  dw_ref = x.double().T @ dy.double()
  _close(dw, dw_ref, 1e-4)
  ops.gemm(x.cuda(), dy.cuda(), a_mn=True, b_mn=True, out=dw, reduce_out=True, splits=2)
  _close(dw, 2 * dw_ref, 1e-4)                          # accumulation semantics


def test_gemm_is_linear_at_full_size(ops):
  """Size-independent property at the benchmark's shapes: (A1 + A2) B == A1 B + A2 B."""
  M, N, K = 1024 * 196, 768, 768
  g = torch.Generator(device="cuda").manual_seed(0)
  a1 = torch.randint(-4, 5, (M, K), generator=g, device="cuda").to(torch.bfloat16)
  a2 = torch.randint(-4, 5, (M, K), generator=g, device="cuda").to(torch.bfloat16)
  w = torch.randint(-2, 3, (K, N), generator=g, device="cuda").to(torch.bfloat16)
  s = ops.gemm(a1 + a2, w, b_mn=True, out_dtype=torch.float32)    # small integers: exact in bf16/fp32
  s1 = ops.gemm(a1, w, b_mn=True, out_dtype=torch.float32)
  s2 = ops.gemm(a2, w, b_mn=True, out_dtype=torch.float32)
  assert torch.equal(s, s1 + s2)
  rows = torch.randint(0, M, (64,), device="cuda")
  assert torch.equal(s1[rows], a1[rows].float() @ w.float())


U32 = 2.0 ** -24


def _ulp(ref, dtype):
  """Spacing of `dtype` at |ref| (fp64), floored at the spacing of the smallest normal number."""
  e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126)))
  return torch.exp2(e - (7 if dtype == torch.bfloat16 else 23))


def _check(got, ref, bound, what):
  """Element-wise |got - ref| <= bound (the bound of each element, not a fraction of the tensor max)."""
  got, ref = got.detach().double(), ref.detach().double().to(got.device)
  bound = torch.as_tensor(bound, dtype=F64, device=got.device).expand_as(ref)
  assert not torch.isnan(got).any(), what
  err = (got - ref).abs()
  ok = err <= bound
  if not bool(ok.all()):
    i = tuple((~ok).nonzero()[0].tolist())
    raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements out of bound; first at {i}: "
                         f"got {got[i].item()!r} ref {ref[i].item()!r} bound {bound[i].item():.3e}")


# widths of every model (Ti 192, mu 32, So400m 1152, H 1280, g 1408, g-opt / G-opt 1536, G 1664, e 1792,
# the 2048 limit; 264 and 1032 leave one chunk in the last register slot) on both sides of the 4096 rows
# where the bf16 streaming kernels take over (nch = d / 256 <= 4; the generic kernels at every nch)
_LN_CASES = ([(1000, 768), (77, 384), (513, 1024), (9, 64), (5000, 768), (4099, 320), (4500, 1024)] +
             [(r, d) for d in (32, 192, 264, 1032, 1152, 1280, 1408, 1536, 1664, 1792, 2048) for r in (777, 4100)])


@pytest.mark.parametrize("rows,d", _LN_CASES)
def test_layernorm(ops, rows, d):
  """Forward and backward for x, y, dy, dx in bf16 and fp32, with and without dres, and each of dscale,
  dbias, dx_colsum absent in one case; rows offset from zero by up to 16 standard deviations (a
  residual stream) and scales away from 1.  Element-wise bounds against fp64:
    * mean and rstd: the summation bound of the fast variance E[x^2] - E[x]^2, chain 8 nch + 6 per lane;
    * y and dx: 1 ulp of the output dtype at the fp64 value computed from the kernel's own mean and
      rstd, plus the fp32 roundings of the formula propagated per element (and, for y, 2^-21 of the
      row's output scale);
    * dscale, dbias, dx_colsum (accumulated into non-zero initial values): the summation bound over
      the per-warp strips, the shared-memory and global atomics."""
  g = torch.Generator(device="cuda").manual_seed(rows * 7 + d)
  dev = "cuda"
  sig = torch.rand(rows, 1, generator=g, device=dev) * 1.5 + 0.5
  off = (torch.rand(rows, 1, generator=g, device=dev) * 32 - 16) * sig
  x32 = torch.randn(rows, d, generator=g, device=dev) * sig + off
  sc = torch.randn(d, generator=g, device=dev) * 0.5 + 1.5
  bi = torch.randn(d, generator=g, device=dev) * 0.3
  nch = -(-(d // 8) // 32)
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  S, Bi = sc.double(), bi.double()
  stats = {}
  for xdt in (torch.bfloat16, torch.float32):
    x = x32.to(xdt)
    X = x.double()
    c = 8 * nch + 6
    m_ref = X.mean(1)
    e2 = (X * X).mean(1)
    dmean = c * U32 * X.abs().mean(1) + 2 * U32 * m_ref.abs()
    dvar = (c + 1) * U32 * e2 + 2 * U32 * e2 + 2 * m_ref.abs() * dmean + 3 * U32 * m_ref * m_ref
    var = torch.clamp(e2 - m_ref * m_ref, min=0)
    for ydt in (torch.bfloat16, torch.float32):
      y, mean, rstd = ops.layernorm_fwd(x, sc, bi, out_dtype=ydt)
      _check(mean, m_ref, dmean, f"mean x {xdt}")
      r_ref = torch.rsqrt(var + 1e-6)
      _check(rstd, r_ref, r_ref * (0.5 * dvar / (var + 1e-6) + 6 * U32), f"rstd x {xdt}")
      M, R = mean.double()[:, None], rstd.double()[:, None]
      xh = (X - M) * R
      yref = xh * S + Bi
      # the fp32 roundings of each element's formula, and 2^-21 of the row's output scale
      noise = U32 * (4 * (xh * S).abs() + yref.abs() + Bi.abs()) + 2.0 ** -21 * yref.abs().amax(1, keepdim=True)
      _check(y, yref, _ulp(yref, ydt) + noise, f"y x {xdt} y {ydt}")
    stats[xdt] = (x, mean, rstd)

  # longest accumulation chain of dscale / dbias / dx_colsum: a warp's rows (at least min(rows, 8 * sms)
  # warps share them), one shared atomic per warp (<= 12), one global atomic per block (<= 2 * sms), init
  chain = -(-rows // min(rows, 8 * sms)) + 12 + 2 * sms + 2
  bf = torch.bfloat16
  cases = [(bf, bf, bf, True, ("dscale", "dbias", "dx_colsum")),
           (bf, bf, bf, False, ("dbias", "dx_colsum")),
           (bf, torch.float32, torch.float32, True, ("dscale", "dx_colsum")),
           (torch.float32, bf, torch.float32, False, ("dscale", "dbias"))]
  for dydt, xdt, dxdt, has_res, sums in cases:
    what = f"dy {dydt} x {xdt} dx {dxdt} dres {has_res}"
    x, mean, rstd = stats[xdt]
    dy = torch.randn(rows, d, generator=g, device=dev).to(dydt)
    dres = torch.randn(rows, d, generator=g, device=dev).to(dxdt) if has_res else None
    init = {k: torch.randn(d, generator=g, device=dev) for k in sums}
    acc = {k: v.clone() for k, v in init.items()}
    dx = ops.layernorm_bwd(dy, x, sc, mean, rstd, dres=dres, dx_dtype=dxdt, dscale=acc.get("dscale"),
                           dbias=acc.get("dbias"), dx_colsum=acc.get("dx_colsum"))
    X, DY = x.double(), dy.double()
    M, R = mean.double()[:, None], rstd.double()[:, None]
    xh = (X - M) * R
    dxh = U32 * (2 * (X.abs() + M.abs()) * R + xh.abs())        # fp32 x * rstd - mean * rstd
    gy = DY * S
    c1, c2 = gy.mean(1, keepdim=True), (gy * xh).mean(1, keepdim=True)
    cl = 8 * nch + 6
    dc1 = cl * U32 * gy.abs().mean(1, keepdim=True)
    dc2 = cl * U32 * (gy * xh).abs().mean(1, keepdim=True) + (gy.abs() * dxh).mean(1, keepdim=True)
    core = R * (gy - c1 - xh * c2)
    ref = core + (dres.double() if has_res else 0)
    noise = R * (4 * U32 * (gy.abs() + c1.abs() + (xh * c2).abs()) + dc1 + xh.abs() * dc2 + dxh * c2.abs()) + \
        2 * U32 * ref.abs()
    bound = _ulp(ref, dxdt) + noise
    _check(dx, ref, bound, f"dx {what}")
    if "dscale" in sums:
      t = DY * xh
      _check(acc["dscale"], init["dscale"].double() + t.sum(0),
             chain * U32 * (init["dscale"].double().abs() + t.abs().sum(0)) + (DY.abs() * dxh).sum(0),
             f"dscale {what}")
    if "dbias" in sums:
      _check(acc["dbias"], init["dbias"].double() + DY.sum(0),
             chain * U32 * (init["dbias"].double().abs() + DY.abs().sum(0)), f"dbias {what}")
    if "dx_colsum" in sums:
      # the generic kernel sums the stored dx, the bf16 streaming one the fp32 values before rounding:
      # either is within `bound` of ref per element
      _check(acc["dx_colsum"], init["dx_colsum"].double() + ref.sum(0),
             chain * U32 * (init["dx_colsum"].double().abs() + ref.abs().sum(0)) + bound.sum(0),
             f"dx_colsum {what}")


def test_layernorm_constant_rows_hit_the_variance_clamp(ops):
  x = torch.full((4, 64), 3.0, dtype=torch.bfloat16)
  y, _, _ = ops.layernorm_fwd(x.cuda(), torch.ones(64).cuda(), torch.zeros(64).cuda(), out_dtype=torch.float32)
  assert torch.equal(y.cpu(), torch.zeros(4, 64))


def _ref_attention(q, k, v, heads):
  B, Nq, d = q.shape
  Nk = k.shape[1]
  dh = d // heads
  qh = q.reshape(B, Nq, heads, dh).transpose(1, 2)
  kh = k.reshape(B, Nk, heads, dh).transpose(1, 2)
  vh = v.reshape(B, Nk, heads, dh).transpose(1, 2)
  s = qh @ kh.transpose(-1, -2) / math.sqrt(dh)
  return (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, Nq, d), torch.logsumexp(s, -1)


@pytest.mark.parametrize("B,H,Nq,Nk", [(3, 2, 64, 64), (2, 12, 196, 196), (5, 3, 197, 197), (4, 2, 1, 196),
                                       (2, 1, 16, 16), (1, 2, 256, 256), (2, 2, 130, 7),
                                       (4, 3, 64, 64), (6, 12, 64, 64)])   # the text tower's 64 tokens
def test_attention_forward_backward(ops, B, H, Nq, Nk):
  g = torch.Generator().manual_seed(B * 1000 + Nq)
  d = H * 64
  qkv = _bf(torch.randn(B, max(Nq, Nk), 3 * d, generator=g))
  do = _bf(torch.randn(B, Nq, d, generator=g))
  qr = qkv[:, :Nq, 0:d].double().requires_grad_(True)
  kr = qkv[:, :Nk, d:2 * d].double().requires_grad_(True)
  vr = qkv[:, :Nk, 2 * d:].double().requires_grad_(True)
  o_ref, lse_ref = _ref_attention(qr, kr, vr, H)
  o_ref.backward(do.double())
  c = qkv.cuda()
  q, k, v = c[:, :Nq, 0:d], c[:, :Nk, d:2 * d], c[:, :Nk, 2 * d:]     # strided views, as in the model
  o, lse = ops.attention_fwd(q, k, v, H)
  _close(o, o_ref, 2 ** -6)
  _close(lse, lse_ref, 1e-5)
  dq, dk, dv = ops.attention_bwd(do.cuda(), q, k, v, o, lse, H)
  _close(dq, qr.grad, 2 ** -5)
  _close(dk, kr.grad, 2 ** -5)
  _close(dv, vr.grad, 2 ** -5)
  # fused bias gradients of the q/k/v projections: column sums over the valid rows, accumulated
  cs = torch.ones(3, d, device="cuda")
  dq2, dk2, dv2 = ops.attention_bwd(do.cuda(), q, k, v, o, lse, H, dq_colsum=cs[0], dk_colsum=cs[1],
                                    dv_colsum=cs[2])
  assert torch.equal(dq2, dq) and torch.equal(dk2, dk) and torch.equal(dv2, dv)
  for i, t in enumerate((dq, dk, dv)):
    ref = 1 + t.double().sum((0, 1))
    assert (cs[i].double() - ref).abs().max().item() <= 1e-4 * (ref.abs().max().item() + 1)


def test_text_tower_attention_is_bitwise_reproducible(ops):
  """The text tower's shape (64 tokens, 12 heads) run twice, forward and backward with the fused bias
  gradients: outputs, log-sum-exps and gradients are identical bit for bit; the bias gradients, which are
  accumulated with fp32 atomics, agree to rounding."""
  g = torch.Generator().manual_seed(11)
  B, H, N = 8, 12, 64
  d = H * 64
  c = _bf(torch.randn(B, N, 3 * d, generator=g)).cuda()
  do = _bf(torch.randn(B, N, d, generator=g)).cuda()
  q, k, v = c[:, :, 0:d], c[:, :, d:2 * d], c[:, :, 2 * d:]
  runs = []
  for _ in range(2):
    o, lse = ops.attention_fwd(q, k, v, H)
    cs = torch.zeros(3, d, device="cuda")
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, H, dq_colsum=cs[0], dk_colsum=cs[1], dv_colsum=cs[2])
    runs.append((o, lse, dq, dk, dv, cs))
  for a, b in zip(runs[0][:5], runs[1][:5]):
    assert torch.equal(a, b)
  _close(runs[1][5], runs[0][5], 1e-6)


def test_attention_rows_are_convex_combinations(ops):
  """Property at benchmark size: with v == const per column every output row equals that const."""
  B, H, N = 64, 12, 196
  d = H * 64
  g = torch.Generator(device="cuda").manual_seed(1)
  q = torch.randn(B, N, d, generator=g, device="cuda").to(torch.bfloat16)
  k = torch.randn(B, N, d, generator=g, device="cuda").to(torch.bfloat16)
  col = torch.randn(1, 1, d, generator=g, device="cuda").to(torch.bfloat16)
  v = col.expand(B, N, d).contiguous()
  o, _ = ops.attention_fwd(q, k, v, H)
  assert (o.float() - col.float()).abs().max().item() <= 2 ** -7 * col.float().abs().max().item()


def test_patchify_embed_pool_l2norm(ops):
  g = torch.Generator().manual_seed(5)
  img = torch.rand(3, 32, 48, 3, generator=g) * 2 - 1
  pt = ops.patchify(img.cuda(), 16)
  ref = img.reshape(3, 2, 16, 3, 16, 3).permute(0, 1, 3, 2, 4, 5).reshape(-1, 768)
  assert torch.equal(pt.cpu(), ref.to(torch.bfloat16))               # pure data movement + rounding
  ids = torch.randint(0, 50, (5, 7), generator=g, dtype=torch.int32)
  ids[:, -1] = 1
  table, pos = torch.randn(50, 64, generator=g), torch.randn(7, 64, generator=g)
  e = ops.embed_fwd(ids.cuda(), table.cuda(), pos.cuda(), out_dtype=torch.float32)
  assert torch.equal(e.cpu(), (table[ids.long()] + pos[None]).reshape(-1, 64))
  dy = torch.randn(35, 64, generator=g)
  dt, dp = torch.zeros(50, 64, device="cuda"), torch.zeros(7, 64, device="cuda")
  ops.embed_bwd(ids.cuda(), dy.cuda(), dt, dp)
  _close(dt, torch.zeros(50, 64).index_add_(0, ids.flatten().long(), dy), 1e-6)   # duplicate ids (pad)
  _close(dp, dy.reshape(5, 7, 64).sum(0), 1e-6)
  x = torch.randn(33, 768, generator=g)
  z, nrm = ops.l2norm_fwd(x.cuda())
  xr = x.double().requires_grad_(True)
  zr = O.l2_normalize(xr)
  _close(z, zr, 1e-6)
  dz = torch.randn(33, 768, generator=g)
  zr.backward(dz.double())
  _close(ops.l2norm_bwd(dz.cuda(), z, nrm), xr.grad, 1e-5)
  xs = torch.randn(40, 64, generator=g)
  assert torch.allclose(ops.pool_fwd(xs.cuda(), 4, 10, 0).cpu(), xs.reshape(4, 10, 64).mean(1), atol=1e-6)
  assert torch.equal(ops.pool_fwd(xs.cuda(), 4, 10, 1, tok=9).cpu(), xs.reshape(4, 10, 64)[:, 9])
  # max pool (text_transformer.py:89-90): bf16 input with many ties at the maximum -- the cotangent is
  # split evenly between them, the rule jnp.max (and torch.amax) differentiates with
  xm = (torch.randn(6, 9, 64, generator=g) * 2).round().bfloat16()
  assert torch.equal(ops.pool_fwd(xm.view(54, 64).cuda(), 6, 9, 2).cpu(), xm.amax(1))
  xr = xm.double().requires_grad_(True)
  dym = torch.randn(6, 64, generator=g)
  torch.amax(xr, dim=1).backward(dym.double())
  assert int((xr.grad != 0).sum()) > 6 * 64          # the case does have ties
  _close(ops.pool_max_bwd(dym.cuda(), xm.view(54, 64).cuda(), 6, 9, dx_dtype=torch.float32).view(6, 9, 64),
         xr.grad, 1e-6)


@pytest.mark.parametrize("vr,inr,clip", [((-1.0, 1.0), (0.0, 255.0), False), ((-0.5, 0.5), (-256.0, 255.0), True),
                                         ((0.0, 1.0), (0.0, 255.0), False)])
def test_patchify_u8_fuses_value_range_bit_exactly(ops, vr, inr, clip):
  """uint8 ingest: value_range (pp/ops_general.py:32-64; the cases of ops_general_test.py:36-49) in
  fp32 with every operation rounded separately, then the same patch layout as the fp32 path."""
  import numpy as np
  rng = np.random.default_rng(3)
  u8 = rng.integers(0, 256, size=(3, 32, 48, 3), dtype=np.uint8)
  f32 = np.float32
  x = (u8.astype(f32) - f32(inr[0])) / (f32(inr[1]) - f32(inr[0]))
  ref = f32(vr[0]) + x * f32(vr[1] - vr[0])
  if clip:
    ref = np.clip(ref, f32(vr[0]), f32(vr[1]))
  assert ref.dtype == np.float32 and ref.min() >= vr[0] and ref.max() <= vr[1]
  want = ops.patchify(torch.from_numpy(ref).cuda(), 16)
  got = ops.patchify(torch.from_numpy(u8).cuda(), 16, value_range=vr, in_range=inr, clip_values=clip)
  assert torch.equal(got.view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize("n,B,off", [(8, 8, 0), (64, 256, 128), (16, 64, 48)])
def test_siglip_loss_slab(ops, n, B, off):
  """One rank's [n, B] slab of the global loss (positives at column off + i)."""
  g = torch.Generator().manual_seed(n)
  zi = O.l2_normalize(torch.randn(B, 32, generator=g).double())
  zt = O.l2_normalize(torch.randn(B, 32, generator=g).double())
  dots = (zi[off:off + n] @ zt.T).float()
  tp, bp = torch.tensor([math.log(10.0)]), torch.tensor([-10.0])
  dr = dots.double().requires_grad_(True)
  tr, br = tp.double().requires_grad_(True), bp.double().requires_grad_(True)
  x = dr * tr.exp() + br
  m = -torch.ones(n, B, dtype=F64)
  m[torch.arange(n), off + torch.arange(n)] = 1
  l = -(torch.nn.functional.logsigmoid(m * x)).sum() / B
  l.backward()
  loss, dt, db = (torch.zeros(1, device="cuda") for _ in range(3))
  G = ops.siglip_loss(dots.cuda(), off, tp.cuda(), bp.cuda(), B, loss, dt, db)
  _close(loss, l.reshape(1), 1e-5)
  _close(G, dr.grad, 2 ** -7)
  _close(dt, tr.grad, 1e-4)
  _close(db, br.grad, 1e-4)


def test_narrow_loss_slab_feeds_the_gradient_gemms(ops):
  """The chunked loss on a tiny per-rank batch produces [4, 4] slabs (2 ranks x 4 pairs,
  tests/test_dist_gpu.py): the bf16 gradient slab must still be a legal TMA operand (row stride a
  multiple of 16 bytes) for G . z and G^T . z."""
  g = torch.Generator().manual_seed(0)
  n = 4
  zi = _bf(torch.randn(n, 64, generator=g) * 0.1)
  zt = _bf(torch.randn(n, 64, generator=g) * 0.1)
  dots = ops.gemm(zi.cuda(), zt.cuda(), out_dtype=torch.float32)
  sc = torch.zeros(3, device="cuda")
  t, b = torch.tensor([math.log(10.0)]).cuda(), torch.tensor([-10.0]).cuda()
  G = ops.siglip_loss(dots, 0, t, b, 8, sc[0:1], sc[1:2], sc[2:3])
  assert G.shape == (n, n) and (G.stride(0) * 2) % 16 == 0
  dzi = ops.gemm(G, zt.cuda(), b_mn=True, out_dtype=torch.float32)
  dzt = ops.gemm(G, zi.cuda(), a_mn=True, b_mn=True, out_dtype=torch.float32)
  _close(dzi, G.double().cpu() @ zt.double(), 1e-4)
  _close(dzt, G.double().cpu().T @ zi.double(), 1e-4)
  G2 = ops.softmax_contrastive_loss(dots, 0, t, 8, 0.5, sc[0:1], sc[1:2], sc[2:3])
  _close(ops.gemm(G2, zt.cuda(), b_mn=True, out_dtype=torch.float32), G2.double().cpu() @ zt.double(), 1e-4)


@pytest.mark.parametrize("n,B,off", [(8, 8, 0), (64, 256, 128), (33, 100, 7)])
def test_softmax_contrastive_slab(ops, n, B, off):
  """One direction of the CLIP softmax loss (_deprecated_contrastive.py:80-101) on a rank's [n, B]
  slab: loss, d loss / d dots, d loss / d t', and the argmax == positive count (integer, exact)."""
  g = torch.Generator().manual_seed(n + B)
  dots = torch.randn(n, B, generator=g) * 0.3
  dots[torch.arange(n), off + torch.arange(n)] += 0.4 * (torch.arange(n) % 3 == 0)   # some correct retrievals
  tp = torch.tensor([math.log(10.0)])
  dr, tr = dots.double().requires_grad_(True), tp.double().requires_grad_(True)
  x = dr * tr.exp()
  idx = torch.arange(n)
  ref = 0.5 * (torch.logsumexp(x, 1) - x[idx, off + idx]).sum() / B
  ref.backward()
  sc = torch.zeros(3, device="cuda")
  dt = torch.zeros(1, device="cuda")
  G = ops.softmax_contrastive_loss(dots.cuda(), off, tp.cuda(), B, 0.5, sc[0:1], dt, sc[1:2])
  _close(sc[0:1], ref.detach().reshape(1), 1e-5)
  _close(G, dr.grad, 2 ** -7)
  _close(dt, tr.grad.reshape(1), 1e-4)
  assert int(sc[1]) == int((x.argmax(1) == off + idx).sum())


def test_classification_losses(ops):
  g = torch.Generator().manual_seed(11)
  lg = torch.randn(37, 1000, generator=g) * 3
  lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (37,), generator=g), 1000).float()
  lab = 0.9 * lab + 0.1 * lab.roll(1, 0)                  # mixup-style dense labels
  for fn, ref_fn in ((ops.sigmoid_xent, O.sigmoid_xent), (ops.softmax_xent, O.softmax_xent)):
    lr = lg.double().requires_grad_(True)
    ref = ref_fn(lr, lab.double())
    ref.backward()
    loss = torch.zeros(1, device="cuda")
    dl = fn(lg.cuda(), lab.cuda(), loss)
    _close(loss, ref.reshape(1), 1e-5)
    _close(dl, lr.grad, 1e-4)


@pytest.mark.parametrize("mu_dtype", [torch.float32, torch.bfloat16])
def test_adam_matches_optax_chain(ops, mu_dtype):
  g = torch.Generator().manual_seed(3)
  n = 4096 * 3 + 4
  p0, gr = torch.randn(n, generator=g), torch.randn(n, generator=g) * 3
  p, mu, nu = p0.cuda(), torch.zeros(n, dtype=mu_dtype, device="cuda"), torch.zeros(n, device="cuda")
  p16 = torch.empty(n, dtype=torch.bfloat16, device="cuda")
  gsq = torch.zeros(1, device="cuda")
  ops.sumsq(gr.cuda(), gsq)
  pr, mr, vr = p0.double().numpy(), np.zeros(n), np.zeros(n)
  gnorm = float(np.linalg.norm(gr.double().numpy()))
  for step in (1, 2, 3):
    ops.adam_step(p, gr.cuda(), mu, nu, p16, lr_eff=1e-3 * 0.5, b1=0.9, b2=0.95, eps=1e-8,
                  wd_eff=1e-4 * 0.5, step=step, clip_norm=1.0, gnorm_sq=gsq)
    pr, mr, vr = O.adam_reference(pr, gr.double().numpy(), mr, vr, step, lr=1e-3, b1=0.9, b2=0.95,
                                  eps=1e-8, wd=1e-4, sched=0.5, clip=1.0, gnorm=gnorm)
    if mu_dtype == torch.bfloat16:
      mr = torch.tensor(mr).float().bfloat16().double().numpy()
  _close(p, torch.tensor(pr), 1e-5)
  assert torch.equal(p16.cpu(), p.cpu().bfloat16())


@pytest.mark.parametrize("n,N,d", [(3, 196, 768), (2, 12, 64), (2, 197, 72), (1, 64, 128), (2, 130, 200)])
def test_token_transposes_are_exact(ops, n, N, d):
  """MLP-Mixer token mixing (models/mlp_mixer.py:49-52): [n, N, d] -> [n, d, Np] with zero padding, and
  back fused with the residual add.  Pure data movement (+ one rounded add): bit-exact."""
  g = torch.Generator().manual_seed(n * 1000 + N)
  x = torch.randn(n, N, d, generator=g).bfloat16()
  Np = (N + 7) // 8 * 8
  yt = ops.transpose_tokens(x.view(n * N, d).cuda(), n, N, d).cpu().view(n, d, Np)
  assert torch.equal(yt[:, :, :N], x.transpose(1, 2))
  assert float(yt[:, :, N:].abs().max()) == 0.0 if Np > N else True
  # garbage in the padded columns of the input must not leak into the output
  y = torch.randn(n, d, Np, generator=g).bfloat16()
  res = torch.randn(n, N, d, generator=g).bfloat16()
  back = ops.untranspose_add(y.view(n * d, Np).cuda(), None, n, N, d).cpu().view(n, N, d)
  assert torch.equal(back, y[:, :, :N].transpose(1, 2))
  fused = ops.untranspose_add(y.view(n * d, Np).cuda(), res.view(n * N, d).cuda(), n, N, d).cpu().view(n, N, d)
  assert torch.equal(fused, (y[:, :, :N].transpose(1, 2).float() + res.float()).bfloat16())
