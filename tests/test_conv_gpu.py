"""GPU: the BiT ResNet-v2 kernels of include/bv_conv.h against float64.

Convolutions (forward, data gradient, kernel gradient) at the shapes of R50x1 and R152x2 and ragged extras,
element-wise under the bound |got - ref| <= REL * |ref| + ACC * ref_abs, where ref_abs is the same
convolution of |operands| in float64: REL covers the one bf16 rounding of an output (none for the fp32 kernel
gradient), ACC the fp32 accumulation.  Weight standardisation, GroupNorm + ReLU, the max pool and the stem's
patch extraction against float64 too."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from big_vision_b200 import lib as L
from big_vision_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF16_REL = 2.0 ** -8
ACC = 2.0 ** -16


def _bf16(shape, gen, scale=1.0):
  return (torch.randn(shape, generator=gen, dtype=torch.float64) * scale).to(torch.bfloat16)


def _nan_padded(t, pad=64):
  """t copied into the middle of a NaN-filled buffer: a kernel that reads past the tensor meets NaN."""
  buf = torch.full((t.numel() + 2 * pad,), float("nan"), dtype=t.dtype, device=DEV)
  view = buf[pad:pad + t.numel()].view(t.shape)
  view.copy_(t.to(DEV))
  return view


def _conv64(x, w, stride):
  """float64 NHWC x HWIO convolution with padding k // 2."""
  k = w.shape[0]
  y = F.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), stride=stride, padding=k // 2)
  return y.permute(0, 2, 3, 1)


def _refs(x, w, dy, stride):
  """(y, dx, dw) and the same of the absolute values, all float64."""
  x64, w64, dy64 = (t.double().requires_grad_() for t in (x, w, dy))
  y = _conv64(x64, w64, stride)
  dx, dw = torch.autograd.grad(y, (x64, w64), dy64)
  xa, wa, dya = (t.double().abs().requires_grad_() for t in (x, w, dy))
  ya = _conv64(xa, wa, stride)
  dxa, dwa = torch.autograd.grad(ya, (xa, wa), dya)
  return (y.detach(), dx, dw), (ya.detach(), dxa, dwa)


def _check(got, ref, ref_abs, rel, what, rounded=None):
  """`rounded`: the value rounded to bf16 before a residual was added to it (so it is rounded twice)."""
  err = (got.double().cpu() - ref).abs()
  bound = rel * ref.abs() + ACC * ref_abs + 1e-30
  if rounded is not None:
    bound = bound + rel * rounded.abs()
  worst = (err / bound).max().item()
  assert torch.isfinite(got).all(), what
  assert worst <= 1.0, f"{what}: error {worst:.3f} x the bound"


def bit_shapes():
  """Every (k, stride, cin, cout, h) of a convolution with more than 3 input channels that R50x1 and R152x2
  meet at 224, 160 and 128 px (h: the input's size; the 1 x 1 stride-1 ones run on bv_gemm)."""
  out = set()
  for blocks, width in (([3, 4, 6, 3], 64), ([3, 8, 36, 3], 128)):
    for px in (224, 160, 128):
      h = ((px - 1) // 2) // 2 + 1                  # root convolution, then max pool
      cin = width
      for b, size in enumerate(blocks):
        nmid, s = width * 2 ** b, 2 if b else 1
        ho = (h - 1) // s + 1
        out |= {(1, s, cin, 4 * nmid, h), (1, 1, cin, nmid, h), (3, s, nmid, nmid, h), (1, 1, nmid, 4 * nmid, ho)}
        out |= {(1, 1, 4 * nmid, nmid, ho), (3, 1, nmid, nmid, ho)} if size > 1 else set()
        cin, h = 4 * nmid, ho
  return sorted(out)


BIT_SHAPES = bit_shapes()
EXTRA_SHAPES = [(3, 2, 64, 192, 7), (1, 2, 64, 128, 9), (3, 1, 192, 64, 3), (7, 1, 64, 64, 9), (7, 2, 64, 128, 11),
                (3, 2, 64, 64, 1), (3, 1, 64, 64, 1)]


@pytest.mark.parametrize("k,stride,cin,cout,h", BIT_SHAPES + EXTRA_SHAPES)
def test_convolutions_match_fp64(k, stride, cin, cout, h):
  gen = torch.Generator().manual_seed(k * 1000 + stride * 100 + h)
  n, w = 2, h + (1 if h > 4 else 0)      # non-square where there is room
  ho, wo = ops.conv_out_size(h, k, stride), ops.conv_out_size(w, k, stride)
  x = _bf16((n, h, w, cin), gen)
  kern = _bf16((k, k, cin, cout), gen, scale=(k * k * cin) ** -0.5)
  dy = _bf16((n, ho, wo, cout), gen)
  resid = _bf16((n, ho, wo, cout), gen)
  dresid = _bf16((n, h, w, cin), gen)
  (y, dx, dw), (ya, dxa, dwa) = _refs(x, kern, dy, stride)

  xd, kd, dyd = _nan_padded(x), _nan_padded(kern), _nan_padded(dy)
  _check(ops.conv_fwd(xd, kd, stride), y, ya, BF16_REL, "forward")
  _check(ops.conv_fwd(xd, kd, stride, resid=_nan_padded(resid)), y + resid.double(), ya + resid.double().abs(),
         BF16_REL, "forward + residual", rounded=y)
  _check(ops.conv_dgrad(dyd, kd, h, w, stride), dx, dxa, BF16_REL, "data gradient")
  _check(ops.conv_dgrad(dyd, kd, h, w, stride, resid=_nan_padded(dresid)), dx + dresid.double(),
         dxa + dresid.double().abs(), BF16_REL, "data gradient + residual", rounded=dx)
  _check(ops.conv_wgrad(xd, dyd, k, stride), dw, dwa, 0.0, "kernel gradient")
  acc = torch.ones((k, k, cin, cout), dtype=torch.float32, device=DEV)
  _check(ops.conv_wgrad(xd, dyd, k, stride, out=acc), dw + 1.0, dwa + 1.0, 0.0, "accumulated kernel gradient")


def test_outputs_stay_inside_their_buffers():
  """Each entry point writes exactly its output: sentinels right before and after it survive."""
  gen = torch.Generator().manual_seed(3)
  n, h, w, cin, cout, k, s = 2, 9, 7, 64, 128, 3, 2
  ho, wo = ops.conv_out_size(h, k, s), ops.conv_out_size(w, k, s)
  x = _bf16((n, h, w, cin), gen).to(DEV)
  kern = _bf16((k, k, cin, cout), gen, scale=0.05).to(DEV)
  dy = _bf16((n, ho, wo, cout), gen).to(DEV)
  pad = 64

  def framed(numel, dtype):
    buf = torch.full((numel + 2 * pad,), 12345.0, dtype=dtype, device=DEV)
    return buf, buf[pad:pad + numel]

  ybuf, y = framed(n * ho * wo * cout, torch.bfloat16)
  dxbuf, dx = framed(n * h * w * cin, torch.bfloat16)
  dwbuf, dw = framed(k * k * cin * cout, torch.float32)
  ws = torch.empty(n * h * w * cin, dtype=torch.bfloat16, device=DEV)
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  a = L.ConvArgs(x=p(x), kernel=p(kern), dy=p(dy), y=p(y), dx=p(dx), dkernel=p(dw), workspace=p(ws), n=n, h=h, w=w,
                 cin=cin, cout=cout, k=k, stride=s)
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  for fn in ("bv_conv_fwd", "bv_conv_dgrad", "bv_conv_wgrad"):
    L.call(fn, ctypes.byref(a), stream)
  torch.cuda.synchronize()
  for buf in (ybuf, dxbuf, dwbuf):
    assert (buf[:pad] == 12345.0).all() and (buf[-pad:] == 12345.0).all()
  assert torch.equal(y.view(n, ho, wo, cout), ops.conv_fwd(x, kern, s))
  assert torch.equal(dx.view(n, h, w, cin), ops.conv_dgrad(dy, kern, h, w, s))


@pytest.mark.parametrize("cin,cout,hw", [(64, 256, 56), (256, 64, 56), (1024, 256, 14), (2048, 512, 7)])
def test_one_by_one_stride_one_is_bv_gemm(cin, cout, hw):
  gen = torch.Generator().manual_seed(cin + cout)
  x = _bf16((2, hw, hw, cin), gen).to(DEV)
  kern = _bf16((1, 1, cin, cout), gen, scale=cin ** -0.5).to(DEV)
  resid = _bf16((2, hw, hw, cout), gen).to(DEV)
  got = ops.conv_fwd(x, kern, 1, resid=resid)
  want = ops.gemm(x.view(-1, cin), kern.view(cin, cout), b_mn=True, aux=resid.view(-1, cout),
                  epilogue=L.EPI_BIAS_RESID)
  assert torch.equal(got.view(-1, cout), want)
  (y, _, _), (ya, _, _) = _refs(x.cpu(), kern.cpu(), resid.cpu(), 1)
  _check(got, y + resid.double().cpu(), ya + resid.double().abs().cpu(), BF16_REL, "1x1 forward", rounded=y)


@pytest.mark.parametrize("shape", [(7, 7, 3, 64), (3, 3, 64, 64), (1, 1, 256, 1024), (3, 3, 512, 512)])
def test_weight_standardisation_matches_fp64(shape):
  gen = torch.Generator().manual_seed(sum(shape))
  w = torch.randn(shape, generator=gen, dtype=torch.float64) * 0.1 + 0.03
  g = torch.randn(shape, generator=gen, dtype=torch.float64)
  w64 = w.clone().requires_grad_()
  mu = w64.mean(dim=(0, 1, 2), keepdim=True)
  d = w64 - mu
  ref = d / torch.sqrt((d * d).mean(dim=(0, 1, 2), keepdim=True) + 1e-10)
  (dref,) = torch.autograd.grad(ref, w64, g)
  wd = w.float().to(DEV)
  ws, mean, rstd = ops.weight_std_fwd(wd)
  err = (ws.double().cpu() - ref.detach()).abs()
  assert (err <= BF16_REL * ref.detach().abs() + 1e-5).all()
  dw = ops.weight_std_bwd(wd, mean, rstd, g.float().to(DEV))
  scale = dref.abs().max()
  assert ((dw.double().cpu() - dref).abs() <= 1e-4 * scale).all()
  ws2, _, _ = ops.weight_std_fwd(wd)
  assert torch.equal(ws, ws2)


@pytest.mark.parametrize("n,hw,c,relu", [(2, 56 * 56, 64, True), (2, 14 * 14, 1024, True), (3, 7 * 7, 4096, True),
                                         (2, 5 * 5, 192, False), (1, 1, 32, True)])
def test_groupnorm_relu_matches_fp64(n, hw, c, relu):
  gen = torch.Generator().manual_seed(n * c + hw)
  x = _bf16((n, hw, c), gen, scale=2.0) + 0.5
  dy = _bf16((n, hw, c), gen)
  scale = torch.randn(c, generator=gen, dtype=torch.float64) * 0.5 + 1.0
  bias = torch.randn(c, generator=gen, dtype=torch.float64) * 0.2
  x64 = x.double().requires_grad_()
  s64, b64 = scale.clone().requires_grad_(), bias.clone().requires_grad_()
  xg = x64.view(n, hw, 32, c // 32)
  mu = xg.mean(dim=(1, 3), keepdim=True)
  dd = xg - mu
  z = (dd / torch.sqrt((dd * dd).mean(dim=(1, 3), keepdim=True) + 1e-5)).view(n, hw, c) * s64 + b64
  ref = torch.relu(z) if relu else z
  dx_ref, ds_ref, db_ref = torch.autograd.grad(ref, (x64, s64, b64), dy.double())
  xd = x.to(DEV)
  y, mean, rstd = ops.groupnorm_fwd(xd, scale.float().to(DEV), bias.float().to(DEV), relu=relu)
  ref = ref.detach()
  assert ((y.double().cpu() - ref).abs() <= BF16_REL * ref.abs() + 1e-4 * (1 + ref.abs().max())).all()
  dscale = torch.zeros(c, dtype=torch.float32, device=DEV)
  dbias = torch.zeros_like(dscale)
  add = _bf16((n, hw, c), gen).to(DEV)
  dx = ops.groupnorm_bwd(dy.to(DEV), xd, scale.float().to(DEV), bias.float().to(DEV), mean, rstd, dscale, dbias,
                         relu=relu, dx_add=add)
  want = dx_ref + add.double().cpu()
  tol = BF16_REL * want.abs() + 1e-3 * (dx_ref.abs().max() + 1e-3)
  assert ((dx.double().cpu() - want).abs() <= tol).all()
  for got, r in ((dscale, ds_ref), (dbias, db_ref)):
    assert ((got.double().cpu() - r).abs() <= 1e-4 * (r.abs().max() + 1e-3)).all()


def _maxpool64(x):
  y = F.max_pool2d(x.double().permute(0, 3, 1, 2), 3, 2, padding=1)
  return y.permute(0, 2, 3, 1)


def _first_max_grad(x, dy):
  """float64 backward that routes each gradient to the first maximal element of its window (row-major)."""
  n, h, w, c = x.shape
  ho, wo = dy.shape[1], dy.shape[2]
  xp = torch.full((n, h + 2, w + 2, c), float("-inf"), dtype=torch.float64)
  xp[:, 1:h + 1, 1:w + 1] = x.double()
  dx = torch.zeros((n, h + 2, w + 2, c), dtype=torch.float64)
  for i in range(ho):
    for j in range(wo):
      win = xp[:, 2 * i:2 * i + 3, 2 * j:2 * j + 3].reshape(n, 9, c)
      first = win.argmax(dim=1)    # torch.argmax returns the first maximal index
      for q in range(9):
        sel = (first == q).double()
        dx[:, 2 * i + q // 3, 2 * j + q % 3] += sel * dy[:, i, j].double()
  return dx[:, 1:h + 1, 1:w + 1]


@pytest.mark.parametrize("h,w", [(112, 112), (7, 9), (2, 3)])
def test_maxpool_forward_and_first_max_backward(h, w):
  gen = torch.Generator().manual_seed(h * w)
  n, c = 2, 64
  # integer values in a small range: many ties, so the backward's routing is checked exactly
  x = torch.randint(-4, 4, (n, h, w, c), generator=gen).to(torch.bfloat16)
  # an all-negative border window: with zero padding its maximum would be 0
  x[0, :2, :2, :] = -3.0
  dy = torch.randint(-8, 8, (n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c), generator=gen).to(torch.bfloat16)
  y = ops.maxpool_fwd(x.to(DEV))
  assert torch.equal(y.double().cpu(), _maxpool64(x))
  assert (y[0, 0, 0].float() == -3.0).all()
  dx = ops.maxpool_bwd(dy.to(DEV), x.to(DEV))
  assert torch.equal(dx.double().cpu(), _first_max_grad(x, dy))


@pytest.mark.parametrize("h,w", [(224, 224), (33, 18)])
def test_stem_convolution_matches_fp64(h, w):
  gen = torch.Generator().manual_seed(h + w)
  n, cout = 2, 64
  img = torch.randn((n, h, w, 3), generator=gen, dtype=torch.float64).float()
  kern = _bf16((7, 7, 3, cout), gen, scale=147 ** -0.5)
  y = ops.stem_conv_fwd(img.to(DEV), kern.to(DEV))
  x_bf = img.to(torch.bfloat16)     # the patches are bf16
  ref = _conv64(x_bf.double(), kern.double(), 2)
  ref_abs = _conv64(x_bf.double().abs(), kern.double().abs(), 2)
  _check(y, ref, ref_abs, BF16_REL, "stem forward")
  dy = _bf16(ref.shape, gen)
  x64, w64 = x_bf.double(), kern.double().requires_grad_()
  (dw,) = torch.autograd.grad(_conv64(x64, w64, 2), (w64,), dy.double())
  wa = kern.double().abs().requires_grad_()
  (dwa,) = torch.autograd.grad(_conv64(x64.abs(), wa, 2), (wa,), dy.double().abs())
  _check(ops.stem_conv_wgrad(img.to(DEV), dy.to(DEV)), dw, dwa, 0.0, "stem kernel gradient")
