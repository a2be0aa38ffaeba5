"""The GEMM epilogues whose aux operand (the residual, gelu''s saved pre-activation) arrives by TMA into
the output's staging buffers: their bf16 outputs equal, bit for bit, an oracle built from paths that
read aux from the registers, with strided aux, ragged shapes, and enough work units per CTA that every
staging buffer and its barrier are reused many times."""
import pytest
import torch

pytestmark = pytest.mark.gpu

M_IMG = 768 * 196          # image-tower tokens of the 768-pair step
D, MLP = 768, 3072


@pytest.fixture(scope="module")
def env():
  from big_vision_b200 import lib, ops
  assert lib.load().bv_device_supported() == 1, "needs a compute-capability 9.x GPU"
  g = torch.Generator(device="cuda")
  g.manual_seed(1)

  def rnd(*shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)
  return lib, ops, rnd


def _same_bits(a, b):
  assert a.shape == b.shape and a.dtype == b.dtype == torch.bfloat16
  assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def _strided(t, lead, trail, fill):
  """t copied into columns [lead, lead + N) of a wider buffer filled with `fill`: (view, buffer)."""
  M, N = t.shape
  buf = torch.full((M + 2, lead + N + trail), fill, device=t.device, dtype=t.dtype)
  v = buf[:M, lead:lead + N]
  v.copy_(t)
  return v, buf


def _resid_oracle(ops, x, w, bias, aux, block_n):
  """round_bf16(x w + bias) + aux in bf16: the fp32-output GEMM has the same accumulators."""
  f = ops.gemm(x, w, b_mn=True, bias=bias, out_dtype=torch.float32, block_n=block_n)
  return (f.to(torch.bfloat16).float() + aux.float()).to(torch.bfloat16)


def _dgelu_oracle(L, ops, x, w, aux):
  """The bf16 reduce-add path reads aux from the registers; adding to zero returns each value exactly
  (a -0 result becomes +0, so the caller compares with -0 mapped to +0).  One K split, so that each
  element is added once."""
  o = torch.zeros(x.shape[0], w.shape[0], device="cuda", dtype=torch.bfloat16)
  ops.gemm(x, w, aux=aux, out=o, epilogue=L.EPI_DGELU, reduce_out=True, splits=1, block_n=128)
  return o


def _plus_zero(t):
  return torch.where(t == 0, torch.zeros_like(t), t)


# (M, N, K): the out_proj and Dense_1 shapes at the text tower's M (each CTA runs >= 4 units at either
# tile width); N = 1000 (a sub-tile partly past the edge); M = 1 (mod 64); M = 1
SHAPES = [(768 * 64, D, D), (768 * 64, D, MLP), (4097, 1000, 256), (65, 640, 128), (1, 1000, 64)]


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_resid_matches_fp32_oracle(env, M, N, K, block_n):
  L, ops, rnd = env
  x, w, bias, aux = rnd(M, K), rnd(K, N, scale=0.05), rnd(N, dtype=torch.float32), rnd(M, N)
  ref = _resid_oracle(ops, x, w, bias, aux, block_n)
  got = ops.gemm(x, w, b_mn=True, bias=bias, aux=aux, epilogue=L.EPI_BIAS_RESID, block_n=block_n)
  _same_bits(got, ref)
  _same_bits(ops.gemm(x, w, b_mn=True, bias=bias, aux=aux, epilogue=L.EPI_BIAS_RESID, block_n=block_n), got)


@pytest.mark.parametrize("M,N,K", SHAPES + [(768 * 64, MLP, D)])
def test_dgelu_matches_register_path(env, M, N, K):
  L, ops, rnd = env
  x, w, aux = rnd(M, K), rnd(N, K, scale=0.05), rnd(M, N)
  ref = _dgelu_oracle(L, ops, x, w, aux)
  got = ops.gemm(x, w, aux=aux, epilogue=L.EPI_DGELU, block_n=128)
  _same_bits(_plus_zero(got), _plus_zero(ref))
  _same_bits(ops.gemm(x, w, aux=aux, epilogue=L.EPI_DGELU, block_n=128), got)
  # BN = 256 runs the other instantiation; the colsum is the column sum of the stored values
  cs = torch.zeros(N, device="cuda")
  got256 = ops.gemm(x, w, aux=aux, epilogue=L.EPI_DGELU, colsum=cs, block_n=256)
  _same_bits(ops.gemm(x, w, aux=aux, epilogue=L.EPI_DGELU, block_n=256), got256)
  ref_cs = got256.double().sum(0)
  assert (cs.double() - ref_cs).abs().max().item() <= 1e-4 * (ref_cs.abs().max().item() + 1)


@pytest.mark.parametrize("block_n", [128, 256])
def test_strided_aux_inside_nan_sentinels(env, block_n):
  """aux is a column slice of a wider buffer (as q, k or v of a fused qkv activation would be); NaN
  around it would reach any output element that read past the slice."""
  L, ops, rnd = env
  M, N, K = 5000, 1000, 256
  x, w, bias = rnd(M, K), rnd(K, N, scale=0.05), rnd(N, dtype=torch.float32)
  aux = rnd(M, N)
  av, abuf = _strided(aux, 104, 96, float("nan"))
  keep = abuf.clone()
  ref = _resid_oracle(ops, x, w, bias, aux, block_n)
  _same_bits(ops.gemm(x, w, b_mn=True, bias=bias, aux=av, epilogue=L.EPI_BIAS_RESID, block_n=block_n), ref)
  wt = w.t().contiguous()
  ref = _dgelu_oracle(L, ops, x, wt, aux)
  got = ops.gemm(x, wt, aux=av, epilogue=L.EPI_DGELU, block_n=block_n)
  if block_n == 128:
    _same_bits(_plus_zero(got), _plus_zero(ref))
  assert not torch.isnan(got.float()).any()
  _same_bits(got, ops.gemm(x, wt, aux=aux, epilogue=L.EPI_DGELU, block_n=block_n))
  assert torch.equal(abuf.view(torch.int16), keep.view(torch.int16))     # aux is only read


@pytest.mark.parametrize("block_n", [128, 256])
def test_resid_in_place(env, block_n):
  """Output and aux the same tensor: each tile's aux is loaded before its output is stored."""
  L, ops, rnd = env
  M, N, K = 768 * 64, D, D
  x, w, bias, aux = rnd(M, K), rnd(K, N, scale=0.05), rnd(N, dtype=torch.float32), rnd(M, N)
  ref = _resid_oracle(ops, x, w, bias, aux, block_n)
  ops.gemm(x, w, b_mn=True, bias=bias, aux=aux, out=aux, epilogue=L.EPI_BIAS_RESID, block_n=block_n)
  _same_bits(aux, ref)


def test_resid_at_step_shape(env):
  L, ops, rnd = env
  M, N, K = M_IMG, D, MLP
  x, w, bias, aux = rnd(M, K), rnd(K, N, scale=0.03), rnd(N, dtype=torch.float32), rnd(M, N)
  ref = _resid_oracle(ops, x, w, bias, aux, 0)
  _same_bits(ops.gemm(x, w, b_mn=True, bias=bias, aux=aux, epilogue=L.EPI_BIAS_RESID), ref)
