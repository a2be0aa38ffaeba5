"""The persistent GEMM at the training step's sizes: each tile's output bits do not depend on how many
work units a CTA runs or where the tile sits in the problem, TMA stores leave everything outside the
output alone, split-K weight gradients match fp64, and plain outputs are reproducible bit for bit."""
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
  g.manual_seed(0)

  def rnd(*shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)
  return lib, ops, rnd


def _bits(t):
  return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _same_bits(a, b):
  assert a.shape == b.shape and a.dtype == b.dtype
  assert torch.equal(_bits(a), _bits(b))


def _epilogue_call(L, ops, rnd, epi, M, N, K, block_n):
  """One bf16-output GEMM with the given epilogue; returns a callable on a row window [r0, r1) that
  computes those rows into fresh outputs (aux and the left operand are sliced, never copied)."""
  x = rnd(M, K)
  w = rnd(K, N, scale=0.03)
  bias = rnd(N, dtype=torch.float32)
  aux = rnd(M, N)
  pos = rnd(196, N)

  def run(r0, r1):
    m = r1 - r0
    o = torch.empty(m, N, device="cuda", dtype=torch.bfloat16)
    o2 = torch.empty(m, N, device="cuda", dtype=torch.bfloat16)
    kw = dict(b_mn=True, bias=bias, out=o, block_n=block_n)
    if epi == "bias":
      ops.gemm(x[r0:r1], w, **kw)
      return [o]
    if epi == "gelu":
      ops.gemm(x[r0:r1], w, out2=o2, epilogue=L.EPI_BIAS_GELU, **kw)
      return [o, o2]
    if epi == "resid":
      ops.gemm(x[r0:r1], w, aux=aux[r0:r1], epilogue=L.EPI_BIAS_RESID, **kw)
      return [o]
    if epi == "posemb":      # row-modulo aux; windows start at multiples of 196 * 128 / gcd = 128 * 49
      ops.gemm(x[r0:r1], w, aux=pos, aux_row_mod=196, epilogue=L.EPI_BIAS_RESID, **kw)
      return [o]
    if epi == "dgelu":
      ops.gemm(x[r0:r1], w.t().contiguous(), out=o, aux=aux[r0:r1], epilogue=L.EPI_DGELU, block_n=block_n)
      return [o]
    raise ValueError(epi)
  return run


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("epi", ["bias", "gelu", "resid", "posemb", "dgelu"])
def test_row_windows_give_identical_bits(env, epi, block_n):
  L, ops, rnd = env
  M, N, K = M_IMG - 41, 640, D          # ragged in M, and N not a multiple of 256
  run = _epilogue_call(L, ops, rnd, epi, M, N, K, block_n)
  full = run(0, M)
  step = 128 * 49                       # a multiple of 128 and of the 196-row position period
  for r0, r1 in ((step * 3, step * 5), (step * (M // step), M)):
    part = run(r0, r1)
    for f, p in zip(full, part):
      _same_bits(f[r0:r1], p)


@pytest.mark.parametrize("block_n", [128, 256])
def test_strided_output_leaves_other_columns(env, block_n):
  L, ops, rnd = env
  M, N, K = 5000, 1000, 256
  x, w, bias = rnd(M, K), rnd(K, N, scale=0.05), rnd(N, dtype=torch.float32)
  ref = {"bias": ops.gemm(x, w, b_mn=True, bias=bias, block_n=block_n)}
  ref["gelu"], ref2 = torch.empty_like(ref["bias"]), torch.empty_like(ref["bias"])
  ops.gemm(x, w, b_mn=True, bias=bias, out=ref["gelu"], out2=ref2, epilogue=L.EPI_BIAS_GELU, block_n=block_n)
  for epi in ("bias", "gelu"):
    wide = torch.full((M + 3, 1200), 7.0, device="cuda", dtype=torch.bfloat16)
    wide2 = torch.full((M + 3, 1200), -3.0, device="cuda", dtype=torch.bfloat16)
    keep, keep2 = wide.clone(), wide2.clone()
    o, o2 = wide[:M, 104:104 + N], wide2[:M, 56:56 + N]
    if epi == "bias":
      ops.gemm(x, w, b_mn=True, bias=bias, out=o, block_n=block_n)
    else:
      ops.gemm(x, w, b_mn=True, bias=bias, out=o, out2=o2, epilogue=L.EPI_BIAS_GELU, block_n=block_n)
      _same_bits(o2, ref2)
      keep2[:M, 56:56 + N] = o2
      _same_bits(wide2, keep2)
    _same_bits(o, ref[epi])
    keep[:M, 104:104 + N] = o
    _same_bits(wide, keep)


def test_small_and_ragged_problems(env):
  """M = 1 (the MAP probe), N = 1000 (a class head), and grids with fewer units than SMs."""
  L, ops, rnd = env
  for M, N, K in ((1, D, D), (3, 1000, 64), (130, 1000, 768), (200, 40, 192)):
    x, w, bias = rnd(M, K), rnd(K, N, scale=0.05), rnd(N, dtype=torch.float32)
    ref = x.double() @ w.double() + bias.double()
    for block_n in (128, 256):
      got = ops.gemm(x, w, b_mn=True, bias=bias, block_n=block_n).double()
      err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)
      assert err <= 2 ** -8, (M, N, K, block_n, err)


def test_split_k_wgrad_at_step_shape(env):
  L, ops, rnd = env
  x, h = rnd(M_IMG, D), rnd(M_IMG, MLP)
  ref = x.double().t() @ h.double()
  dw = torch.zeros(D, MLP, device="cuda", dtype=torch.float32)
  ops.gemm(x, h, a_mn=True, b_mn=True, out=dw, reduce_out=True)
  scale = ref.abs().max().item()
  assert (dw.double() - ref).abs().max().item() <= 1e-4 * scale
  start = rnd(D, MLP, dtype=torch.float32) * scale
  dw = start.clone()
  ops.gemm(x, h, a_mn=True, b_mn=True, out=dw, reduce_out=True)
  assert (dw.double() - (ref + start.double())).abs().max().item() <= 1e-4 * 2 * scale


def test_run_to_run_bits(env):
  L, ops, rnd = env
  for epi in ("bias", "gelu", "resid", "posemb", "dgelu"):
    run = _epilogue_call(L, ops, rnd, epi, M_IMG // 4, MLP, D, 0)
    a, b = run(0, M_IMG // 4), run(0, M_IMG // 4)
    for x, y in zip(a, b):
      _same_bits(x, y)
  # the colsum (bias gradient) goes through atomics and is only close; the output itself is exact
  x, w, aux = rnd(M_IMG // 4, D), rnd(MLP, D, scale=0.03), rnd(M_IMG // 4, MLP)
  outs = []
  for _ in range(2):
    cs = torch.zeros(MLP, device="cuda")
    outs.append((ops.gemm(x, w, aux=aux, epilogue=L.EPI_DGELU, colsum=cs), cs))
  _same_bits(outs[0][0], outs[1][0])
  ref = outs[0][0].double().sum(0)
  for _, cs in outs:
    assert (cs.double() - ref).abs().max().item() <= 1e-4 * (ref.abs().max().item() + 1)
