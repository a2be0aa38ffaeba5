"""GPU parity of the key-block streaming attention kernels (attention.cu) against the fp64 reference
attention: long sequences (config 5: 576 / 577 keys; ragged and very long cases) and the short shapes
of the ViT and text towers.  Tolerances as in test_kernels_gpu.py (bf16 operands, un-normalised bf16
probabilities, fp32 accumulation)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _bf(x):
  return x.to(torch.bfloat16)


def _close(got, ref, tol):
  got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
  assert not torch.isnan(got).any()
  err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)
  assert err <= tol, f"rel err {err:.3e} > {tol}"


def _ref_attention(q, k, v, H):
  B, Nq, d = q.shape
  Nk = k.shape[1]
  qh = q.reshape(B, Nq, H, 64).transpose(1, 2)
  kh = k.reshape(B, Nk, H, 64).transpose(1, 2)
  vh = v.reshape(B, Nk, H, 64).transpose(1, 2)
  s = qh @ kh.transpose(-1, -2) / 8.0
  return (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, Nq, d), torch.logsumexp(s, -1)


@pytest.fixture(scope="module")
def ops():
  from big_vision_b200 import lib, ops as _ops
  assert lib.load().bv_device_supported() == 1
  return _ops


SHAPES = [(2, 16, 576, 576), (2, 3, 577, 577), (1, 2, 300, 700), (3, 2, 1, 576), (1, 1, 1025, 130),
          (3, 2, 64, 64), (2, 12, 196, 196), (5, 3, 197, 197), (4, 2, 1, 196), (2, 1, 16, 16), (2, 2, 130, 7)]


@pytest.mark.parametrize("B,H,Nq,Nk", SHAPES)
def test_stream_forward(ops, B, H, Nq, Nk):
  g = torch.Generator().manual_seed(B * 1000 + Nq)
  d = H * 64
  qkv = _bf(torch.randn(B, max(Nq, Nk), 3 * d, generator=g))
  # a few large scores per row: the per-block maxima differ by far more than the bf16 range of P
  qkv[:, ::37, 0:d] *= 4.0
  q64, k64, v64 = qkv[:, :Nq, 0:d].double(), qkv[:, :Nk, d:2 * d].double(), qkv[:, :Nk, 2 * d:].double()
  o_ref, lse_ref = _ref_attention(q64, k64, v64, H)
  c = qkv.cuda()
  o, lse = ops.attention_fwd(c[:, :Nq, 0:d], c[:, :Nk, d:2 * d], c[:, :Nk, 2 * d:], H)
  torch.cuda.synchronize()
  _close(o, o_ref, 2 ** -6)
  _close(lse, lse_ref, 1e-5)


REPRO_SHAPES = [(8, 12, 196, 196), (2, 16, 576, 576), (3, 2, 1, 576)]


@pytest.mark.parametrize("B,H,Nq,Nk", REPRO_SHAPES)
def test_attention_forward_is_bitwise_reproducible(ops, B, H, Nq, Nk):
  """Same inputs twice through the forward: identical outputs and log-sum-exps, bit for bit."""
  g = torch.Generator().manual_seed(3 + Nq)
  d = H * 64
  c = _bf(torch.randn(B, max(Nq, Nk), 3 * d, generator=g)).cuda()
  q, k, v = c[:, :Nq, 0:d], c[:, :Nk, d:2 * d], c[:, :Nk, 2 * d:]
  o1, l1 = ops.attention_fwd(q, k, v, H)
  o2, l2 = ops.attention_fwd(q, k, v, H)
  assert torch.equal(o1, o2) and torch.equal(l1, l2)


def test_stream_forward_rows_are_convex_combinations_at_config5_size(ops):
  """Size-independent property at the config-5 shape (576 keys, 16 heads): with v constant per
  column every output row equals that constant, whatever the scores are."""
  B, H, N = 32, 16, 576
  d = H * 64
  g = torch.Generator(device="cuda").manual_seed(1)
  q = torch.randn(B, N, d, generator=g, device="cuda").to(torch.bfloat16) * 3
  k = torch.randn(B, N, d, generator=g, device="cuda").to(torch.bfloat16)
  col = torch.randn(1, 1, d, generator=g, device="cuda").to(torch.bfloat16)
  o, _ = ops.attention_fwd(q, k, col.expand(B, N, d).contiguous(), H)
  assert (o.float() - col.float()).abs().max().item() <= 2 ** -7 * col.float().abs().max().item()


BWD_SHAPES = [(2, 16, 576, 576), (2, 3, 577, 577), (1, 2, 300, 700), (3, 2, 1, 576),
              (3, 2, 64, 64), (2, 12, 196, 196), (5, 3, 197, 197), (4, 2, 1, 196), (2, 2, 130, 7)]


@pytest.mark.parametrize("B,H,Nq,Nk", BWD_SHAPES)
def test_stream_backward(ops, B, H, Nq, Nk):
  """Key-block streaming backward (per-key-block fp32 dQ slices, delta pre-kernel) against autograd
  through the fp64 reference, with caller-provided destination views."""
  g = torch.Generator().manual_seed(B * 1000 + Nq)
  d = H * 64
  qkv = _bf(torch.randn(B, max(Nq, Nk), 3 * d, generator=g))
  do = _bf(torch.randn(B, Nq, d, generator=g))
  qr = qkv[:, :Nq, 0:d].double().requires_grad_(True)
  kr = qkv[:, :Nk, d:2 * d].double().requires_grad_(True)
  vr = qkv[:, :Nk, 2 * d:].double().requires_grad_(True)
  o_ref, _ = _ref_attention(qr, kr, vr, H)
  o_ref.backward(do.double())
  c = qkv.cuda()
  q, k, v = c[:, :Nq, 0:d], c[:, :Nk, d:2 * d], c[:, :Nk, 2 * d:]
  o, lse = ops.attention_fwd(q, k, v, H)
  dqkv = torch.zeros_like(c)
  cs = torch.ones(3, d, device="cuda")
  dq, dk, dv = ops.attention_bwd(do.cuda(), q, k, v, o, lse, H, dq=dqkv[:, :Nq, 0:d], dk=dqkv[:, :Nk, d:2 * d],
                                 dv=dqkv[:, :Nk, 2 * d:], dq_colsum=cs[0], dk_colsum=cs[1], dv_colsum=cs[2])
  torch.cuda.synchronize()
  _close(dq, qr.grad, 2 ** -5)
  _close(dk, kr.grad, 2 ** -5)
  _close(dv, vr.grad, 2 ** -5)
  for i, t in enumerate((dq, dk, dv)):      # fused bias gradients: column sums over the valid rows
    ref = 1 + t.double().sum((0, 1))
    assert (cs[i].double() - ref).abs().max().item() <= 1e-4 * (ref.abs().max().item() + 1)
  # rows past Nq / Nk of the destination buffers were not touched
  assert float(dqkv[:, Nq:, 0:d].abs().max() if Nq < dqkv.shape[1] else 0) == 0
  assert float(dqkv[:, Nk:, d:].abs().max() if Nk < dqkv.shape[1] else 0) == 0


@pytest.mark.parametrize("B,H,Nq,Nk", REPRO_SHAPES)
def test_attention_backward_is_bitwise_reproducible(ops, B, H, Nq, Nk):
  """Same inputs twice through the backward: identical dq / dk / dv, bit for bit (each key block's dQ
  contribution has its own fp32 slice, and the slices are summed in key-block order)."""
  g = torch.Generator().manual_seed(4 + Nq)
  d = H * 64
  c = _bf(torch.randn(B, max(Nq, Nk), 3 * d, generator=g)).cuda()
  do = _bf(torch.randn(B, Nq, d, generator=g)).cuda()
  q, k, v = c[:, :Nq, 0:d], c[:, :Nk, d:2 * d], c[:, :Nk, 2 * d:]
  o, lse = ops.attention_fwd(q, k, v, H)
  r = ops.attention_bwd(do, q, k, v, o, lse, H)
  t = ops.attention_bwd(do, q, k, v, o, lse, H)
  for a, b in zip(t, r):
    assert torch.equal(a, b)
