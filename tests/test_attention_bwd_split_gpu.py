"""The attention backward as two kernels that each own their outputs (dQ per query block, dK / dV per
key block): every head dim against autograd through the fp64 reference on shapes with several key
blocks and ragged edges, bit-for-bit reproducibility, the raw C ABI call, and the memory
one call allocates (no workspace that grows with the number of key blocks)."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

HEAD_DIMS = [64, 72, 80, 96, 104]
# ViT-B/16 with its class token, L/14 @ 336 with its class token, Nq != Nk both ways, the MAP head's
# single query over 196 keys
SHAPES = [(2, 3, 197, 197), (1, 2, 577, 577), (2, 2, 150, 300), (2, 2, 300, 129), (3, 2, 1, 196)]


@pytest.fixture(scope="module")
def ops():
  from big_vision_b200 import lib, ops as _ops
  assert lib.load().bv_device_supported() == 1
  return _ops


def _bf(x):
  return x.to(torch.bfloat16)


def _close(got, ref, tol):
  got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
  assert not torch.isnan(got).any()
  err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)
  assert err <= tol, f"rel err {err:.3e} > {tol}"


def _ref_attention(q, k, v, H):
  B, Nq, d = q.shape
  Nk, dh = k.shape[1], d // H
  qh = q.reshape(B, Nq, H, dh).transpose(1, 2)
  kh = k.reshape(B, Nk, H, dh).transpose(1, 2)
  vh = v.reshape(B, Nk, H, dh).transpose(1, 2)
  s = qh @ kh.transpose(-1, -2) / math.sqrt(dh)
  return (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, Nq, d)


def _inputs(B, H, Nq, Nk, dh, seed):
  g = torch.Generator().manual_seed(seed)
  d = H * dh
  qkv = _bf(torch.randn(B, max(Nq, Nk), 3 * d, generator=g))
  qkv[:, ::37, 0:d] *= 4.0     # a few large scores per row
  do = _bf(torch.randn(B, Nq, d, generator=g))
  return qkv, do


@pytest.mark.parametrize("dh", HEAD_DIMS)
@pytest.mark.parametrize("B,H,Nq,Nk", SHAPES)
def test_backward_matches_fp64(ops, dh, B, H, Nq, Nk):
  d = H * dh
  qkv, do = _inputs(B, H, Nq, Nk, dh, B * 1000 + Nq + Nk + dh)
  qr = qkv[:, :Nq, 0:d].double().requires_grad_(True)
  kr = qkv[:, :Nk, d:2 * d].double().requires_grad_(True)
  vr = qkv[:, :Nk, 2 * d:].double().requires_grad_(True)
  _ref_attention(qr, kr, vr, H).backward(do.double())
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


@pytest.mark.parametrize("dh", [80, 96])
def test_backward_is_bitwise_reproducible(ops, dh):
  B, H, Nq, Nk = 2, 4, 197, 261
  d = H * dh
  qkv, do = _inputs(B, H, Nq, Nk, dh, 21 + dh)
  c, do = qkv.cuda(), do.cuda()
  q, k, v = c[:, :Nq, 0:d], c[:, :Nk, d:2 * d], c[:, :Nk, 2 * d:]
  o, lse = ops.attention_fwd(q, k, v, H)
  runs = []
  for _ in range(2):
    cs = torch.zeros(3, d, device="cuda")
    runs.append(ops.attention_bwd(do, q, k, v, o, lse, H, dq_colsum=cs[0], dk_colsum=cs[1], dv_colsum=cs[2]))
  for a, b in zip(*runs):
    assert torch.equal(a, b)


@pytest.mark.parametrize("dh", [64, 104])
def test_raw_abi_without_dq_accum(ops, dh):
  """bv_attention_bwd_hd called through the raw C ABI gives the bits of ops.attention_bwd."""
  from big_vision_b200 import lib as L
  B, H, N = 2, 3, 197
  d = H * dh
  qkv, do = _inputs(B, H, N, N, dh, 5 + dh)
  c, do = qkv.cuda(), do.cuda()
  q, k, v = c[:, :, 0:d], c[:, :, d:2 * d], c[:, :, 2 * d:]
  o, lse = ops.attention_fwd(q, k, v, H)
  want = ops.attention_bwd(do, q, k, v, o, lse, H)
  f = ops._attn_args(q, k, v, o, lse, H, 1 / math.sqrt(dh))  # pylint: disable=protected-access
  dq, dk, dv = (torch.empty(B, N, d, dtype=torch.bfloat16, device="cuda") for _ in range(3))
  delta = torch.empty(B, H, N, device="cuda")
  a = L.AttnBwdArgs(fwd=f, d_o=do.data_ptr(), lddo=d, bsdo=N * d, dq=dq.data_ptr(), dk=dk.data_ptr(),
                    dv=dv.data_ptr(), lddq=d, lddk=d, lddv=d, bsdq=N * d, bsdk=N * d, bsdv=N * d,
                    delta=delta.data_ptr())
  L.call("bv_attention_bwd_hd", ctypes.byref(a), dh, None)
  torch.cuda.synchronize()
  for got, ref in zip((dq, dk, dv), want):
    assert torch.equal(got, ref)


def test_backward_allocates_only_its_outputs(ops):
  """One call at the L/14 @ 336 geometry (16 heads, 576 tokens, nine key blocks) allocates dq, dk, dv
  and delta and nothing that scales with the number of key blocks."""
  B, H, N, dh = 32, 16, 576, 64
  d = H * dh
  g = torch.Generator(device="cuda").manual_seed(3)
  c = torch.randn(B, N, 3 * d, device="cuda", generator=g).to(torch.bfloat16)
  do = torch.randn(B, N, d, device="cuda", generator=g).to(torch.bfloat16)
  q, k, v = c[:, :, 0:d], c[:, :, d:2 * d], c[:, :, 2 * d:]
  o, lse = ops.attention_fwd(q, k, v, H)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  base = torch.cuda.memory_allocated()
  out = ops.attention_bwd(do, q, k, v, o, lse, H)
  torch.cuda.synchronize()
  grew = torch.cuda.max_memory_allocated() - base
  allowed = 3 * B * N * d * 2 + B * H * N * 4
  assert grew <= allowed + (1 << 20), f"{grew} bytes allocated, outputs and delta are {allowed}"
  assert all(bool(torch.isfinite(t.float()).all()) for t in out)
