"""GPU: attention with a key-padding mask (head_dim | BV_ATTN_KEY_MASK, head dim 64).

Forward and backward against an fp64 reference computed from the same bf16 inputs, element-wise, at
N = 16 (BERT's captions), 64, 128 and 577, with suffix masks (zero padding), random masks (masked keys
inside every 64-key block) and batches whose keys are all masked (O = 0, lse = 0, zero gradients).
Masked keys get exactly zero dK and dV.  An all-ones mask gives the bits of no mask, and two runs give
the same bits.  Without a mask the kernels give the bits recorded from the kernels before the mask
existed (tests/golden/attention_unmasked.json, written by tests/golden/make_attention_golden.py)."""
import hashlib
import json
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
H, DH = 3, 64
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "attention_unmasked.json")


def make_inputs(B, N, seed, dh=DH, heads=H):
  """q, k, v as column slices of one fused [B, N, 3 H dh] bf16 buffer, and dO [B, N, H dh]."""
  rng = np.random.default_rng(seed)
  qkv = torch.from_numpy(rng.standard_normal((B, N, 3 * heads * dh)).astype(np.float32) * 1.5).cuda().bfloat16()
  do = torch.from_numpy(rng.standard_normal((B, N, heads * dh)).astype(np.float32)).cuda().bfloat16()
  d = heads * dh
  return qkv[:, :, :d], qkv[:, :, d:2 * d], qkv[:, :, 2 * d:], do


def make_mask(B, N, kind, seed):
  rng = np.random.default_rng(seed)
  if kind == "suffix":                  # zero padding: the first len keys are attended
    lens = rng.integers(1, N + 1, size=B)
    lens[0] = N
    m = np.arange(N)[None, :] < lens[:, None]
  elif kind == "random":                # anywhere, including inside a key block
    m = rng.random((B, N)) < 0.6
    m[:, 0] = True
  elif kind == "empty":                 # batch 1 has no attended key
    m = rng.random((B, N)) < 0.5
    m[:, 0] = True
    m[1] = False
  else:
    raise ValueError(kind)
  return torch.from_numpy(m.astype(np.uint8)).cuda()


def reference(q, k, v, do, mask, heads=H):
  """fp64 O, lse and dQ, dK, dV; a query with no attended key gets O = 0 and lse = 0."""
  B, N, d = q.shape
  dh = d // heads
  split = lambda t: t.double().reshape(B, -1, heads, dh).transpose(1, 2).requires_grad_(True)
  q6, k6, v6 = split(q), split(k), split(v)
  keys = mask.bool()[:, None, None, :]
  s = (q6 @ k6.transpose(-1, -2)) / math.sqrt(dh)
  s = s.masked_fill(~keys, -math.inf)
  live = keys.any(-1, keepdim=True)
  m = torch.where(live, s.amax(-1, keepdim=True), 0.0).detach()
  e = torch.where(keys, torch.exp(s - m), 0.0)
  den = e.sum(-1, keepdim=True)
  o = (e @ v6) / torch.where(live, den, 1.0)
  lse = torch.where(live, torch.log(den) + m, 0.0).squeeze(-1)
  o = o.transpose(1, 2).reshape(B, N, d)
  o.backward(do.double())
  merge = lambda t: t.grad.transpose(1, 2).reshape(B, -1, d)
  return o.detach(), lse.detach(), merge(q6), merge(k6), merge(v6)


def run(q, k, v, do, mask, heads=H):
  from big_vision_b200 import ops
  kw = {} if mask is None else {"key_mask": mask}     # no keyword: the golden file's writer runs older ops
  o, lse = ops.attention_fwd(q, k, v, heads, **kw)
  dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, heads, **kw)
  torch.cuda.synchronize()
  return o, lse, dq, dk, dv


def _close(got, ref, name, rel=2.0 ** -7):
  """Element-wise within `rel` of the tensor's scale per batch item (bf16 outputs, DESIGN §4)."""
  got = got.double()
  for b in range(ref.shape[0]):
    scale = ref[b].abs().max().item()
    err = (got[b] - ref[b]).abs()
    assert torch.isfinite(got[b]).all(), name
    assert err.max().item() <= rel * scale + 1e-30, (name, b, err.max().item(), scale)


@pytest.mark.parametrize("N", [16, 64, 128, 577])
@pytest.mark.parametrize("kind", ["suffix", "random", "empty"])
def test_masked_attention_matches_fp64(N, kind):
  B = 4
  q, k, v, do = make_inputs(B, N, seed=N)
  mask = make_mask(B, N, kind, seed=N + 1)
  o, lse, dq, dk, dv = run(q, k, v, do, mask)
  ro, rlse, rdq, rdk, rdv = reference(q, k, v, do, mask)
  _close(o, ro, "o")
  assert torch.isfinite(lse).all()
  assert (lse.double() - rlse).abs().max().item() <= 1e-4 * max(rlse.abs().max().item(), 1.0)
  # the backward's dS = P (dP - delta) takes delta from the bf16 O: one more bf16 rounding than O
  _close(dq, rdq, "dq", rel=2.0 ** -6)
  _close(dk, rdk, "dk", rel=2.0 ** -6)
  _close(dv, rdv, "dv")
  masked = ~mask.bool()
  assert not dk[masked].any() and not dv[masked].any(), "a masked key has a nonzero gradient"
  if kind == "empty":
    assert not o[1].any() and not lse[1].any() and not dq[1].any()
    assert not dk[1].any() and not dv[1].any()


@pytest.mark.parametrize("N", [16, 197, 577])
def test_all_ones_mask_gives_the_bits_of_no_mask(N):
  q, k, v, do = make_inputs(3, N, seed=7 * N)
  ones = torch.ones((3, N), dtype=torch.uint8, device="cuda")
  for a, b in zip(run(q, k, v, do, ones), run(q, k, v, do, None)):
    assert torch.equal(a, b)


@pytest.mark.parametrize("kind", ["suffix", "random", "empty"])
def test_masked_attention_is_run_to_run_identical(kind):
  q, k, v, do = make_inputs(4, 128, seed=11)
  mask = make_mask(4, 128, kind, seed=12)
  for a, b in zip(run(q, k, v, do, mask), run(q, k, v, do, mask)):
    assert torch.equal(a, b)


def test_a_strided_mask_reads_its_own_rows():
  """A mask that is a column slice of a wider buffer (batch stride > Nk) gives the contiguous mask's bits."""
  q, k, v, do = make_inputs(4, 100, seed=13)
  mask = make_mask(4, 100, "random", seed=14)
  wide = torch.full((4, 160), 7, dtype=torch.uint8, device="cuda")
  wide[:, 30:130] = mask
  for a, b in zip(run(q, k, v, do, wide[:, 30:130]), run(q, k, v, do, mask)):
    assert torch.equal(a, b)


def digests(results):
  return {name: hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
          for name, t in zip(("o", "lse", "dq", "dk", "dv"), results)}


# (B, N, heads, dh): the shapes the golden file records, unmasked
GOLDEN_CASES = [(2, 16, 12, 64), (3, 197, 3, 64), (2, 577, 2, 64), (2, 130, 2, 72), (2, 257, 2, 104)]


def golden_results():
  out = {}
  for B, N, heads, dh in GOLDEN_CASES:
    q, k, v, do = make_inputs(B, N, seed=B * 1000 + N, dh=dh, heads=heads)
    out[f"{B}x{N}x{heads}x{dh}"] = digests(run(q, k, v, do, None, heads=heads))
  return out


def test_unmasked_kernels_give_the_recorded_bits():
  with open(GOLDEN) as f:
    want = json.load(f)["digests"]
  assert golden_results() == want
