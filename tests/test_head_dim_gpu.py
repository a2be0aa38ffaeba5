"""GPU parity of the attention kernels at head dims 72, 80 and 96 (So400m, H, g-opt) against the fp64
reference attention, in place in fused QKV buffers, bit for bit reproducible, and the So400m geometry through
whole models against the fp64 oracle.
Tolerances as in test_attention_gpu.py / test_model_gpu.py / test_precision_gpu.py."""
import json
import math

import numpy as np
import pytest
import torch

import common
from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu

HEAD_DIMS = [72, 80, 96]
# So400m/14 @224 and @384, the MAP head's single query, the text tower, then ragged shapes
SHAPES = [(2, 16, 256, 256), (1, 16, 729, 729), (3, 16, 1, 256), (2, 16, 64, 64), (2, 3, 197, 197),
          (1, 2, 300, 700), (2, 2, 130, 7)]


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
  return (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, Nq, d), torch.logsumexp(s, -1)


def _qkv(B, N, d, seed):
  g = torch.Generator().manual_seed(seed)
  qkv = _bf(torch.randn(B, N, 3 * d, generator=g))
  qkv[:, ::37, 0:d] *= 4.0     # a few large scores per row
  return qkv, g


@pytest.mark.parametrize("dh", HEAD_DIMS)
@pytest.mark.parametrize("B,H,Nq,Nk", SHAPES)
def test_forward_matches_fp64(ops, dh, B, H, Nq, Nk):
  d = H * dh
  qkv, _ = _qkv(B, max(Nq, Nk), d, B * 1000 + Nq + dh)
  o_ref, lse_ref = _ref_attention(qkv[:, :Nq, 0:d].double(), qkv[:, :Nk, d:2 * d].double(),
                                  qkv[:, :Nk, 2 * d:].double(), H)
  c = qkv.cuda()
  o, lse = ops.attention_fwd(c[:, :Nq, 0:d], c[:, :Nk, d:2 * d], c[:, :Nk, 2 * d:], H)
  torch.cuda.synchronize()
  _close(o, o_ref, 2 ** -6)
  _close(lse, lse_ref, 1e-5)


@pytest.mark.parametrize("dh", HEAD_DIMS)
@pytest.mark.parametrize("B,H,Nq,Nk", SHAPES)
def test_backward_matches_fp64(ops, dh, B, H, Nq, Nk):
  d = H * dh
  qkv, g = _qkv(B, max(Nq, Nk), d, B * 1000 + Nq + dh)
  do = _bf(torch.randn(B, Nq, d, generator=g))
  qr = qkv[:, :Nq, 0:d].double().requires_grad_(True)
  kr = qkv[:, :Nk, d:2 * d].double().requires_grad_(True)
  vr = qkv[:, :Nk, 2 * d:].double().requires_grad_(True)
  o_ref, _ = _ref_attention(qr, kr, vr, H)
  o_ref.backward(do.double())
  c = qkv.cuda()
  q, k, v = c[:, :Nq, 0:d], c[:, :Nk, d:2 * d], c[:, :Nk, 2 * d:]
  o, lse = ops.attention_fwd(q, k, v, H)
  cs = torch.ones(3, d, device="cuda")
  dq, dk, dv = ops.attention_bwd(do.cuda(), q, k, v, o, lse, H, dq_colsum=cs[0], dk_colsum=cs[1], dv_colsum=cs[2])
  torch.cuda.synchronize()
  _close(dq, qr.grad, 2 ** -5)
  _close(dk, kr.grad, 2 ** -5)
  _close(dv, vr.grad, 2 ** -5)
  for i, t in enumerate((dq, dk, dv)):      # fused bias gradients: column sums over the valid rows
    ref = 1 + t.double().sum((0, 1))
    assert (cs[i].double() - ref).abs().max().item() <= 1e-4 * (ref.abs().max().item() + 1)


@pytest.mark.parametrize("dh", HEAD_DIMS)
def test_in_place_in_fused_buffers(ops, dh):
  """q/k/v and dq/dk/dv as column views of [B, N, 3*H*dh + 8] buffers.  The 8 columns past the views
  hold NaN in the input (a tile that read past the last head's dh columns would turn S into NaN) and a
  sentinel in the gradient buffer; rows past N and the sentinel columns must come back untouched."""
  B, H, N = 2, 3, 130
  d = H * dh
  qkv, g = _qkv(B, N + 5, d, 7 + dh)
  buf = torch.cat([qkv, torch.full((B, N + 5, 8), float("nan"), dtype=torch.bfloat16)], 2).cuda()
  do = _bf(torch.randn(B, N, d, generator=g))
  qr = qkv[:, :N, 0:d].double().requires_grad_(True)
  kr = qkv[:, :N, d:2 * d].double().requires_grad_(True)
  vr = qkv[:, :N, 2 * d:].double().requires_grad_(True)
  o_ref, lse_ref = _ref_attention(qr, kr, vr, H)
  o_ref.backward(do.double())
  q, k, v = buf[:, :N, 0:d], buf[:, :N, d:2 * d], buf[:, :N, 2 * d:3 * d]
  o, lse = ops.attention_fwd(q, k, v, H)
  sentinel = 1234.0
  dbuf = torch.full((B, N + 5, 3 * d + 8), sentinel, dtype=torch.bfloat16, device="cuda")
  dq, dk, dv = ops.attention_bwd(do.cuda(), q, k, v, o, lse, H, dq=dbuf[:, :N, 0:d], dk=dbuf[:, :N, d:2 * d],
                                 dv=dbuf[:, :N, 2 * d:3 * d])
  torch.cuda.synchronize()
  _close(o, o_ref, 2 ** -6)
  _close(lse, lse_ref, 1e-5)
  _close(dbuf[:, :N, 0:d], qr.grad, 2 ** -5)
  _close(dbuf[:, :N, d:2 * d], kr.grad, 2 ** -5)
  _close(dbuf[:, :N, 2 * d:3 * d], vr.grad, 2 ** -5)
  assert bool((dbuf[:, N:, :] == sentinel).all())
  assert bool((dbuf[:, :, 3 * d:] == sentinel).all())


def test_head_dim_72_is_bitwise_reproducible(ops):
  B, H, N, dh = 2, 16, 256, 72
  d = H * dh
  g = torch.Generator().manual_seed(11)
  c = _bf(torch.randn(B, N, 3 * d, generator=g)).cuda()
  do = _bf(torch.randn(B, N, d, generator=g)).cuda()
  q, k, v = c[:, :, 0:d], c[:, :, d:2 * d], c[:, :, 2 * d:]
  o1, l1 = ops.attention_fwd(q, k, v, H)
  o2, l2 = ops.attention_fwd(q, k, v, H)
  assert torch.equal(o1, o2) and torch.equal(l1, l2)
  r = ops.attention_bwd(do, q, k, v, o1, l1, H)
  t = ops.attention_bwd(do, q, k, v, o1, l1, H)
  for a, b in zip(t, r):
    assert torch.equal(a, b)


# ---- whole models --------------------------------------------------------------------------------
# So400m geometry scaled down: head dim 72, mlp not 4x width (K tail of 24 past a multiple of 64),
# patch 14
TINY_SO400M = dict(
    image=dict(width=144, depth=2, mlp_dim=536, num_heads=2, patch_size=(14, 14), pool_type="map"),
    text=dict(width=144, depth=2, mlp_dim=536, num_heads=2, vocab_size=64),
    out_dim=(None, 144), temperature_init=10.0, bias_init=-10.0)


def _scan_to_pyloop(flat):
  from big_vision_b200 import utils as u
  from big_vision_b200.models import vit
  nested = u.recover_tree(list(flat.keys()), list(flat.values()))
  nested["img"] = vit.scan_to_pyloop(nested["img"], "Transformer")
  nested["txt"] = vit.scan_to_pyloop(nested["txt"], "Encoder_0")
  return dict(u.tree_flatten_with_names(nested)[0])


@pytest.mark.parametrize("scan", [False, True])
def test_tiny_so400m_two_towers_match_oracle(scan):
  from big_vision_b200.models.proj.image_text import two_towers
  from big_vision_b200.trainers.proj.image_text import siglip
  kw = dict(TINY_SO400M, image=dict(TINY_SO400M["image"], scan=scan), text=dict(TINY_SO400M["text"], scan=scan))
  image_shape, text_shape = (8, 56, 56, 3), (8, 16)
  model = two_towers.Model(**kw)
  P = model.init(5, image_shape, text_shape, device="cuda")
  tree = P.numpy_tree("f")
  if scan:
    tree = _scan_to_pyloop(tree)
  image, text = common.synthetic_batch(image_shape, text_shape, 64, seed=6)
  loss, _ = siglip.loss_and_grads(model, P, torch.from_numpy(image).cuda(), torch.from_numpy(text).cuda())
  p64 = O.to_f64_tree(tree, requires_grad=True)
  zi, zt, ex = O.two_towers_forward(p64, torch.from_numpy(image), torch.from_numpy(text),
                                    common.oracle_cfg(TINY_SO400M), "float32")
  ref = O.siglip_loss(zi, zt, ex["t"], ex["b"])
  ref = ref[0] if isinstance(ref, tuple) else ref
  ref.backward()
  assert float(loss) == pytest.approx(float(ref), rel=5e-3)
  grads = P.numpy_tree("g")
  if scan:
    grads = _scan_to_pyloop(grads)
  assert set(grads) == set(p64)
  gmax = max(float(v.grad.abs().max()) for v in p64.values() if v.grad is not None)
  bad = {}
  for k, g in grads.items():
    r = p64[k].grad.numpy() if p64[k].grad is not None else np.zeros_like(g)
    err = float(np.abs(g.astype(np.float64) - r).max())
    tol = 6e-2 * float(np.abs(r).max()) + 3e-3 * gmax
    if err > tol:
      bad[k] = (err, tol)
  assert not bad, sorted(bad.items(), key=lambda kv: -kv[1][0])[:8]


def _rel(got, ref):
  got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
  return float(np.abs(got - ref).max() / (np.abs(ref).max() + 1e-30))


def _rel_l2(got, ref):
  got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
  return float(np.linalg.norm(got - ref) / (np.linalg.norm(ref) + 1e-30))


def test_so400m14_real_width_image_tower_precision():
  """The So400m/14 image tower at its real width (1152, 16 heads of 72, mlp 4304, 256 tokens, MAP head,
  a classifier head for a loss), depth cut to 2 so the fp64 oracle stays short; bounds of
  test_precision_gpu.py."""
  from big_vision_b200 import train
  from big_vision_b200.models import vit
  n, C, depth = 4, 128, 2
  shape = (n, 224, 224, 3)
  model = vit.Model(C, variant="So400m/14", depth=depth, pool_type="map")
  P = model.init(0, shape, device="cuda")
  rng = np.random.default_rng(1)
  tree = P.numpy_tree("f")
  for k, v in tree.items():                      # zero-initialised head: small values instead
    if not np.any(v):
      tree[k] = (rng.standard_normal(v.shape) * 0.02).astype(np.float32)
  P.load_tree(tree)
  image = rng.uniform(-1, 1, size=shape).astype(np.float32)
  labels = np.eye(C, dtype=np.float32)[rng.integers(0, C, size=n)]
  loss, logits = train.loss_and_grads(model, P, torch.from_numpy(image).cuda(), torch.from_numpy(labels).cuda(),
                                      "sigmoid_xent")
  cfg = dict(depth=depth, num_heads=16, pool_type="map", posemb="learn", rep_size=False, num_classes=C)
  with torch.no_grad():
    ref16 = O.vit_forward(O.to_f64_tree(tree), torch.from_numpy(image), cfg, "bfloat16").numpy()
  p64 = O.to_f64_tree(tree, requires_grad=True)
  ref64 = O.vit_forward(p64, torch.from_numpy(image), cfg, "float32")
  ref_loss = O.sigmoid_xent(ref64, torch.from_numpy(labels).double())
  ref_loss.backward()
  got = logits.double().cpu().numpy()
  res = {"logits_vs_bf16_oracle_max": _rel(got, ref16), "logits_vs_fp64_oracle_max": _rel(got, ref64.detach().numpy()),
         "logits_vs_fp64_oracle_l2": _rel_l2(got, ref64.detach().numpy()),
         "loss_rel": abs(float(loss) - float(ref_loss)) / abs(float(ref_loss))}
  grads = P.numpy_tree("g")
  worst, l2s = ("", 0.0), []
  gmax = max(float(v.grad.abs().max()) for v in p64.values() if v.grad is not None)
  for k, g in grads.items():
    ref = p64[k].grad.numpy() if p64[k].grad is not None else np.zeros_like(g)
    e = float(np.abs(g - ref).max() / (np.abs(ref).max() + 1e-3 * gmax))
    l2s.append(_rel_l2(g, ref) if np.abs(ref).max() > 1e-3 * gmax else 0.0)
    if e > worst[1]:
      worst = (k, e)
  res.update(grad_worst_tensor=worst[0], grad_worst_rel_max=worst[1], grad_median_rel_l2=float(np.median(l2s)),
             grad_max_rel_l2=float(np.max(l2s)))
  print(json.dumps({f"so400m14_depth{depth}_map_n{n}": res}))
  assert res["logits_vs_bf16_oracle_max"] <= 1.5e-2, res
  assert res["logits_vs_fp64_oracle_max"] <= 3e-2 and res["loss_rel"] <= 2e-3, res
  assert res["grad_worst_rel_max"] <= 1.2e-1 and res["grad_median_rel_l2"] <= 3e-2, res
