"""GPU: attention at head dim 104 (ViT-G) against fp64 attention, in place and bit-reproducible; the strided
xent kernels and the scalar mixup path; tiny classifiers with padded heads (C % 8 != 0) against the fp64
oracle through loss, optimizer steps, evaluation and checkpoints; and the real-width ViT-G/14 with the
29,593-class head against the oracle at the precision bounds of the So400m tower test."""
import json
import os

import numpy as np
import pytest
import torch

import test_classifier_gpu as cls_t
import test_head_dim_gpu as hd
from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
  from big_vision_b200 import lib, ops as _ops
  assert lib.load().bv_device_supported() == 1
  return _ops


# ---- attention at head dim 104 -------------------------------------------------------------------
@pytest.mark.parametrize("B,H,Nq,Nk", hd.SHAPES)
def test_attention_104_forward_matches_fp64(ops, B, H, Nq, Nk):
  hd.test_forward_matches_fp64(ops, 104, B, H, Nq, Nk)


@pytest.mark.parametrize("B,H,Nq,Nk", hd.SHAPES)
def test_attention_104_backward_matches_fp64(ops, B, H, Nq, Nk):
  hd.test_backward_matches_fp64(ops, 104, B, H, Nq, Nk)


def test_attention_104_in_place_in_fused_buffers(ops):
  hd.test_in_place_in_fused_buffers(ops, 104)


def test_attention_104_is_bitwise_reproducible(ops):
  B, H, N, dh = 2, 16, 256, 104
  d = H * dh
  g = torch.Generator().manual_seed(13)
  c = hd._bf(torch.randn(B, N, 3 * d, generator=g)).cuda()
  do = hd._bf(torch.randn(B, N, d, generator=g)).cuda()
  q, k, v = c[:, :, 0:d], c[:, :, d:2 * d], c[:, :, 2 * d:]
  o1, l1 = ops.attention_fwd(q, k, v, H)
  o2, l2 = ops.attention_fwd(q, k, v, H)
  assert torch.equal(o1, o2) and torch.equal(l1, l2)
  for a, b in zip(ops.attention_bwd(do, q, k, v, o1, l1, H), ops.attention_bwd(do, q, k, v, o1, l1, H)):
    assert torch.equal(a, b)


# ---- losses and mixup -----------------------------------------------------------------------------
def _logits_labels(n, C, seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(n, C, generator=g) * 3
  y = torch.nn.functional.one_hot(torch.randint(0, C, (n,), generator=g), C).float()
  return x, 0.9 * y + 0.1 * y.roll(1, 0)


@pytest.mark.parametrize("name", ["sigmoid_xent", "softmax_xent"])
@pytest.mark.parametrize("C", [21843, 37])
def test_xent_ld_ignores_padding_and_zeroes_dlogits_padding(ops, name, C):
  Cp = (C + 7) // 8 * 8
  x, y = (t.cuda() for t in _logits_labels(16, C, 4))
  fn = getattr(ops, name)
  loss_ref = torch.zeros(1, device="cuda")
  dl_ref = fn(x, y, loss_ref)
  xp = torch.full((16, Cp), float("nan"), device="cuda")
  xp[:, :C] = x
  loss = torch.zeros(1, device="cuda")
  dl = fn(xp[:, :C], y, loss, dlogits_cols=Cp)
  torch.cuda.synchronize()
  assert dl.shape == (16, Cp)
  assert torch.equal(loss, loss_ref) and torch.equal(dl[:, :C], dl_ref)
  assert bool((dl[:, C:] == 0).all())


@pytest.mark.parametrize("C,offset", [(21843, 0), (21843, 1), (1000, 1), (37, 0)])
def test_mixup_scalar_path_is_bit_exact(ops, C, offset):
  """Rows of any length and 4-byte (not 16-byte) aligned buffers: the scalar path, same fp32 expression."""
  rng = np.random.default_rng(C + offset)
  x = rng.standard_normal((8, C)).astype(np.float32)
  a = np.float32(0.7312)
  buf = torch.zeros(8 * C + offset, device="cuda")
  src = buf[offset:].view(8, C)
  src.copy_(torch.from_numpy(x))
  got = ops.mixup(src, float(a)).cpu().numpy()
  want = a * x + (np.float32(1) - a) * np.roll(x, 1, axis=0)
  assert np.array_equal(got, want)


# ---- tiny classifiers with padded heads against the oracle ------------------------------------------
TINY_VIT = dict(width=208, depth=2, mlp_dim=416, num_heads=2, patch_size=(16, 16), pool_type="map")


def _tiny(kind, C):
  from big_vision_b200.models import mlp_mixer, vit
  if kind == "vit":
    model = vit.Model(C, **TINY_VIT)
    cfg = dict(depth=2, num_heads=2, pool_type="map", posemb="learn", rep_size=False, num_classes=C)
    return model, (lambda p, img, mm: O.vit_forward(p, img, cfg, mm))
  model = mlp_mixer.Model(C, patch_size=(16, 16), num_blocks=2, hidden_dim=64, tokens_mlp_dim=32,
                          channels_mlp_dim=128)
  cfg = dict(num_blocks=2, num_classes=C)
  return model, (lambda p, img, mm: O.mixer_forward(p, img, cfg, mm))


@pytest.mark.parametrize("kind,C,loss", [("vit", 29593, "sigmoid_xent"), ("vit", 21843, "softmax_xent"),
                                         ("mixer", 21843, "sigmoid_xent"), ("mixer", 29593, "softmax_xent"),
                                         ("vit", 37, "softmax_xent")])
def test_padded_head_classifier_matches_oracle(kind, C, loss):
  model, fwd = _tiny(kind, C)
  cls_t._check(model, fwd, (4, 64, 48, 3), loss, C)


def test_padded_head_with_mixup_matches_oracle(ops):
  """Mixed images and labels (the [n, 21843] labels take the scalar mixup path) into the padded head."""
  from big_vision_b200 import train
  C, shape = 21843, (4, 64, 48, 3)
  model, fwd = _tiny("vit", C)
  P = model.init(0, shape, device="cuda")
  tree = cls_t._randomize_zero_inits(P.numpy_tree("f"), 1)
  P.load_tree(tree)
  rng = np.random.default_rng(2)
  image = rng.uniform(-1, 1, size=shape).astype(np.float32)
  labels = np.eye(C, dtype=np.float32)[rng.integers(0, C, size=4)]
  a = 0.8125
  mix = lambda t: ops.mixup(torch.from_numpy(t).cuda(), a)   # noqa: E731
  img_m, lab_m = mix(image), mix(labels)
  loss, logits = train.loss_and_grads(model, P, img_m, lab_m, "sigmoid_xent")
  p64 = O.to_f64_tree(tree, requires_grad=True)
  ref_logits = fwd(p64, img_m.cpu(), "float32")
  ref = O.sigmoid_xent(ref_logits, lab_m.cpu().double())
  ref.backward()
  scale = float(ref_logits.abs().max())
  assert float((logits.double().cpu() - ref_logits.detach()).abs().max()) <= 6e-2 * scale
  assert float(loss) == pytest.approx(float(ref), rel=2e-2)
  g = P.numpy_tree("g")["head/kernel"]
  r = p64["head/kernel"].grad.numpy()
  assert float(np.abs(g - r).max()) <= 6e-2 * float(np.abs(r).max()) + 1e-12


def _padding(P):
  k, b = P.f("head/kernel_pad"), P.f("head/bias_pad")
  C = P.tree("f")["head/bias"].shape[0]
  return torch.cat([k[:, C:].reshape(-1), b[C:], P.g("head/kernel_pad")[:, C:].reshape(-1), P.g("head/bias_pad")[C:],
                    P.h("head/kernel_pad")[:, C:].float().reshape(-1), P.h("head/bias_pad")[C:].float()])


@pytest.mark.parametrize("optax_name", ["scale_by_adam", "big_vision.scale_by_adafactor"])
@pytest.mark.parametrize("kind,C", [("vit", 29593), ("mixer", 21843)])
def test_padding_stays_zero_and_measurements_match_the_reference_tree(optax_name, kind, C, tmp_path):
  from big_vision_b200 import optax as bv_optax, train, utils as u
  from big_vision_b200.evaluators import classification
  model, fwd = _tiny(kind, C)
  n, shape = 8, (8, 64, 48, 3)
  P = model.init(0, shape, device="cuda")
  P.load_tree(cls_t._randomize_zero_inits(P.numpy_tree("f"), 1))
  config = dict(optax_name=optax_name, lr=1e-2, wd=1e-2, grad_clip_norm=1.0, loss="softmax_xent",
                wd_mults=[(".*head/kernel", 100.0), (".*/kernel", 1.0)],
                schedule=dict(decay_type="cosine", warmup_steps=0))
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=100, batch_size=n, data_size=1000))
  state = {"params": P, "opt": tx.init(P)}
  fn = train.make_update_fn(model, tx, config)
  rng = np.random.default_rng(3)
  image = rng.uniform(-1, 1, shape).astype(np.float32)
  labels = np.eye(C, dtype=np.float32)[rng.integers(0, C, n)]
  batch = {"image": torch.from_numpy(image).cuda(), "labels": torch.from_numpy(labels).cuda()}
  for step in range(4):
    before = P.numpy_tree("f")
    state, m = fn(state, None, batch)
    torch.cuda.synchronize()
    assert float(_padding(P).abs().max()) == 0.0, step
    after, grads = P.numpy_tree("f"), P.numpy_tree("g")
    assert set(after) == set(before) and after["head/kernel"].shape == (model.head.rep, C)
    # l2 measurements over the reference-shaped tree (the padding contributes nothing)
    l2 = lambda tree: np.sqrt(sum(float(np.sum(np.asarray(v, np.float64) ** 2)) for v in tree.values()))  # noqa: E731
    assert float(m["l2_grads"]) == pytest.approx(l2(grads), rel=1e-4)
    assert float(m["l2_params"]) == pytest.approx(l2(after), rel=1e-4)
    assert float(m["l2_updates"]) == pytest.approx(l2({k: after[k] - before[k] for k in after}), rel=2e-3)
  # gradients of this step against the fp64 oracle on the reference tree
  p64 = O.to_f64_tree(before, requires_grad=True)
  ref = O.softmax_xent(fwd(p64, torch.from_numpy(image), "float32"), torch.from_numpy(labels).double())
  ref.backward()
  assert float(m["training_loss"]) == pytest.approx(float(ref), rel=2e-2)
  assert float(m["l2_grads"]) == pytest.approx(
      np.sqrt(sum(float((v.grad ** 2).sum()) for v in p64.values() if v.grad is not None)), rel=3e-2)
  # top-1 counts on the strided logits
  logits, _ = model.fwd(P, batch["image"])
  assert logits.shape == (n, C) and logits.stride(0) == (C + 7) // 8 * 8
  nc, ns, idx = classification.top1_counts(logits, batch["labels"])
  enc, ens, eidx = O.top1_counts(logits.double().cpu().numpy(), labels, None)
  assert (nc, ns) == (float(enc), float(ens)) and np.array_equal(idx.cpu().numpy(), np.asarray(eidx))
  # npz save / load round trip is bit-exact and leaves the padding zero
  path = os.path.join(tmp_path, "ckpt.npz")
  flat = P.numpy_tree("f")
  u.save_checkpoint_np(u.recover_tree(list(flat.keys()), list(flat.values())), path)
  P2 = model.init(7, shape, device="cuda")
  P2.load_tree(dict(u.tree_flatten_with_names(u.load_params(path))[0]))
  for k, v in P2.numpy_tree("f").items():
    assert np.array_equal(v, flat[k]), k
  assert torch.equal(P2.flat, P.flat)


def test_vit_G14_real_width_with_jft_head_precision():
  """ViT-G/14 at its real width (1664, 16 heads of 104, mlp 8192, 256 tokens, MAP head, the 29,593-class
  head), depth cut to 2 so the fp64 oracle stays short; bounds of the So400m/14 tower test."""
  from big_vision_b200 import train
  from big_vision_b200.models import vit
  n, C, depth = 4, 29_593, 2
  shape = (n, 224, 224, 3)
  model = vit.Model(C, variant="G/14", depth=depth, pool_type="map")
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
  res = {"logits_vs_bf16_oracle_max": hd._rel(got, ref16), "logits_vs_fp64_oracle_max": hd._rel(got, ref64.detach().numpy()),
         "loss_rel": abs(float(loss) - float(ref_loss)) / abs(float(ref_loss))}
  grads = P.numpy_tree("g")
  worst, l2s = ("", 0.0), []
  gmax = max(float(v.grad.abs().max()) for v in p64.values() if v.grad is not None)
  for k, g in grads.items():
    ref = p64[k].grad.numpy() if p64[k].grad is not None else np.zeros_like(g)
    e = float(np.abs(g - ref).max() / (np.abs(ref).max() + 1e-3 * gmax))
    l2s.append(hd._rel_l2(g, ref) if np.abs(ref).max() > 1e-3 * gmax else 0.0)
    if e > worst[1]:
      worst = (k, e)
  res.update(grad_worst_tensor=worst[0], grad_worst_rel_max=worst[1], grad_median_rel_l2=float(np.median(l2s)))
  print(json.dumps({f"vit_G14_depth{depth}_map_jft_n{n}": res}))
  assert res["logits_vs_bf16_oracle_max"] <= 1.5e-2, res
  assert res["logits_vs_fp64_oracle_max"] <= 3e-2 and res["loss_rel"] <= 2e-3, res
  assert res["grad_worst_rel_max"] <= 1.2e-1 and res["grad_median_rel_l2"] <= 3e-2, res
