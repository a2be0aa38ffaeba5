"""GPU: dropout in the ViT and text towers.  The kernels bit for bit against the numpy restatement of the mask
stream (tests/dropout_oracle.py), and the towers, a SigLIP step and the trainers' keys against float64
towers that apply the same masks."""
import math

import numpy as np
import pytest
import torch

import common
import dropout_oracle as D

pytestmark = pytest.mark.gpu


def _key(site=3, row0=0, rate=0.1, seed=123, step=9):
  from big_vision_b200 import lib as L
  return L.DropoutKey(seed=seed, step=step, site=site, row0=row0, rate=rate)


def _bits(t):
  return t.cpu().contiguous().view(torch.int16).numpy()


def _bf16(rows, cols, seed=0, ld=None):
  """bf16 [rows, cols] on the device, a view into [rows, ld] when ld > cols."""
  g = torch.Generator().manual_seed(seed)
  full = torch.randn((rows, ld or cols), generator=g).bfloat16().cuda()
  return full[:, :cols]


# ---- kernels --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols,ld,row0,rate", [
    (197, 768, None, 0, 0.1), (64, 3072, None, 394, 0.1), (50, 13, None, 7, 0.25), (33, 8, 24, 5, 0.5),
    (17, 24, 40, 0, 0.1), (9, 3, 5, 11, 0.9), (128, 64, None, 0, 0.0)])
def test_dropout_is_numpy_bit_for_bit(rows, cols, ld, row0, rate):
  from big_vision_b200 import ops
  x = _bf16(rows, cols, ld=ld)
  key = _key(row0=row0, rate=rate)
  y = ops.dropout(x, key)
  keep = D.key_mask(key, rate, rows, cols)
  want = D.dropout_bf16(x.float().cpu(), keep, rate)
  assert np.array_equal(_bits(y), _bits(want))
  # in place gives the same bits
  z = x.clone()
  ops.dropout(z, key, out=z)
  assert np.array_equal(_bits(z), _bits(want))
  # kept values are fp32(x) / (1 - rate) rounded once, dropped ones are +0
  xs = x.float().cpu().numpy()
  q = (xs / np.float32(D.keep_divisor(rate))).astype(np.float32)
  assert np.array_equal(y.float().cpu().numpy()[keep], torch.from_numpy(q[keep]).bfloat16().float().numpy())
  assert (_bits(y)[~keep] == 0).all()


@pytest.mark.parametrize("rows,cols,ld,row0", [(197, 768, None, 3), (31, 13, 21, 2), (40, 16, 32, 0)])
def test_dropout_add_is_numpy_bit_for_bit(rows, cols, ld, row0):
  from big_vision_b200 import ops
  rate = 0.1
  r, y = _bf16(rows, cols, seed=1, ld=ld), _bf16(rows, cols, seed=2, ld=ld)
  key = _key(row0=row0, rate=rate, site=77)
  out = ops.dropout_add(r, y, key)
  want = D.dropout_bf16(y.float().cpu(), D.key_mask(key, rate, rows, cols), rate, resid=r.float().cpu())
  assert np.array_equal(_bits(out), _bits(want))
  yy = y.clone()
  ops.dropout_add(r, yy, key, out=yy)
  assert np.array_equal(_bits(yy), _bits(want))


def test_column_sums_match_fp64_and_runs_repeat():
  from big_vision_b200 import ops
  rows, cols = 1000, 768
  x = _bf16(rows, cols, seed=3)
  key = _key(rate=0.1)
  s = torch.full((cols,), 0.5, dtype=torch.float32, device="cuda")
  y = ops.dropout(x, key, colsum_into=s)
  ref = 0.5 + y.double().sum(0)
  assert torch.allclose(s.double(), ref, rtol=1e-5, atol=1e-4)
  s2 = torch.full((cols,), 0.5, dtype=torch.float32, device="cuda")
  y2 = ops.dropout(x, key, colsum_into=s2)
  assert np.array_equal(_bits(y), _bits(y2)) and torch.equal(s, s2)


def test_realized_rate_at_b16_shapes():
  """The GELU site of one ViT-B/16 block at 64 images: [64 * 197, 3072]."""
  from big_vision_b200 import ops
  rows, cols, rate = 64 * 197, 3072, 0.1
  x = torch.ones((rows, cols), dtype=torch.bfloat16, device="cuda")
  y = ops.dropout(x, _key(rate=rate))
  n = rows * cols
  p = D.threshold(rate) / 65536
  dropped = int((y == 0).sum())
  assert abs(dropped / n - p) <= 5 * math.sqrt(p * (1 - p) / n)
  assert abs(p - rate) <= 2.0 ** -17 + 1e-8


# ---- towers ---------------------------------------------------------------------------------------------
def _relerr(a, b):
  a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
  return np.abs(a - b).max() / (np.abs(b).max() + 1e-30)


def _check_grads(grads, ref, rel=6e-2, floor=2e-3):
  gmax = max(float(np.abs(r).max()) for r in ref.values())
  bad = {}
  for k, g in grads.items():
    err = float(np.abs(g.astype(np.float64) - ref[k]).max())
    tol = rel * float(np.abs(ref[k]).max()) + floor * gmax
    if err > tol:
      bad[k] = (err, tol)
  assert not bad, sorted(bad.items(), key=lambda kv: -kv[1][0])[:8]


def _leaves(P):
  return {k: torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for k, v in P.numpy_tree().items()}


def _vit(pool, width=64, heads=1, depth=2, mlp=128, scan=False, rate=0.1):
  from big_vision_b200.models import vit
  return vit.Model(10, width=width, depth=depth, mlp_dim=mlp, num_heads=heads, patch_size=(16, 16),
                   pool_type=pool, scan=scan, dropout=rate, head_zeroinit=False)


def _vit_vs_oracle(model, P, image, key):
  """Forward and backward of the model at `key` against the float64 oracle with the same masks."""
  logits, saved = model.fwd(P, image, dropout=key)
  dlogits = torch.randn(logits.shape, generator=torch.Generator().manual_seed(5)).cuda()
  P.zero_grad()
  model.bwd(P, torch.nn.functional.pad(dlogits, (0, model.head.Cp - logits.shape[1])), saved)
  p64 = _leaves(P)
  cfg = dict(depth=model.depth, num_heads=model.num_heads, pool_type=model.pool_type, posemb=model.posemb,
             num_classes=10)
  ref = D.vit_forward(p64, image.cpu(), cfg, D.Masks(model.dropout, key.seed, key.step, key.sample0))
  ref.backward(dlogits.cpu().double())
  assert _relerr(logits.cpu().numpy(), ref.detach().numpy()) < 4e-2
  _check_grads(P.numpy_tree("g"), {k: v.grad.numpy() for k, v in p64.items()})
  return logits


@pytest.mark.parametrize("pool", ["gap", "tok", "map"])
def test_vit_tiny_against_the_oracle(pool):
  from big_vision_b200 import engine as E
  model = _vit(pool)
  P = model.init(0, (8, 64, 64, 3))
  image = torch.rand((8, 64, 64, 3), generator=torch.Generator().manual_seed(1)).mul(2).sub(1).cuda()
  key = E.DropoutKey(seed=3, step=11, sample0=16)
  y = _vit_vs_oracle(model, P, image, key)
  # the masks matter: without a key (evaluation) the output differs
  y0, _ = model.fwd(P, image)
  assert _relerr(y0.cpu().numpy(), y.cpu().numpy()) > 1e-3


def test_vit_b_width_against_the_oracle():
  from big_vision_b200 import engine as E
  model = _vit("gap", width=768, heads=12, depth=2, mlp=3072)
  P = model.init(0, (4, 64, 64, 3))
  image = torch.rand((4, 64, 64, 3), generator=torch.Generator().manual_seed(2)).mul(2).sub(1).cuda()
  _vit_vs_oracle(model, P, image, E.DropoutKey(seed=1, step=2))


@pytest.mark.parametrize("pool", ["gap", "tok"])
def test_scan_gives_the_unrolled_bits(pool):
  from big_vision_b200 import engine as E, utils
  from big_vision_b200.models import vit
  image = torch.rand((4, 64, 64, 3), generator=torch.Generator().manual_seed(3)).mul(2).sub(1).cuda()
  key = E.DropoutKey(seed=4, step=5)
  loop = _vit(pool)
  P = loop.init(0, (4, 64, 64, 3))
  flat = P.numpy_tree()
  scan = _vit(pool, scan=True)
  Ps = scan.init(1, (4, 64, 64, 3))
  stacked = vit.pyloop_to_scan(utils.recover_tree(list(flat), list(flat.values())))
  Ps.load_tree(dict(utils.tree_flatten_with_names(stacked)[0]))
  outs, grads = [], []
  for model, params in ((loop, P), (scan, Ps)):
    y, saved = model.fwd(params, image, dropout=key)
    params.zero_grad()
    model.bwd(params, torch.ones((4, model.head.Cp), device="cuda"), saved)
    outs.append(y)
    grads.append(params.numpy_tree("g"))
  assert torch.equal(outs[0], outs[1])
  # the gradients may differ by the order of accumulating reductions only
  g_scan = dict(utils.tree_flatten_with_names(vit.scan_to_pyloop(
      utils.recover_tree(list(grads[1]), list(grads[1].values()))))[0])
  for k, g in grads[0].items():
    assert np.abs(g - g_scan[k]).max() <= 1e-3 * np.abs(g).max() + 1e-7, k


def test_ranks_draw_the_global_batchs_masks():
  """Two ranks of 4 images each (sample0 = 0 and 4) compute the two halves of one rank's 8-image forward."""
  from big_vision_b200 import engine as E
  model = _vit("gap")
  P = model.init(0, (8, 64, 64, 3))
  image = torch.rand((8, 64, 64, 3), generator=torch.Generator().manual_seed(4)).mul(2).sub(1).cuda()
  whole, _ = model.fwd(P, image, frozen=True, dropout=E.DropoutKey(7, 3))
  for r in range(2):
    part, _ = model.fwd(P, image[4 * r:4 * r + 4].contiguous(), frozen=True, dropout=E.DropoutKey(7, 3, 4 * r))
    assert torch.equal(part, whole[4 * r:4 * r + 4])


def test_text_tower_against_the_oracle():
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.image_text import text_transformer
  model = text_transformer.Model(16, width=64, depth=2, mlp_dim=128, num_heads=1, vocab_size=64, dropout=0.1)
  P = model.init(0, common.TINY_TEXT_SHAPE)
  _, text = common.synthetic_batch(common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE, 64, seed=1)
  text = torch.from_numpy(text).cuda()
  key = E.DropoutKey(seed=2, step=6, tower=1)
  y, saved = model.fwd(P, text, dropout=key)
  dy = torch.randn(y.shape, generator=torch.Generator().manual_seed(5)).cuda()
  P.zero_grad()
  model.bwd(P, dy, saved)
  p64 = _leaves(P)
  ref = D.text_forward(p64, text.cpu(), dict(depth=2, num_heads=1, num_classes=16), D.Masks(0.1, 2, 6, 0, 1))
  ref.backward(dy.cpu().double())
  assert _relerr(y.cpu().numpy(), ref.detach().numpy()) < 4e-2
  _check_grads(P.numpy_tree("g"), {k: v.grad.numpy() for k, v in p64.items()})


def _siglip(img_rate, txt_rate, **image_kw):
  from big_vision_b200.models.proj.image_text import two_towers
  kw = dict(common.TINY, image=dict(common.TINY["image"], dropout=img_rate, **image_kw),
            text=dict(common.TINY["text"], dropout=txt_rate))
  model = two_towers.Model(**kw)
  P = model.init(0, common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE)
  image, text = common.synthetic_batch(common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE, 64, seed=2)
  return model, P, torch.from_numpy(image).cuda(), torch.from_numpy(text).cuda(), kw


def test_siglip_step_with_dropout_in_both_towers_against_the_oracle():
  from big_vision_b200 import engine as E
  from big_vision_b200.trainers.proj.image_text import siglip
  from oracle import bv_oracle as O
  model, P, image, text, kw = _siglip(0.1, 0.2)
  key = E.DropoutKey(seed=8, step=3)
  loss, _ = siglip.loss_and_grads(model, P, image, text, dropout=key)
  p64 = _leaves(P)
  zimg, ztxt = D.two_towers_forward(p64, image.cpu(), text.cpu(), common.oracle_cfg(kw), 0.1, 0.2, 8, 3)
  ref = O.siglip_loss(zimg, ztxt, torch.exp(p64["t"]), p64["b"])
  ref.backward()
  assert float(loss) == pytest.approx(float(ref.detach()), rel=5e-3)
  _check_grads(P.numpy_tree("g"), {k: v.grad.numpy() for k, v in p64.items()})


def test_siglit_frozen_image_tower_still_drops():
  from big_vision_b200 import engine as E
  model, P, image, text, _ = _siglip(0.1, 0.0)
  frozen = frozenset(k for k in P.offsets if k.startswith("img/"))
  key = E.DropoutKey(seed=8, step=3)
  z_frozen, _, saved = model.fwd(P, image, text, frozen=frozen, dropout=key)
  z_trained, _, _ = model.fwd(P, image, text, dropout=key)
  z_eval, _, _ = model.fwd(P, image, text, frozen=frozen)
  assert saved["img"] is None
  assert torch.equal(z_frozen, z_trained) and not torch.equal(z_frozen, z_eval)


def test_train_step_masks_follow_the_step_count():
  from big_vision_b200 import train
  from big_vision_b200.trainers.proj.image_text.siglip import Dist
  model = _vit("gap")
  P = model.init(0, (8, 64, 64, 3))
  image = torch.rand((8, 64, 64, 3), generator=torch.Generator().manual_seed(6)).mul(2).sub(1).cuda()
  labels = torch.nn.functional.one_hot(torch.arange(8) % 10, 10).float().cuda()
  d = Dist()

  def step(count):
    key = train.dropout_key(0, {"count": count}, d, 8)
    loss, logits = train.loss_and_grads(model, P, image, labels, dropout=key)
    return float(loss), logits.clone()

  a, b, c = step(4), step(4), step(5)
  assert a[0] == b[0] and torch.equal(a[1], b[1])
  assert not torch.equal(a[1], c[1])


def test_gsam_passes_see_the_same_masks(monkeypatch):
  """Both GSAM passes run their forward with one key, so they drop the same elements."""
  from big_vision_b200 import engine as E
  from big_vision_b200.trainers.proj.gsam import gsam as G
  model = _vit("gap")
  P = model.init(0, (8, 64, 64, 3))
  image = torch.rand((8, 64, 64, 3), generator=torch.Generator().manual_seed(7)).mul(2).sub(1).cuda()
  labels = torch.nn.functional.one_hot(torch.arange(8) % 10, 10).float().cuda()
  seen, fwd = [], model.fwd

  def spy(*a, **kw):
    seen.append(kw.get("dropout"))
    return fwd(*a, **kw)
  monkeypatch.setattr(model, "fwd", spy)
  key = E.DropoutKey(seed=1, step=2)
  G.gsam_gradient(model, P, image, labels, rho_max=0.05, rho_min=0.05, alpha=0.1, lr=1e-3, lr_max=1e-3,
                  lr_min=1e-3, dropout=key)
  assert seen == [key, key]
