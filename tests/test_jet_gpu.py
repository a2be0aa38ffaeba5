"""GPU: the Jet kernels of include/bv_b200_jet.h against numpy and float64 -- bit for bit where the operation
is exact (layout, noise, gathers), element by element within rounding-derived bounds where it is not --, the
tiny Jet model against the float64 oracle (bits, z and every gradient), invertibility, checkpoint loading of
other masks, the trainer and a 2-rank NCCL step."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import jet_oracle as JO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24                      # unit roundoff of fp32
TINY = dict(depth=5, block_depth=1, emb_dim=64, num_heads=1, ps=4)     # kinds c, c, s, c, c
TINY_SHAPE = (4, 16, 16, 3)
NOISE = np.float32(1 / 127.5)


def _np_patchify(image, ps):
  n, H, W, C = image.shape
  return image.reshape(n, H // ps, ps, W // ps, ps, C).transpose(0, 1, 3, 2, 4, 5).reshape(n, -1, ps * ps * C)


def _np_noise(seed, counter, offset, count):
  gen = np.random.Generator(np.random.Philox(key=seed, counter=[0, counter, 0, 0]))
  return gen.random(offset + count, dtype=np.float32)[offset:]


def _image(shape, seed=0):
  return np.random.default_rng(seed).uniform(-1, 1, shape).astype(np.float32)


# ---- layout and noise ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,hw,offset", [(1, (64, 64), 0), (3, (16, 24), 0), (3, (16, 24), 2 * 3 * 16 * 24 * 3),
                                         (5, (8, 8), 13)])
def test_dequantize_patchify_is_numpy_bit_for_bit(n, hw, offset):
  from big_vision_b200 import ops
  image = _image((n,) + hw + (3,))
  seed, counter = 1234, 17
  u = _np_noise(seed, counter, offset, image.size).reshape(image.shape)
  want = _np_patchify(image + u * NOISE, 4)           # two float32 roundings, as the reference
  got = ops.jet_dequantize_patchify(torch.from_numpy(image).cuda(), 4, seed, counter, offset).cpu().numpy()
  np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))


def test_noise_of_a_global_batch_does_not_depend_on_the_rank_count():
  from big_vision_b200 import ops
  image = torch.from_numpy(_image((6, 16, 16, 3))).cuda()
  whole = ops.jet_dequantize_patchify(image, 4, 9, 3, 0)
  per = image[0].numel() * 3
  halves = [ops.jet_dequantize_patchify(image[3 * r:3 * r + 3].contiguous(), 4, 9, 3, r * per) for r in range(2)]
  assert torch.equal(whole, torch.cat(halves))
  assert not torch.equal(whole, ops.jet_dequantize_patchify(image, 4, 9, 4, 0))     # the counter matters


def test_unpatchify_and_plain_patchify_are_exact():
  from big_vision_b200 import ops
  image = _image((3, 16, 8, 3))
  plain = ops.jet_dequantize_patchify(torch.from_numpy(image).cuda(), 4, noise_scale=0.0)
  np.testing.assert_array_equal(plain.cpu().numpy(), _np_patchify(image, 4))
  back = ops.jet_unpatchify(plain, image.shape, 4)
  np.testing.assert_array_equal(back.cpu().numpy(), image)


def test_split_and_merge_grad_are_exact():
  from big_vision_b200 import ops
  n, T, c = 3, 16, 24
  D = 2 * T * c
  x = torch.randn(n, T, 2 * c, device="cuda") * 3
  idx = torch.randperm(D, device="cuda").int()
  x1 = ops.jet_split(x, idx, T, c)
  assert x1.shape == (n * T, c) and x1.dtype == torch.bfloat16
  assert torch.equal(x1.view(n, -1), x.view(n, D)[:, idx[:D // 2].long()].bfloat16())
  dy, dx1 = torch.randn(n, T, 2 * c, device="cuda"), torch.randn(n * T, c, device="cuda")
  want = dy.clone().view(n, D)
  sel = idx[:D // 2].long()
  want[:, sel] = dy.view(n, D)[:, sel] + dx1.view(n, -1)
  dx = torch.full_like(dy, float("nan")).view(n, D)
  dx[:, idx[D // 2:].long()] = dy.view(n, D)[:, idx[D // 2:].long()]
  ops.jet_merge_grad(dy, dx1, idx, T, c, dx=dx)
  assert torch.equal(dx, want)
  ops.jet_merge_grad(dy, dx1, idx, T, c, dx=dy)                                   # in place
  assert torch.equal(dy.view(n, D), want)


# ---- coupling kernels -------------------------------------------------------------------------------------
def _coupling_case(n=3, T=16, c=24, raw_scale=4.0, seed=0):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(n, T, 2 * c, generator=g) * 2
  br = torch.randn(n * T, 2 * c, generator=g)
  br[:, c:] *= raw_scale
  idx = torch.randperm(2 * T * c, generator=g).int()
  return x, br, idx


def _ref_affine(x, br, idx, T, c):
  n = x.shape[0]
  D = 2 * T * c
  xd = x.double().view(n, D)
  x2 = xd[:, idx[D // 2:].long()].view(n * T, c)
  bias, raw = br[:, :c].double(), br[:, c:].double()
  return x2, bias, raw, torch.sigmoid(raw) * 2


@pytest.mark.parametrize("inverse", [False, True])
def test_coupling_fwd_elementwise(inverse):
  from big_vision_b200 import ops
  n, T, c = 3, 16, 24
  D = 2 * T * c
  x, br, idx = _coupling_case(n, T, c)
  x2, bias, raw, s = _ref_affine(x, br, idx, T, c)
  ld0 = torch.randn(n)
  logdet = ld0.cuda()
  y = ops.jet_coupling_fwd(x.cuda(), idx.cuda(), br.cuda(), logdet, T, c, 2.0, inverse=inverse).cpu()
  if inverse:
    ref = x2 / s - bias
    bound = 8 * U * (x2.abs() / s + bias.abs())
  else:
    ref = (x2 + bias) * s
    bound = 8 * U * (x2.abs() + bias.abs()) * s
  got = y.view(n, D)[:, idx[D // 2:].long()].view(n * T, c).double()
  assert ((got - ref).abs() <= bound).all(), float(((got - ref).abs() / bound).max())
  assert torch.equal(y.view(n, D)[:, idx[:D // 2].long()], x.view(n, D)[:, idx[:D // 2].long()])
  terms = (torch.nn.functional.logsigmoid(raw) + math.log(2)).view(n, -1)
  ref_ld = ld0.double() + (-1 if inverse else 1) * terms.sum(1)
  ld_bound = 32 * U * (terms.abs().sum(1) + ld0.double().abs())
  assert ((logdet.cpu().double() - ref_ld).abs() <= ld_bound).all()
  # in place: the same bits
  xi, ldi = x.cuda(), ld0.cuda()
  ops.jet_coupling_fwd(xi, idx.cuda(), br.cuda(), ldi, T, c, 2.0, inverse=inverse, out=xi)
  assert torch.equal(xi.cpu(), y) and torch.equal(ldi, logdet)


def test_coupling_bwd_elementwise():
  from big_vision_b200 import ops
  n, T, c = 3, 16, 24
  D = 2 * T * c
  x, br, idx = _coupling_case(n, T, c, seed=1)
  dy = torch.randn(n, T, 2 * c)
  dlogdet = -1.0 / (n * D * math.log(2))
  x2, bias, raw, s = _ref_affine(x, br, idx, T, c)
  dy2 = dy.double().view(n, D)[:, idx[D // 2:].long()].view(n * T, c)
  sig = torch.sigmoid(raw)
  ref_dx2 = dy2 * s
  ref_draw = dy2 * (x2 + bias) * s * (1 - sig) + dlogdet * (1 - sig)
  dx = torch.full((n, T, 2 * c), float("nan"), device="cuda")
  _, dbr = ops.jet_coupling_bwd(dy.cuda(), x.cuda(), idx.cuda(), br.cuda(), dlogdet, T, c, 2.0, dx=dx)
  dx, dbr = dx.cpu().view(n, D), dbr.cpu().double()
  got_dx2 = dx[:, idx[D // 2:].long()].view(n * T, c).double()
  assert ((got_dx2 - ref_dx2).abs() <= 4 * U * ref_dx2.abs()).all()
  assert torch.isnan(dx[:, idx[:D // 2].long()]).all()          # x1's positions belong to bv_jet_merge_grad
  # one bf16 rounding (half an ulp: at most 2^-8 relative) on top of a few fp32 roundings
  assert ((dbr[:, :c] - ref_dx2).abs() <= 2.0 ** -8 * ref_dx2.abs() + 8 * U * ref_dx2.abs()).all()
  draw_bound = 2.0 ** -8 * ref_draw.abs() + 16 * U * ((dy2 * (x2.abs() + bias.abs()) * s).abs() + abs(dlogdet)) * (1 - sig)
  assert ((dbr[:, c:] - ref_draw).abs() <= draw_bound).all()
  # dx may alias dy
  dyc = dy.cuda()
  ops.jet_coupling_bwd(dyc, x.cuda(), idx.cuda(), br.cuda(), dlogdet, T, c, 2.0, dx=dyc)
  assert torch.equal(dyc.cpu().view(n, D)[:, idx[D // 2:].long()], dx[:, idx[D // 2:].long()])
  assert torch.equal(dyc.cpu().view(n, D)[:, idx[:D // 2].long()], dy.view(n, D)[:, idx[:D // 2].long()])


def test_extreme_raw_scales_stay_finite():
  from big_vision_b200 import ops
  n, T, c = 2, 16, 24
  x, br, idx = _coupling_case(n, T, c, seed=2)
  vals = torch.tensor([80.0, -80.0, 1e4, -1e4])
  br[:, c:] = vals.repeat(n * T * c // 4 + 1)[:n * T * c].view(n * T, c)
  logdet = torch.zeros(n, device="cuda")
  y = ops.jet_coupling_fwd(x.cuda(), idx.cuda(), br.cuda(), logdet, T, c, 2.0)
  assert torch.isfinite(y).all() and torch.isfinite(logdet).all()
  ref = (torch.nn.functional.logsigmoid(br[:, c:].double()) + math.log(2)).view(n, -1).sum(1)
  assert ((logdet.cpu().double() - ref).abs() <= 32 * U * ref.abs()).all()
  dx, dbr = ops.jet_coupling_bwd(torch.randn(n, T, 2 * c, device="cuda"), x.cuda(), idx.cuda(), br.cuda(), -1e-3,
                                 T, c, 2.0)
  D = 2 * T * c
  assert torch.isfinite(dx.view(n, D)[:, idx[D // 2:].long().cuda()]).all() and torch.isfinite(dbr.float()).all()


def test_bits_elementwise():
  from big_vision_b200 import ops
  n, D = 5, 12288
  z = torch.randn(n, 256, 48) * 1.5
  logdet = torch.randn(n) * 1000
  grad_scale = 1.0 / (n * D * math.log(2))
  rows, means, dz = ops.jet_bits(z.cuda(), logdet.cuda(), grad_scale)
  zd = z.double().view(n, -1)
  nll = (0.5 * zd * zd).sum(1) + D * (0.5 * math.log(2 * math.pi) + math.log(127.5))
  norm = D * math.log(2)
  ref = torch.stack([(nll - logdet.double()) / norm, nll / norm, logdet.double() / norm])
  assert ((rows.cpu().double() - ref).abs() <= 1e-5 * ref.abs() + 1e-6).all()
  assert ((means.cpu().double() - ref.mean(1)).abs() <= 1e-5 * ref.abs().mean(1) + 1e-6).all()
  assert torch.equal(dz.cpu(), z * torch.tensor(grad_scale, dtype=torch.float32))
  rows2, means2 = ops.jet_bits(z.cuda(), logdet.cuda())
  assert torch.equal(rows2, rows) and torch.equal(means2, means)


def test_logdet_and_bits_are_bit_identical_across_runs():
  from big_vision_b200 import ops
  n, T, c = 64, 256, 24
  x, br, idx = _coupling_case(n, T, c, seed=3)
  x, br, idx = x.cuda(), br.cuda(), idx.cuda()
  outs = []
  for _ in range(2):
    logdet = torch.zeros(n, device="cuda")
    y = ops.jet_coupling_fwd(x, idx, br, logdet, T, c, 2.0)
    rows, means, dz = ops.jet_bits(y, logdet, 1e-3)
    outs.append((y, logdet, rows, means, dz))
  for a, b in zip(*outs):
    assert torch.equal(a, b)


def test_refusals():
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  img = torch.zeros(1, 6, 8, 3, device="cuda")
  with pytest.raises(L.BvError, match="bv_jet_dequantize_patchify"):
    ops.jet_dequantize_patchify(img, 4)
  with pytest.raises(L.BvError, match="offset"):
    ops.jet_dequantize_patchify(torch.zeros(1, 8, 8, 3, device="cuda"), 4, offset=-1)
  with pytest.raises(L.BvError, match="bv_jet_unpatchify"):
    ops.jet_unpatchify(torch.zeros(1, 3, 48, device="cuda"), (1, 6, 8, 3), 4)
  x, idx = torch.zeros(1, 4, 16, device="cuda"), torch.arange(64, dtype=torch.int32, device="cuda")
  with pytest.raises(L.BvError, match="bv_jet_split"):
    ops.jet_split(torch.zeros(0, 4, 16, device="cuda"), idx, 4, 8)        # an empty batch
  with pytest.raises(L.BvError, match="scale_factor"):
    ops.jet_coupling_fwd(x, idx, torch.zeros(4, 16, device="cuda"), torch.zeros(1, device="cuda"), 4, 8,
                         scale_factor=0.0)


# ---- the model ----------------------------------------------------------------------------------------------
def _model(**kw):
  from big_vision_b200.models.proj.jet import jet
  return jet.Model(**{**TINY, **kw})


def _randomise_final_proj(P, seed=0, scale=0.1):
  g = torch.Generator().manual_seed(seed)
  for k in ("couplings/dnn/final_proj/kernel", "couplings/dnn/final_proj/bias"):
    P.f(k).copy_(torch.randn(P.f(k).shape, generator=g) * scale)
  P.sync_half()


def _setup(seed=0, shape=TINY_SHAPE, scale=0.03, **kw):
  """A tiny Jet whose final_proj is random (zero at init, where every other DNN gradient is zero too).  The
  couplings multiply x2 by s in (0, 2) and so amplify the bf16 DNN's rounding differences from one coupling to
  the next; `scale` keeps them comparable to the tolerances below."""
  model = _model(**kw)
  P = model.init(seed, shape, device="cuda")
  _randomise_final_proj(P, seed, scale)
  return model, P


def _oracle_cfg(model):
  return dict(depth=model.depth, block_depth=model.block_depth, num_heads=model.num_heads, ps=model.ps,
              kinds=model.kinds, scale_factor=model.scale_factor)


def _noisy(image, seed, counter, offset=0):
  return image + _np_noise(seed, counter, offset, image.size).reshape(image.shape) * NOISE


def test_model_matches_the_fp64_oracle():
  from big_vision_b200.trainers.proj.jet import train as jt
  model, P = _setup()
  assert sorted(k for k, _, _ in model.couplings) == [0, 1, 1, 1, 1]
  image = _image(TINY_SHAPE, 1)
  rows, means = jt.loss_and_grads(model, P, torch.from_numpy(image).cuda(), (7, 2, 0))
  (z, _), _ = model.fwd(P, torch.from_numpy(image).cuda(), frozen=True, noise=(7, 2, 0))
  tree = P.numpy_tree("f")
  loss, ref_rows, ref_z, ref_g = JO.value_and_grad(tree, _noisy(image, 7, 2), _oracle_cfg(model), "bfloat16")
  rows = rows.cpu().double().numpy()
  ref_zt = _np_patchify(ref_z, model.ps)
  errs = {"loss": abs(float(means[0]) - loss) / abs(loss),
          "rows": float((np.abs(rows - ref_rows) / np.abs(ref_rows)).max()),
          "z": float(np.abs(z.cpu().numpy() - ref_zt).max() / np.abs(ref_zt).max())}
  grads = P.numpy_tree("g")
  for k, ref in ref_g.items():
    if k.endswith("FREEZE_ME"):
      assert not np.any(grads[k]), k
      continue
    # the key bias has no gradient in exact arithmetic (softmax ignores a per-query shift): bound it by the
    # scale of the value bias's gradient instead
    scale = np.abs(ref_g[k.replace("key/bias", "value/bias")]).max() if k.endswith("key/bias") else np.abs(ref).max()
    assert scale > 0, k
    errs[k] = float(np.abs(grads[k] - ref).max() / scale)
  print(errs)
  assert errs.pop("loss") <= 5e-3 and errs.pop("rows") <= 5e-3
  assert errs.pop("z") <= 2.0 ** -7
  assert max(errs.values()) <= 6e-2, errs


def test_inverse_of_forward_returns_the_image_and_recomputes_bias_and_scale_bit_for_bit():
  from big_vision_b200 import ops
  model, P = _setup(seed=4)
  image = torch.from_numpy(_image(TINY_SHAPE, 2)).cuda()
  z, ld = model.forward(P, image)
  x, ld_inv = model.inverse(P, z)
  assert (x - image).abs().max() <= 1e-5 * image.abs().max()
  assert (ld + ld_inv).abs().max() <= 1e-5 * ld.abs().max()
  assert ld.abs().min() > 0
  # per coupling: the DNN sees the same x1 bits before and after the coupling, so the inverse recomputes the
  # forward's bias and raw scale exactly
  stage = model._stages[1]
  x = ops.jet_dequantize_patchify(image, model.ps, noise_scale=0.0)
  n = image.shape[0]
  for i in range(model.depth):
    idx = P.jet_tables[i]
    br_fwd, _ = stage.dnn_fwd(P, i, ops.jet_split(x, idx, model.T, model.c), n, save=False)
    y = ops.jet_coupling_fwd(x, idx, br_fwd, torch.zeros(n, device="cuda"), model.T, model.c)
    br_inv, _ = stage.dnn_fwd(P, i, ops.jet_split(y, idx, model.T, model.c), n, save=False)
    assert torch.equal(br_fwd, br_inv), i
    x = y


def test_checkpoint_with_other_masks_loads_and_the_outputs_follow_them(tmp_path):
  from big_vision_b200 import utils as u
  from big_vision_b200.models.proj.jet import jet
  model, P = _setup(seed=0)
  src_model, src = _setup(seed=11)
  cm = "channel_coupling_masks-FREEZE_ME"
  assert not np.array_equal(P.numpy_tree("f")[cm], src.numpy_tree("f")[cm])
  path = str(tmp_path / "jet.npz")
  np.savez(path, **src.numpy_tree("f"))
  image = torch.from_numpy(_image(TINY_SHAPE, 3)).cuda()
  before, _ = model.forward(P, image)
  init = u.recover_tree(*zip(*P.numpy_tree("f").items()))
  P.load_tree(jet.load(init, path, dict(TINY)))
  after, ld = model.forward(P, image)
  want, want_ld = src_model.forward(src, image)
  assert torch.equal(after, want) and torch.equal(ld, want_ld)
  assert not torch.equal(after, before)
  p = {k: torch.from_numpy(v).double() for k, v in P.numpy_tree("f").items()}
  ref_z, ref_ld = JO.forward(p, image.cpu().double(), _oracle_cfg(model), "bfloat16")
  assert (after.cpu().double() - ref_z).abs().max() <= 2.0 ** -7 * ref_z.abs().max()
  assert ((ld.cpu().double() - ref_ld).abs() <= 5e-3 * ref_ld.abs()).all()


# ---- the trainer -------------------------------------------------------------------------------------------
def _config():
  return dict(seed=5, optax_name="scale_by_adam", optax=dict(mu_dtype="bfloat16", b2=0.95), grad_clip_norm=1.0,
              lr=3e-4, wd=1e-5, wd_mults=((".*", 1.0),),
              schedule=[(".*FREEZE_ME.*", None), (".*", dict(decay_type="cosine", warmup_percent=0.1))])


def test_trainer_steps_keep_the_masks_and_report_the_reference_measurements():
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.models.proj.jet import jet
  from big_vision_b200.trainers.proj.jet import train as jt
  model, P = _setup(seed=0)
  config = _config()
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=20))
  state = {"params": P, "opt": tx.init(P)}
  masks = {k: P.f(k).clone() for k in jet.MASKS}
  tables = P.jet_tables.clone()
  update_fn = jt.make_update_fn(model, tx, config)
  image = torch.from_numpy(_image(TINY_SHAPE, 4)).cuda()
  for step in range(3):
    noisy = _noisy(image.cpu().numpy(), 5, step)
    want = JO.bits_per_dim(*JO.forward({k: torch.from_numpy(v).double() for k, v in P.numpy_tree("f").items()},
                                       torch.from_numpy(noisy).double(), _oracle_cfg(model), "bfloat16"))[0].mean()
    state, m = update_fn(state, None, {"image": image})
    assert set(m) == set(jt.MEASUREMENTS)
    assert abs(float(m["training_loss"]) - float(want)) <= 5e-3 * abs(float(want))
    assert float(m["bits"]) == float(m["training_loss"])
    all_sq = float((P.flat.double() ** 2).sum())
    mask_sq = sum(float((v.double() ** 2).sum()) for v in masks.values())
    assert float(m["l2_params"]) == pytest.approx(math.sqrt(all_sq), rel=1e-4)
    assert mask_sq > 1e-2 * all_sq          # so the first check tells whether the masks are counted
    assert all(math.isfinite(float(v)) for v in m.values())
  assert state["opt"]["count"] == 3
  for k, v in masks.items():
    assert torch.equal(P.f(k), v), k
  assert torch.equal(P.jet_tables, tables)
  preds = jt.make_predict_fns(model, config)["loss"](P, {"image": image}, 5, 0)
  assert set(preds) == {"bits", "nll", "logdet"} and preds["bits"].shape == (TINY_SHAPE[0],)


def _worker(rank, world, port, ret):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  from big_vision_b200.trainers.proj.image_text.siglip import Dist
  from big_vision_b200.trainers.proj.jet import train as jt
  import test_jet_gpu as t
  model, P = t._setup(seed=0)
  image = t._image(TINY_SHAPE, 5)
  n = TINY_SHAPE[0] // world
  shard = torch.from_numpy(image[rank * n:(rank + 1) * n]).cuda()
  d = Dist()
  _, means = jt.loss_and_grads(model, P, shard, (5, 1, rank * shard.numel()), d)
  d.all_reduce_sum(means)
  torch.cuda.synchronize()
  if rank == 0:
    ret["grad"] = (P.grad / world).cpu().numpy()
    ret["bits"] = float(means[0]) / world
  dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_step_equals_the_single_rank_global_batch():
  import torch.multiprocessing as mp
  from big_vision_b200.trainers.proj.jet import train as jt
  ctx = mp.get_context("spawn")
  ret = ctx.Manager().dict()
  port = 29700 + os.getpid() % 150 + 3
  procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  model, P = _setup(seed=0)
  _, means = jt.loss_and_grads(model, P, torch.from_numpy(_image(TINY_SHAPE, 5)).cuda(), (5, 1, 0))
  g1, g2 = P.grad.cpu().numpy(), ret["grad"]
  assert ret["bits"] == pytest.approx(float(means[0]), rel=1e-5)
  assert np.abs(g1 - g2).max() <= 2e-2 * np.abs(g1).max()
  assert np.linalg.norm(g1 - g2) <= 1e-2 * np.linalg.norm(g1)
