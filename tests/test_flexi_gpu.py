"""GPU: the FlexiViT resampling kernels (include/bv_b200_flexi.h) element by element against float64, and
the FlexiViT model and trainer (models/proj/flexi, trainers/proj/flexi) against the float64 oracle
(tests/flexi_oracle.py on oracle/bv_oracle.py): forward and backward at every sequence length of
configs/proj/flexivit/i21k_sup.py on 240 px images, vit.Model's forward bits where nothing is resampled,
three Adam steps on drawn sequence lengths, the predict functions and a 2-rank NCCL step."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

import flexi_oracle as FO
from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEQHW = (5, 6, 8, 10, 12, 15, 16, 20, 24, 30)            # configs/proj/flexivit/i21k_sup.py
EPS = 2.0 ** -24


def _fv():
  from big_vision_b200.models.proj.flexi import vit as fv
  return fv


# ---- the kernels ---------------------------------------------------------------------------------------
def _matrix(kind, a, b):
  fv = _fv()
  return fv.pi_resize_matrix(a, b) if kind == "patch" else fv.posemb_resize_matrix((a, a), b)


# (kind, base, target, J): the kernel at every patch size of i21k_sup (J = 3 * 768), the posemb at every
# seqhw (J = 768), base 32 kernels, and the smallest legal shape
SHAPES = ([("patch", 8, 240 // s, 3 * 768) for s in SEQHW if 240 // s != 8]
          + [("posemb", 7, s, 768) for s in SEQHW]
          + [("patch", 32, p, 3 * 768) for p in (8, 16, 48)]
          + [("one", 1, 1, 4)])


def _operands(kind, a, b, J, seed):
  M = np.ones((1, 1)) if kind == "one" else _matrix(kind, a, b)
  M32 = M.astype(np.float32)
  g = torch.Generator().manual_seed(seed)
  R, K = M32.shape
  x = torch.randn(K, J, generator=g, dtype=torch.float64).float()
  dy = torch.randn(R, J, generator=g, dtype=torch.float64).float()
  return torch.from_numpy(M32), x, dy


def _shape_id(s):
  return f"{s[0]}{s[1]}to{s[2]}_J{s[3]}"


@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
def test_resample_fwd_elementwise(shape):
  """y = bf16(M x): within the bf16 half-ulp of the exact value plus K * 2^-24 * sum |M||x| of fp32 sums."""
  from big_vision_b200 import ops
  M, x, _ = _operands(*shape, seed=1)
  y = ops.resample_fwd(M.cuda(), x.cuda()).cpu().double()
  M64, x64 = M.double(), x.double()
  ref = M64 @ x64
  K = M.shape[1]
  acc = K * EPS * (M64.abs() @ x64.abs())
  bound = 2.0 ** -8 * (ref.abs() + acc) + acc + 1e-30
  err = (y - ref).abs()
  assert bool((err <= bound).all()), float((err / bound).max())
  assert y.shape == (M.shape[0], x.shape[1])


@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
def test_resample_bwd_elementwise(shape):
  """dx += M^T dy into a nonzero dx: within R * 2^-24 * sum |M||dy| plus the final fp32 add's rounding."""
  from big_vision_b200 import ops
  M, _, dy = _operands(*shape, seed=2)
  R, K = M.shape
  dx0 = torch.randn(K, dy.shape[1], generator=torch.Generator().manual_seed(3), dtype=torch.float64).float()
  dx = dx0.cuda()
  ops.resample_bwd(M.cuda(), dy.cuda(), dx)
  M64, dy64 = M.double(), dy.double()
  ref = dx0.double() + M64.T @ dy64
  acc = R * EPS * (M64.abs().T @ dy64.abs())
  bound = acc * (1 + EPS) + EPS * ref.abs() + 1e-30
  err = (dx.cpu().double() - ref).abs()
  assert bool((err <= bound).all()), float((err / bound).max())


def test_resample_bit_identical_across_runs():
  from big_vision_b200 import ops
  for shape in (("patch", 8, 48, 3 * 768), ("posemb", 7, 30, 768), ("patch", 32, 16, 3 * 768)):
    M, x, dy = (t.cuda() for t in _operands(*shape, seed=4))
    y1, y2 = ops.resample_fwd(M, x), ops.resample_fwd(M, x)
    assert torch.equal(y1, y2)
    d1 = torch.zeros_like(x)
    d2 = torch.zeros_like(x)
    ops.resample_bwd(M, dy, d1)
    ops.resample_bwd(M, dy, d2)
    assert torch.equal(d1, d2)


def test_resample_refusals():
  """Every malformed call returns BV_ERR_INVALID (-1) before anything is launched and leaves the output
  untouched."""
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  lib = L.load()
  M = torch.ones(4, 4, device="cuda")
  x = torch.ones(4 * 8 + 4, device="cuda")
  y = torch.full((4 * 8 + 8,), 7.0, device="cuda").bfloat16()
  dx = torch.full((4 * 8 + 4,), 7.0, device="cuda")
  pm, px, py, pd = (t.data_ptr() for t in (M, x, y, dx))
  s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  fwd = lambda m, a, o, R, K, J: lib.bv_resample_fwd(m, a, o, R, K, J, s)
  bwd = lambda m, a, o, R, K, J: lib.bv_resample_bwd(m, a, o, R, K, J, s)
  cases = [fwd(pm, px, py, 4, 4, 6), fwd(pm, px, py, 0, 4, 8), fwd(pm, px, py, 4, 0, 8), fwd(pm, px, py, 4, 4, 0),
           fwd(None, px, py, 4, 4, 8), fwd(pm, None, py, 4, 4, 8), fwd(pm, px, None, 4, 4, 8),
           fwd(pm, px + 4, py, 4, 4, 8), fwd(pm, px, py + 2, 4, 4, 8),
           bwd(pm, px, pd, 4, 4, 6), bwd(pm, px, pd, 0, 4, 8), bwd(pm, px, pd, 4, 0, 8),
           bwd(None, px, pd, 4, 4, 8), bwd(pm, None, pd, 4, 4, 8), bwd(pm, px, None, 4, 4, 8),
           bwd(pm, px + 4, pd, 4, 4, 8), bwd(pm, px, pd + 8, 4, 4, 8)]
  assert cases == [-1] * len(cases)
  assert "bv_resample_bwd" in lib.bv_last_error_string().decode()
  with pytest.raises(L.BvError, match="multiple of 4"):
    ops.resample_fwd(M, x[:24].view(4, 6))
  with pytest.raises(L.BvError, match="multiple of 4"):
    ops.resample_bwd(M, x[:24].view(4, 6), dx[:24].view(4, 6))
  torch.cuda.synchronize()
  assert bool((y.float() == 7.0).all()) and bool((dx == 7.0).all())


# ---- the model -----------------------------------------------------------------------------------------
NC = 13        # C % 8 != 0: the padded head
D, HEADS, DEPTH = 128, 2, 2


def _model(pool="tok", posemb="learn", **kw):
  fv = _fv()
  return fv.Model(NC, width=D, depth=DEPTH, mlp_dim=2 * D, num_heads=HEADS, patch_size=(8, 8), pool_type=pool,
                  posemb=posemb, **kw)


def _cfg(pool="tok", posemb="learn"):
  return dict(depth=DEPTH, num_heads=HEADS, pool_type=pool, posemb=posemb, posemb_size=(7, 7), num_classes=NC)


def _setup(model, n=2, hw=240, seed=0):
  P = model.init(seed, (n, hw, hw, 3), device="cuda")
  rng = np.random.default_rng(seed + 10)
  tree = {k: ((rng.standard_normal(v.shape) * 0.05).astype(np.float32) if not np.any(v) else v)
          for k, v in P.numpy_tree("f").items()}
  P.load_tree(tree)
  image = rng.uniform(-1, 1, size=(n, hw, hw, 3)).astype(np.float32)
  labels = np.eye(NC, dtype=np.float32)[rng.integers(0, NC, size=n)]
  return P, tree, image, labels


def _assert_close(grads, ref):
  gmax = max(float(np.abs(v).max()) for v in ref.values())
  bad = {}
  for k, g in grads.items():
    err = float(np.abs(g.astype(np.float64) - ref[k]).max())
    tol = 6e-2 * float(np.abs(ref[k]).max()) + 3e-3 * gmax
    if err > tol:
      bad[k] = (err, tol)
  assert not bad, sorted(bad.items(), key=lambda kv: -kv[1][0])[:8]
  assert gmax > 0


@pytest.mark.parametrize("seqhw", SEQHW)
@pytest.mark.parametrize("pool,posemb", [("tok", "learn"), ("gap", "learn"), ("map", "learn"), ("tok", "sincos2d"),
                                         ("gap", "sincos2d"), ("map", "sincos2d")])
def test_forward_and_backward_match_oracle(pool, posemb, seqhw):
  """Logits, loss and every gradient -- embedding/kernel [8, 8, 3, d] and pos_embedding [1, 49, d] among
  them -- at patch 240 // seqhw and seqhw^2 (+ cls) tokens, against float64."""
  from big_vision_b200 import train
  model = _model(pool, posemb)
  P, tree, image, labels = _setup(model, seed=seqhw)
  loss, logits = train.loss_and_grads(model, P, torch.from_numpy(image).cuda(), torch.from_numpy(labels).cuda(),
                                      seqhw=seqhw)
  ref_loss, ref_g = FO.value_and_grad(tree, image, labels, _cfg(pool, posemb), seqhw)
  ref_logits = FO.flexi_forward(O.to_f64_tree(tree), torch.from_numpy(image), _cfg(pool, posemb), seqhw).detach()
  got = logits.cpu().double()
  assert got.shape == (2, NC)
  assert float((got - ref_logits).abs().max()) <= 4e-2 * float(ref_logits.abs().max())
  assert float(loss) == pytest.approx(ref_loss, rel=5e-3)
  grads = P.numpy_tree("g")
  assert grads["embedding/kernel"].shape == (8, 8, 3, D)
  if posemb == "learn":
    assert grads["pos_embedding"].shape == (1, 49, D) and np.abs(grads["pos_embedding"]).max() > 0
  _assert_close(grads, ref_g)


@pytest.mark.parametrize("pool,posemb", [("tok", "learn"), ("gap", "sincos2d"), ("map", "learn")])
def test_no_resample_path_is_bitwise_vit(pool, posemb):
  """At p == p0 and a 7 x 7 grid (56 px, seqhw 7) the step is vit.Model's: the logits and the loss are its
  bits, and every gradient agrees to fp32 reassociation.  (The gradients cannot be held to their bits: the
  split-K and column-sum accumulations of the backward add with atomics, whose order differs from run to
  run of the same model.)"""
  from big_vision_b200 import train
  from big_vision_b200.models import vit
  model = _model(pool, posemb)
  P, tree, image, labels = _setup(model, n=4, hw=56)
  ref_model = vit.Model(NC, width=D, depth=DEPTH, mlp_dim=2 * D, num_heads=HEADS, patch_size=(8, 8), pool_type=pool,
                        posemb=posemb)
  Pv = ref_model.init(0, (4, 56, 56, 3), device="cuda").load_tree(tree)
  img, lab = torch.from_numpy(image).cuda(), torch.from_numpy(labels).cuda()
  loss, logits = train.loss_and_grads(model, P, img, lab, seqhw=7)
  loss_v, logits_v = train.loss_and_grads(ref_model, Pv, img, lab)
  assert torch.equal(logits, logits_v) and torch.equal(loss, loss_v)
  g, gv = P.numpy_tree("g"), Pv.numpy_tree("g")
  assert set(g) == set(gv)
  # the floor tied to the largest gradient covers gradients that are zero in exact arithmetic (key/bias:
  # softmax ignores a per-query constant), whose stored values are rounding noise of either run
  gmax = max(float(np.abs(v).max()) for v in gv.values())
  for k in g:
    assert np.abs(g[k] - gv[k]).max() <= 1e-5 * np.abs(gv[k]).max() + 1e-7 * gmax, k


def test_frozen_embedding_resamples_and_saves_nothing():
  from big_vision_b200 import train
  model = _model()
  P, _, image, labels = _setup(model)
  img = torch.from_numpy(image).cuda()
  x_all, saved = model.fwd(P, img, seqhw=12, frozen=True)
  assert all(s is None for s in saved["stages"])
  x, _ = model.fwd(P, img, seqhw=12)
  assert torch.equal(x, x_all)
  frozen = {n for n in P.offsets if not n.startswith("head/")}
  train.loss_and_grads(model, P, img, torch.from_numpy(labels).cuda(), frozen=frozen, seqhw=12)
  assert float(P.g("embedding/kernel_flat").abs().max()) == 0.0 and float(P.g("head/kernel_pad").abs().max()) > 0


# ---- training and prediction ------------------------------------------------------------------------------
def _config(**kw):
  return dict(optax_name="scale_by_adam", optax=dict(mu_dtype="float32"), lr=1e-3, wd=0.0, grad_clip_norm=1.0,
              schedule=dict(decay_type="linear", warmup_steps=0, linear_end=0.01), loss="sigmoid_xent",
              flexi=dict(seqhw=dict(v=SEQHW, p=(1,) * len(SEQHW))), **kw)


def _flat(tree):
  return np.concatenate([np.asarray(tree[k], dtype=np.float64).ravel() for k in sorted(tree)])


def test_update_fn_three_adam_steps_track_oracle():
  """make_update_fn with Adam and mixup at the seqhw flexi_args draws for steps 0, 1, 2 follows the
  oracle's trajectory."""
  from big_vision_b200 import optax as bv_optax, utils as u
  from big_vision_b200.trainers.proj.flexi import train as ft
  model = _model("tok")
  P, tree, image, labels = _setup(model, n=4)
  config = _config(mixup=dict(p=0.8))
  lr = config["lr"]
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=10, batch_size=4, data_size=1000))
  state = {"params": P, "opt": tx.init(P)}
  fn = ft.make_update_fn(model, tx, config)
  p_ref = {k: v.astype(np.float64) for k, v in tree.items()}
  m_ref = {k: np.zeros_like(v) for k, v in p_ref.items()}
  v_ref = {k: np.zeros_like(v) for k, v in p_ref.items()}
  rng, rng_ref = np.random.default_rng(21), np.random.default_rng(21)
  seen = []
  for step in range(3):
    kw = ft.flexi_args(config, step)
    seen.append(kw["seqhw"])
    state, m = fn(state, rng, {"image": torch.from_numpy(image).cuda(), "labels": torch.from_numpy(labels).cuda()},
                  **kw)
    a32 = np.float32(u.get_mixup(rng_ref, 0.8).a)
    mix = lambda v: a32 * v + (np.float32(1) - a32) * np.roll(v, 1, axis=0)
    ref_loss, g = FO.value_and_grad(p_ref, mix(image), mix(labels), _cfg("tok"), kw["seqhw"])
    assert float(m["training_loss"]) == pytest.approx(ref_loss, rel=5e-3), step
    gnorm = math.sqrt(sum(float((v ** 2).sum()) for v in g.values()))
    assert float(m["l2_grads"]) == pytest.approx(gnorm, rel=5e-2)
    sched = tx.sched_fns[0](step)
    for k in p_ref:
      p_ref[k], m_ref[k], v_ref[k] = O.adam_reference(p_ref[k], g[k], m_ref[k], v_ref[k], step + 1, lr=lr, b1=0.9,
                                                      b2=0.999, eps=1e-8, wd=0.0, sched=sched, clip=1.0, gnorm=gnorm)
  assert seen == [ft.flexi_args(config, s)["seqhw"] for s in range(3)]
  got = P.numpy_tree("f")
  d_got, d_ref = _flat(got) - _flat(tree), _flat(p_ref) - _flat(tree)
  cos = float(d_got @ d_ref / (np.linalg.norm(d_got) * np.linalg.norm(d_ref)))
  assert cos > 0.95, cos
  assert np.linalg.norm(d_got) == pytest.approx(np.linalg.norm(d_ref), rel=0.1)
  assert np.abs(_flat(got) - _flat(p_ref)).max() <= 10 * lr


def test_predict_fns_equal_apply_at_each_seqhw():
  from big_vision_b200.trainers.proj.flexi import train as ft
  model = _model("map")
  P, _, image, _ = _setup(model)
  img = torch.from_numpy(image).cuda()
  fns = ft.make_predict_fns(model, _config())
  assert list(fns) == [f"predict_seqhw={s}" for s in SEQHW]
  for s in SEQHW:
    logits, out = fns[f"predict_seqhw={s}"](P, img)
    ref, _ = model.apply({"params": P}, img, seqhw=s)
    assert torch.equal(logits, ref) and torch.equal(out["logits"], ref), s


def _half_batch_average(model, P, image, labels, seqhw):
  from big_vision_b200 import train
  acc = torch.zeros_like(P.grad)
  for r in range(2):
    sl = slice(2 * r, 2 * r + 2)
    train.loss_and_grads(model, P, torch.from_numpy(image[sl]).cuda(), torch.from_numpy(labels[sl]).cuda(),
                         seqhw=seqhw)
    acc += P.grad
  return acc / 2


def _worker(rank, world, port, ret):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.trainers.proj.flexi import train as ft
  import test_flexi_gpu as t
  model = t._model("tok")
  P, _, image, labels = t._setup(model, n=4)
  config = t._config()
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=100))
  fn = ft.make_update_fn(model, tx, config)
  sl = slice(2 * rank, 2 * rank + 2)
  fn({"params": P, "opt": tx.init(P)}, None,
     {"image": torch.from_numpy(image[sl]).cuda(), "labels": torch.from_numpy(labels[sl]).cuda()},
     **ft.flexi_args(config, 5))
  torch.cuda.synchronize()
  if rank == 0:
    ret["grad"] = (P.grad / world).cpu().numpy()
  dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_nccl_step_is_the_global_batch_step():
  import torch.multiprocessing as mp
  from big_vision_b200.trainers.proj.flexi import train as ft
  ctx = mp.get_context("spawn")
  ret = ctx.Manager().dict()
  port = 29700 + os.getpid() % 150
  procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  model = _model("tok")
  P, _, image, labels = _setup(model, n=4)
  g1 = _half_batch_average(model, P, image, labels, ft.flexi_args(_config(), 5)["seqhw"]).cpu().numpy()
  g2 = ret["grad"]
  assert np.abs(g1 - g2).max() <= 2e-2 * np.abs(g1).max()
  assert np.linalg.norm(g1 - g2) <= 1e-2 * np.linalg.norm(g1)
