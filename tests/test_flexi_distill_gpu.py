"""GPU: the FlexiViT distillation step (trainers/proj/flexi/distill.py) on a tiny FlexiViT student (56 px, base
patch 8, 7 x 7 grid) under a tiny frozen ViT teacher at 96 px, against the float64 oracle built from
tests/flexi_oracle.py (the student) and tests/distill_oracle.py (the loss and its gradient) on
oracle/bv_oracle.py's ViT (the teacher); against distill.loss_and_grads called directly; and as a 2-rank NCCL
step."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import distill_oracle as DO
import flexi_oracle as FO
from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NC = 13                                    # C % 8 != 0: padded heads
S_HW, T_HW = 56, 96
# seqhw 7 resamples nothing; 4 (patch 14) and 14 (patch 4) resample the kernel up and down and the grid
SEQHW = (4, 7, 14)
S_CFG = dict(depth=2, num_heads=2, pool_type="tok", posemb="learn", posemb_size=(7, 7), num_classes=NC)
T_CFG = dict(depth=2, num_heads=1, pool_type="tok", posemb="learn", rep_size=False, num_classes=NC)
LR = 1e-3


def _models():
  from big_vision_b200.models import vit
  from big_vision_b200.models.proj.flexi import vit as fv
  return {"student": fv.Model(NC, width=128, depth=2, mlp_dim=256, num_heads=2, patch_size=(8, 8), pool_type="tok"),
          "prof": vit.Model(NC, width=64, depth=2, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type="tok",
                            rep_size=False)}


def _randomize_zero_inits(tree, seed):
  rng = np.random.default_rng(seed)
  return {k: ((rng.standard_normal(v.shape) * 0.05).astype(np.float32) if not np.any(v) else v)
          for k, v in tree.items()}


def _setup(n=4, seed=0):
  """models, params (the teacher without a gradient buffer), float32 trees, host data with the teacher's
  own 96 px input under "prof"."""
  models = _models()
  rng = np.random.default_rng(seed + 100)
  data = {"labels": np.eye(NC, dtype=np.float32)[rng.integers(0, NC, size=n)],
          "image": rng.uniform(-1, 1, size=(n, S_HW, S_HW, 3)).astype(np.float32),
          "prof": rng.uniform(-1, 1, size=(n, T_HW, T_HW, 3)).astype(np.float32)}
  params, trees = {}, {}
  for i, (name, hw) in enumerate((("student", S_HW), ("prof", T_HW))):
    P = models[name].init(seed + i, (n, hw, hw, 3), device="cuda")
    trees[name] = _randomize_zero_inits(P.numpy_tree("f"), seed + 10 + i)
    P.load_tree(trees[name])
    params[name] = P
  params["prof"].drop_grad()
  return models, params, trees, data


def _cuda(data, rows=slice(None)):
  return {k: torch.from_numpy(v[rows]).cuda() for k, v in data.items()}


def _oracle(trees, data, seqhw, **kw):
  fwds = {"student": lambda p, img: FO.flexi_forward(p, img, S_CFG, seqhw),
          "prof": lambda p, img: O.vit_forward(p, img, T_CFG, "float32")}
  return DO.value_and_grad(fwds, trees, data, ("prof",), **kw)


def _config(**kw):
  return dict(optax_name="scale_by_adam", optax=dict(mu_dtype="float32"), lr=LR, wd=0.0, grad_clip_norm=1.0,
              schedule=dict(decay_type="linear", warmup_steps=0, linear_end=0.01), teachers=["prof"],
              flexi=dict(seqhw=dict(v=SEQHW, p=(1,) * len(SEQHW))), **kw)


def _assert_close(grads, ref):
  """Every gradient within 6 % of its own largest element plus 0.3 % of the largest gradient anywhere
  (bf16 operands, fp32 accumulation, against float64)."""
  gmax = max(float(np.abs(v).max()) for v in ref.values())
  bad = {}
  for k, g in grads.items():
    err = float(np.abs(g.astype(np.float64) - ref[k]).max())
    tol = 6e-2 * float(np.abs(ref[k]).max()) + 3e-3 * gmax
    if err > tol:
      bad[k] = (err, tol)
  assert not bad, sorted(bad.items(), key=lambda kv: -kv[1][0])[:8]
  assert gmax > 0


def _flat(tree):
  return np.concatenate([np.asarray(tree[k], dtype=np.float64).ravel() for k in sorted(tree)])


@pytest.mark.parametrize("seqhw", SEQHW)
def test_step_matches_oracle(seqhw):
  """One update_fn step with mixup (p 0.8) and Adam (clip 1) at `seqhw`, against float64:
    - the measurements within 3 % (1e-4 absolute);
    - every student gradient as _assert_close states, l2_grads within 5 %;
    - the updated student parameters: Adam's first step moves each by lr * g / (|g| + eps), so a
      gradient near zero whose sign differs from the oracle's moves its parameter by at most 2 lr the
      other way.  Every parameter is within 2 lr (+ fp32 rounding) of the oracle's, and the update as a
      whole points the oracle's way (cosine > 0.95, norm within 10 %);
    - the teacher has no gradient buffer, keeps nothing from its forward and is bit-unchanged."""
  from big_vision_b200 import optax as bv_optax, utils as u
  from big_vision_b200.trainers.proj.flexi import distill as fd
  models, params, trees, data = _setup()
  P = params["student"]
  config = _config(distance="kl", distance_kw=dict(t=2.0), mixup=dict(p=0.8))
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=10, batch_size=4, data_size=1000))
  state = {"params": params, "opt": tx.init(P)}
  teacher_bits = (params["prof"].flat.clone(), params["prof"].half.clone())
  fn = fd.make_update_fn(models, tx, config)
  state, m = fn(state, np.random.default_rng(21), _cuda(data), seqhw=seqhw)

  a32 = np.float32(u.get_mixup(np.random.default_rng(21), 0.8).a)
  mixed = {k: a32 * v + (np.float32(1) - a32) * np.roll(v, 1, axis=0) for k, v in data.items()}
  ref_m, ref_g = _oracle(trees, mixed, seqhw, distance="kl", distance_kw=dict(t=2.0))
  assert set(ref_m) <= set(m)
  assert float(m["training_loss"]) == float(m["distill_loss"]) == float(m["distill_loss_prof"])
  for k, v in ref_m.items():
    assert float(m[k]) == pytest.approx(v, rel=3e-2, abs=1e-4), k
  grads = P.numpy_tree("g")
  assert grads["embedding/kernel"].shape == (8, 8, 3, 128) and grads["pos_embedding"].shape == (1, 49, 128)
  _assert_close(grads, ref_g)
  gnorm = math.sqrt(sum(float((v ** 2).sum()) for v in ref_g.values()))
  assert float(m["l2_grads"]) == pytest.approx(gnorm, rel=5e-2)

  sched = tx.sched_fns[0](0)
  p_ref = {}
  for k, p0 in trees["student"].items():
    p0 = p0.astype(np.float64)
    p_ref[k], _, _ = O.adam_reference(p0, ref_g[k], np.zeros_like(p0), np.zeros_like(p0), 1, lr=LR, b1=0.9,
                                      b2=0.999, eps=1e-8, wd=0.0, sched=sched, clip=1.0, gnorm=gnorm)
  got = P.numpy_tree("f")
  pmax = float(np.abs(_flat(p_ref)).max())
  assert np.abs(_flat(got) - _flat(p_ref)).max() <= 2 * LR * sched + 1e-6 * pmax
  d_got, d_ref = _flat(got) - _flat(trees["student"]), _flat(p_ref) - _flat(trees["student"])
  cos = float(d_got @ d_ref / (np.linalg.norm(d_got) * np.linalg.norm(d_ref)))
  assert cos > 0.95, cos
  assert np.linalg.norm(d_got) == pytest.approx(np.linalg.norm(d_ref), rel=0.1)
  assert float(m["l2_params"]) == pytest.approx(np.linalg.norm(_flat(got)), rel=1e-3)

  assert params["prof"].grad is None
  assert torch.equal(params["prof"].flat, teacher_bits[0]) and torch.equal(params["prof"].half, teacher_bits[1])
  _, saved = models["prof"].fwd(params["prof"], _cuda(data)["prof"], frozen=True)
  assert all(s is None for s in saved["stages"])


@pytest.mark.parametrize("seqhw", SEQHW)
def test_step_gradient_is_distill_loss_and_grads(seqhw):
  """The step's student gradient is distill.loss_and_grads's at the same seqhw.  Its measurements (the
  forward only) are the same bits.  The gradients are held to fp32 reassociation, not to their bits: the
  backward's split-K and column-sum accumulations add with atomics, so two calls of loss_and_grads itself
  differ in the last bits from run to run."""
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.trainers.proj.distill import distill as D
  from big_vision_b200.trainers.proj.flexi import distill as fd
  models, params, _, data = _setup()
  P = params["student"]
  config = _config(distance="kl", distance_kw=dict(t=1.0))
  batch = _cuda(data)
  m0 = D.loss_and_grads(models, params, batch, ("prof",), "kl", dict(t=1.0), seqhw=seqhw)
  g0 = P.numpy_tree("g")
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=10, batch_size=4, data_size=1000))
  _, m = fd.make_update_fn(models, tx, config)({"params": params, "opt": tx.init(P)}, None, batch, seqhw=seqhw)
  g = P.numpy_tree("g")
  for k, v in m0.items():
    assert torch.equal(m[k], v), k
  gmax = max(float(np.abs(v).max()) for v in g0.values())
  for k in g0:
    assert np.abs(g[k] - g0[k]).max() <= 1e-5 * np.abs(g0[k]).max() + 1e-7 * gmax, k
  assert gmax > 0


def _worker(rank, world, port, ret):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.trainers.proj.flexi import distill as fd
  import test_flexi_distill_gpu as t
  models, params, _, data = t._setup(n=8)
  P = params["student"]
  config = t._config(distance="kl", distance_kw=dict(t=2.0))
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=100))
  kw = fd.flexi_args(config, 5)                   # each rank draws for itself
  h = 8 // world
  _, m = fd.make_update_fn(models, tx, config)({"params": params, "opt": tx.init(P)}, None,
                                               t._cuda(data, slice(rank * h, (rank + 1) * h)), **kw)
  torch.cuda.synchronize()
  ret[f"seqhw{rank}"] = kw["seqhw"]
  if rank == 0:
    ret["grad"] = (P.grad / world).cpu().numpy()
    ret["m"] = {k: float(v) for k, v in m.items()}
  dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_nccl_step_is_the_whole_batch_step():
  """Both ranks draw the same seqhw; the all-reduced gradient and the measurements are those of one
  process on the whole batch, up to fp32 summation order."""
  import torch.multiprocessing as mp
  from big_vision_b200.trainers.proj.distill import distill as D
  from big_vision_b200.trainers.proj.flexi import distill as fd
  ctx = mp.get_context("spawn")
  ret = ctx.Manager().dict()
  port = 29700 + os.getpid() % 150
  procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  seqhw = fd.flexi_args(_config(), 5)["seqhw"]
  assert ret["seqhw0"] == ret["seqhw1"] == seqhw
  models, params, _, data = _setup(n=8)
  m1 = D.loss_and_grads(models, params, _cuda(data), ("prof",), "kl", dict(t=2.0), seqhw=seqhw)
  g1, g2 = params["student"].grad.cpu().numpy(), ret["grad"]
  assert np.abs(g1 - g2).max() <= 2e-2 * np.abs(g1).max()
  assert np.linalg.norm(g1 - g2) <= 1e-2 * np.linalg.norm(g1)
  for k, v in m1.items():
    assert ret["m"][k] == pytest.approx(float(v), rel=1e-3, abs=1e-6), k
