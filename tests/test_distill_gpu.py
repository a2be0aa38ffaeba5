"""GPU: the distillation kernels (include/bv_b200_distill.h) element by element against float64, and the
distillation step (trainers/proj/distill) against the float64 oracle (tests/distill_oracle.py on
oracle/bv_oracle.py's models): a ViT student under a deeper ViT teacher at another resolution, an MLP-Mixer
student, two teachers, three Adam steps with mixup, the per-rank-then-mean identity and a 2-rank NCCL step."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import distill_oracle as DO
from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = {"kl_t1": ("kl", dict(t=1.0)), "kl_t2": ("kl", dict(t=2.0)), "kl_t8": ("kl", dict(t=8.0)),
         "hard": ("hard", dict(ls=0.0)), "hard_ls": ("hard", dict(ls=0.1))}


def _randn(n, C, seed, scale=3.0):
  g = torch.Generator().manual_seed(seed)
  return (torch.randn(n, C, generator=g, dtype=torch.float64) * scale).float()


def _strided(x, ld, offset=0):
  """x as the [n, C] view of NaN-filled [n, ld] device storage that starts `offset` floats into its buffer:
  ld % 4 == 0 and offset == 0 take the 16-byte loads, anything else the 4-byte ones."""
  n, C = x.shape
  buf = torch.full((n * ld + offset,), float("nan"), device="cuda")
  view = buf[offset:].view(n, ld)[:, :C]
  view.copy_(x)
  return view


def _reference(s, u, labels, kind, kw):
  """float64: (measurements as bv_distill_loss orders them, per-row distances, d mean distance / d s)."""
  s64 = s.double().requires_grad_()
  rows = DO.dist(s64, u.double(), kind, **kw)
  rows.mean().backward()
  _, m = DO.loss_fn({"student": s.double(), "teacher": u.double()}, ("teacher",),
                    labels.double() if labels is not None else None, kind, kw)
  means = [m["distill_loss"], m["entropy_student"], m["entropy_teacher"], m.get("task_loss_student", 0.0),
           m.get("task_loss_teacher", 0.0)]
  return [float(v) for v in means], rows.detach(), s64.grad


def _check_loss(s, u, labels, kind, kw, sd, ud, ld_lab, dl_cols, rel=1e-5):
  from big_vision_b200 import ops
  n, C = s.shape
  out, rows, dl = ops.distill_loss(sd, ud, ld_lab, kind, dlogits_cols=dl_cols, **kw)
  means, ref_rows, ref_grad = _reference(s, u, labels, kind, kw)
  got = out.cpu().double().tolist()
  for name, g, r in zip(ops.L.DISTILL_OUTPUTS, got, means):
    assert g == pytest.approx(r, rel=rel, abs=1e-6), (name, g, r)
  torch.testing.assert_close(rows[0].cpu().double(), ref_rows, rtol=rel, atol=2e-6)
  assert out[0].item() == pytest.approx(rows[0].double().mean().item(), rel=1e-6, abs=1e-7)
  scale = (kw.get("t", 1.0) if kind == "kl" else 1.0) / n
  err = float((dl[:, :C].cpu().double() - ref_grad).abs().max())
  assert err <= 1e-6 * scale, (err / scale)
  assert dl.shape == (n, dl_cols) and bool((dl[:, C:] == 0).all())
  return out, rows, dl


@pytest.mark.parametrize("n", [1, 8, 256])
@pytest.mark.parametrize("C", [1, 37, 1000, 1001, 21843])
@pytest.mark.parametrize("mode", list(MODES))
def test_distill_loss_elementwise(mode, C, n):
  """Distance, measurements, per-row distances and gradient against float64; logits and gradient in head
  storage padded to a multiple of 8 columns (16-byte loads, with a 4-byte tail when C % 4 != 0), labels
  on every other case."""
  from big_vision_b200 import lib as L, ops
  kind, kw = MODES[mode]
  s, u = _randn(n, C, 1), _randn(n, C, 2)
  Cp = (C + 7) // 8 * 8
  sd, ud = _strided(s, Cp), _strided(u, Cp)
  if kind == "hard" and kw["ls"] and C == 1:
    with pytest.raises(L.BvError, match="C >= 2"):      # ls / (C - 1): nothing to smooth over
      ops.distill_loss(sd, ud, None, kind, **kw)
    return
  labels = None
  if (n + C) % 2:
    g = torch.Generator().manual_seed(3)
    labels = torch.nn.functional.one_hot(torch.randint(0, C, (n,), generator=g), C).float()
    labels = 0.7 * labels + 0.3 * labels.roll(1, 0)       # mixed labels
  _check_loss(s, u, labels, kind, kw, sd, ud, labels.cuda() if labels is not None else None, Cp)


@pytest.mark.parametrize("mode", ["kl_t2", "hard_ls"])
def test_distill_loss_scalar_path_and_accumulate(mode):
  """Rows that are not 16-byte aligned (odd stride, buffer offset by one float) take the 4-byte loads and
  give the same numbers; with a gradient passed in, the new one is added to it and the padding is kept."""
  from big_vision_b200 import ops
  kind, kw = MODES[mode]
  n, C = 8, 1001
  s, u = _randn(n, C, 4), _randn(n, C, 5)
  labels = torch.nn.functional.one_hot(torch.arange(n) * 7 % C, C).float()
  out_v, rows_v, dl_v = _check_loss(s, u, labels, kind, kw, _strided(s, 1008), _strided(u, 1008), labels.cuda(), 1008)
  out_s, rows_s, dl_s = _check_loss(s, u, labels, kind, kw, _strided(s, 1003, 1), _strided(u, 1005, 1),
                                    _strided(labels, 1001, 1), 1001)
  torch.testing.assert_close(out_s, out_v, rtol=1e-6, atol=1e-7)
  torch.testing.assert_close(dl_s, dl_v[:, :C], rtol=0, atol=1e-6 / n)
  for cols, off in ((1008, 0), (1003, 1)):                 # accumulate on both paths
    prev = _strided(_randn(n, C, 6, 1e-3), cols, off)
    prev_pad = torch.zeros(n, cols, device="cuda")
    prev_pad[:, :C] = prev
    buf = prev_pad if off == 0 else prev
    before = buf.clone()
    _, _, dl = ops.distill_loss(_strided(s, cols, off), _strided(u, cols, off), None, kind, dlogits=buf, **kw)
    assert dl is buf
    torch.testing.assert_close(buf[:, :C], before[:, :C] + dl_v[:, :C], rtol=0, atol=2e-6 / n)
    assert bool((buf[:, C:] == 0).all())


def test_distill_loss_extreme_logits_and_clip():
  """Logits of magnitude 1e4 and a row of equal logits stay finite and right; teacher probabilities below
  1e-8 enter as p log(1e-8), which shows when student == teacher: the textbook KL is 0, this one is not."""
  from big_vision_b200 import ops
  n, C = 8, 1000
  s, u = _randn(n, C, 7, 1e4), _randn(n, C, 8, 1e4)
  s[3] = 5.0
  u[3] = -2.0                                             # equal logits in both: distance 0, entropy log C
  for kind, kw in (("kl", dict(t=1.0)), ("kl", dict(t=8.0)), ("hard", dict(ls=0.1))):
    out, rows, dl = ops.distill_loss(s.cuda(), u.cuda(), None, kind, **kw)
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(rows).all()) and bool(torch.isfinite(dl).all())
    means, ref_rows, ref_grad = _reference(s, u, None, kind, kw)
    torch.testing.assert_close(rows[0].cpu().double(), ref_rows, rtol=1e-4, atol=1e-5)
    assert float((dl.cpu().double() - ref_grad).abs().max()) <= 1e-5 * kw.get("t", 1.0) / n
    if kind == "kl":
      assert abs(float(rows[0, 3])) <= 1e-6
    assert float(rows[1, 3]) == pytest.approx(math.log(C), rel=1e-6)
  C = 21843
  u = torch.full((2, C), -19.5)
  u[:, 0] = 0.0                                           # 21842 classes at p = 3.4e-9 each
  ref = DO.dist(u.double(), u.double(), "kl")
  assert float(ref.min()) > 5e-5
  _, rows, dl = ops.distill_loss(u.cuda(), u.cuda(), None, "kl")
  torch.testing.assert_close(rows[0].cpu().double(), ref, rtol=1e-3, atol=0)
  assert float(dl.abs().max()) == 0.0


def test_distill_loss_bit_identical_across_runs():
  from big_vision_b200 import ops
  for n, C, kind, kw in ((256, 1000, "kl", dict(t=2.0)), (64, 21843, "kl", dict(t=1.0)), (256, 1000, "hard", dict(ls=0.1))):
    s, u = _randn(n, C, 9).cuda(), _randn(n, C, 10).cuda()
    labels = torch.nn.functional.one_hot(torch.arange(n) % C, C).float().cuda()
    seen = set()
    for _ in range(6):
      out, rows, dl = ops.distill_loss(s, u, labels, kind, **kw)
      seen.add((tuple(out.cpu().view(torch.int32).tolist()), int(rows.view(torch.int32).sum(dtype=torch.int64)),
                int(dl.view(torch.int32).sum(dtype=torch.int64))))
    assert len(seen) == 1, seen


@pytest.mark.parametrize("n,C,ld", [(8, 37, 40), (5, 1001, 1003), (3, 21843, 21848)])
def test_distance_every_kind(n, C, ld):
  from big_vision_b200 import ops
  from big_vision_b200.evaluators.proj.distill import distance as dd
  s, u = _randn(n, C, 11), _randn(n, C, 12)
  sd, ud = _strided(s, ld), _strided(u, ld, 1 if ld % 4 else 0)
  cases = [("euclidean", dict(epsilon=1e-12)), ("euclidean", dict(epsilon=0.5)), ("l2", {}), ("hard", {}),
           ("hard", dict(ls=0.1)), ("kl", {}), ("kl", dict(t=2.0)), ("logsoftmax_euclidean", dict(epsilon=1e-12))]
  for kind, kw in cases:
    got = ops.distance(sd, ud, kind, **kw)
    assert got.dtype == torch.float32 and got.shape == (n,)
    torch.testing.assert_close(got.cpu().double(), DO.dist(s, u, kind, **kw), rtol=1e-5, atol=1e-6, msg=kind)
  for k in (1, 5):
    got = ops.distance(sd, ud, "agree", k=k)
    assert got.dtype == torch.int32
    assert got.cpu().tolist() == DO.dist(s, u, "agree", k=k).tolist()
  # dist(): any feature axis, leading axes kept; the evaluator flattens feature maps
  x, y = _randn(6, 35, 13).view(2, 3, 5, 7), _randn(6, 35, 14).view(2, 3, 5, 7)
  got = dd.dist(x.cuda(), y.cuda(), "l2", feat_axis=2)
  torch.testing.assert_close(got.cpu().double(), DO.dist(x.transpose(2, 3), y.transpose(2, 3), "l2"), rtol=1e-5, atol=0)
  got, = dd.batch_distances(x.cuda(), y.cuda(), [dict(kind="kl", t=2)])
  torch.testing.assert_close(got.cpu().double(), DO.dist(x.reshape(2, -1), y.reshape(2, -1), "kl", t=2), rtol=1e-5,
                             atol=1e-6)


@pytest.mark.parametrize("k", [1, 5])
def test_distance_agree_is_exact_on_ties(k):
  """Integer-valued logits from {0..3}: nearly every comparison is a tie, resolved by index as lax.top_k
  (student) and argmax (teacher) do."""
  from big_vision_b200 import ops
  g = torch.Generator().manual_seed(15)
  for n, C in ((64, 50), (16, 1001), (4, 21843)):
    s = torch.randint(0, 4, (n, C), generator=g).float()
    u = torch.randint(0, 4, (n, C), generator=g).float()
    got = ops.distance(s.cuda(), u.cuda(), "agree", k=k).cpu()
    ref = DO.dist(s, u, "agree", k=k)
    assert got.tolist() == ref.tolist()
    if C == 50:
      assert 0 < int(ref.sum()) < n                        # both outcomes occur
  s = torch.tensor([[4.0, 1.0, 4.0, 4.0]]).cuda()
  u = torch.tensor([[0.0, 1.0, 5.0, 2.0]]).cuda()
  assert int(ops.distance(s, u, "agree", k=k)) == (0 if k == 1 else 1)


# ---- the step ------------------------------------------------------------------------------------
NC = 16


def _randomize_zero_inits(tree, seed):
  rng = np.random.default_rng(seed)
  return {k: ((rng.standard_normal(v.shape) * 0.05).astype(np.float32) if not np.any(v) else v)
          for k, v in tree.items()}


def _vit(depth=2, pool="gap"):
  from big_vision_b200.models import vit
  model = vit.Model(NC, width=64, depth=depth, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type=pool,
                    rep_size=False)
  cfg = dict(depth=depth, num_heads=1, pool_type=pool, posemb="learn", rep_size=False, num_classes=NC)
  return model, lambda p, img: O.vit_forward(p, img, cfg, "float32")


def _mixer():
  from big_vision_b200.models import mlp_mixer
  model = mlp_mixer.Model(NC, patch_size=(16, 16), num_blocks=2, hidden_dim=64, tokens_mlp_dim=32,
                          channels_mlp_dim=128)
  cfg = dict(num_blocks=2, num_classes=NC)
  return model, lambda p, img: O.mixer_forward(p, img, cfg, "float32")


def _setup(specs, n=4, seed=0, teacher_grad=False):
  """specs {name: ((model, oracle_fwd), image_hw)} -> models, params, oracle fwds, trees, host data.  Every
  model but the student gets its own input under its name when its resolution differs."""
  models, params, fwds, trees = {}, {}, {}, {}
  rng = np.random.default_rng(seed + 100)
  data = {"labels": np.eye(NC, dtype=np.float32)[rng.integers(0, NC, size=n)]}
  for i, (name, ((model, fwd), hw)) in enumerate(specs.items()):
    shape = (n, hw, hw, 3)
    P = model.init(seed + i, shape, device="cuda")
    trees[name] = _randomize_zero_inits(P.numpy_tree("f"), seed + 10 + i)
    P.load_tree(trees[name])
    if name != "student" and not teacher_grad:
      P.drop_grad()
    models[name], params[name], fwds[name] = model, P, fwd
    data["image" if name == "student" else name] = rng.uniform(-1, 1, size=shape).astype(np.float32)
  return models, params, fwds, trees, data


def _cuda(data, rows=slice(None)):
  return {k: torch.from_numpy(v[rows]).cuda() for k, v in data.items()}


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


def _flat(tree):
  return np.concatenate([np.asarray(tree[k], dtype=np.float64).ravel() for k in sorted(tree)])


SETUPS = {
    "vit_under_deeper_vit_at_96px": (lambda: {"student": (_vit(), 64), "prof": (_vit(3, "tok"), 96)}, "kl", dict(t=2.0)),
    "mixer_under_vit": (lambda: {"student": (_mixer(), 64), "prof": (_vit(3, "tok"), 64)}, "kl", dict(t=4.0)),
    "two_teachers": (lambda: {"student": (_vit(), 64), "a": (_vit(3, "tok"), 96), "b": (_vit(2, "gap"), 64)}, "kl", {}),
}


@pytest.mark.parametrize("setup", list(SETUPS))
def test_distill_gradient_matches_oracle(setup):
  """The gradient of every student parameter and the measurements against the float64 oracle; the teachers
  hold no gradient buffer, keep nothing from their forward and are bit-unchanged by the step."""
  from big_vision_b200.trainers.proj.distill import distill as D
  make, kind, kw = SETUPS[setup]
  models, params, fwds, trees, data = _setup(make())
  teachers = tuple(n for n in models if n != "student")
  before = {n: (params[n].flat.clone(), params[n].half.clone()) for n in teachers}
  m = D.loss_and_grads(models, params, _cuda(data), teachers, kind, kw)
  ref_m, ref_g = DO.value_and_grad(fwds, trees, data, teachers, distance=kind, distance_kw=kw)
  assert set(m) == set(ref_m)
  for k, v in ref_m.items():
    assert float(m[k]) == pytest.approx(v, rel=3e-2, abs=1e-4), k
  if len(teachers) == 2:
    assert float(m["distill_loss"]) == pytest.approx(float(m["distill_loss_a"]) + float(m["distill_loss_b"]), rel=1e-6)
  _assert_close(params["student"].numpy_tree("g"), ref_g)
  for n in teachers:
    assert params[n].grad is None
    assert torch.equal(params[n].flat, before[n][0]) and torch.equal(params[n].half, before[n][1])
    _, saved = models[n].fwd(params[n], _cuda(data)[n if n in data else "image"], frozen=True)
    assert all(s is None for s in saved["stages"])


def _config(**kw):
  return dict(optax_name="scale_by_adam", optax=dict(mu_dtype="float32"), lr=1e-3, wd=0.0, grad_clip_norm=1.0,
              schedule=dict(decay_type="linear", warmup_steps=0, linear_end=0.01), teachers=["prof"], **kw)


def test_update_fn_three_adam_steps_with_mixup_track_oracle():
  """make_update_fn with Adam and mixup: image, the teacher's own input and the labels are mixed with ONE
  coefficient, and three steps follow the oracle's trajectory; the teacher is never written."""
  from big_vision_b200 import optax as bv_optax, utils as u
  from big_vision_b200.trainers.proj.distill import distill as D
  models, params, fwds, trees, data = _setup({"student": (_vit(), 64), "prof": (_vit(3, "tok"), 96)})
  P = params["student"]
  config = _config(distance="kl", distance_kw=dict(t=2.0), mixup=dict(p=0.8))
  lr = config["lr"]
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=10, batch_size=4, data_size=1000))
  state = {"params": params, "opt": tx.init(P)}
  fn = D.make_update_fn(models, tx, config)
  with pytest.raises(ValueError, match="rng"):
    fn(state, None, _cuda(data))
  teacher_bits = params["prof"].flat.clone()
  p_ref = {k: v.astype(np.float64) for k, v in trees["student"].items()}
  m_ref = {k: np.zeros_like(v) for k, v in p_ref.items()}
  v_ref = {k: np.zeros_like(v) for k, v in p_ref.items()}
  rng, rng_ref = np.random.default_rng(21), np.random.default_rng(21)
  for step in range(3):
    state, m = fn(state, rng, _cuda(data))
    a32 = np.float32(u.get_mixup(rng_ref, 0.8).a)
    mixed = {k: a32 * v + (np.float32(1) - a32) * np.roll(v, 1, axis=0) for k, v in data.items()}
    ref_m, g = DO.value_and_grad(fwds, {"student": p_ref, "prof": trees["prof"]}, mixed, ("prof",), distance="kl",
                                 distance_kw=dict(t=2.0))
    assert float(m["training_loss"]) == float(m["distill_loss"]) == float(m["distill_loss_prof"])
    for k in ("distill_loss", "entropy_student", "entropy_prof", "task_loss_student", "task_loss_prof"):
      assert float(m[k]) == pytest.approx(ref_m[k], rel=3e-2, abs=1e-4), (step, k)
    gnorm = math.sqrt(sum(float((v ** 2).sum()) for v in g.values()))
    assert float(m["l2_grads"]) == pytest.approx(gnorm, rel=5e-2)
    sched = tx.sched_fns[0](step)
    for k in p_ref:
      p_ref[k], m_ref[k], v_ref[k] = O.adam_reference(p_ref[k], g[k], m_ref[k], v_ref[k], step + 1, lr=lr, b1=0.9,
                                                      b2=0.999, eps=1e-8, wd=0.0, sched=sched, clip=1.0, gnorm=gnorm)
  got = P.numpy_tree("f")
  d_got, d_ref = _flat(got) - _flat(trees["student"]), _flat(p_ref) - _flat(trees["student"])
  cos = float(d_got @ d_ref / (np.linalg.norm(d_got) * np.linalg.norm(d_ref)))
  assert cos > 0.95, cos
  assert np.linalg.norm(d_got) == pytest.approx(np.linalg.norm(d_ref), rel=0.1)
  assert np.abs(_flat(got) - _flat(p_ref)).max() <= 10 * lr
  assert float(m["l2_params"]) == pytest.approx(np.linalg.norm(_flat(got)), rel=1e-3)
  assert torch.equal(params["prof"].flat, teacher_bits)


def test_frozen_student_parameters_get_no_gradient():
  """A schedule entry of None: only the head is trained, the student's body runs forward-only too."""
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.trainers.proj.distill import distill as D
  models, params, _, _, data = _setup({"student": (_vit(), 64), "prof": (_vit(3, "tok"), 96)})
  P = params["student"]
  config = dict(_config(), schedule=[("head/.*", dict(decay_type="cosine", warmup_steps=0)), (".*", None)])
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=10, batch_size=4, data_size=1000))
  before = P.flat.clone()
  D.make_update_fn(models, tx, config)({"params": params, "opt": tx.init(P)}, None, _cuda(data))
  mask = torch.zeros_like(before, dtype=torch.bool)
  for lo, hi in P.trained_ranges(tx.frozen()):
    mask[lo:hi] = True
  assert torch.equal(P.flat[~mask], before[~mask]) and not torch.equal(P.flat[mask], before[mask])
  assert float(P.grad[~mask].abs().max()) == 0.0


def _half_batch_average(models, params, data, n):
  from big_vision_b200.trainers.proj.distill import distill as D
  P = params["student"]
  acc, ms = torch.zeros_like(P.grad), []
  h = n // 2
  for r in range(2):
    ms.append(D.loss_and_grads(models, params, _cuda(data, slice(r * h, (r + 1) * h)), ("prof",), "kl", dict(t=2.0)))
    acc += P.grad
  return acc / 2, {k: (float(ms[0][k]) + float(ms[1][k])) / 2 for k in ms[0]}


def test_per_rank_then_mean_is_the_whole_batch_step():
  """Every row's loss depends on that row alone and each rank scales by 1 / (its rows): the mean of two
  half-batch gradients and measurements is the whole-batch step, up to fp32 summation order."""
  from big_vision_b200.trainers.proj.distill import distill as D
  models, params, _, _, data = _setup({"student": (_vit(), 64), "prof": (_vit(3, "tok"), 96)}, n=8)
  g2, m2 = _half_batch_average(models, params, data, 8)
  m1 = D.loss_and_grads(models, params, _cuda(data), ("prof",), "kl", dict(t=2.0))
  g1 = params["student"].grad
  assert float((g1 - g2).abs().max()) <= 2e-2 * float(g1.abs().max())
  assert float((g1 - g2).norm()) <= 1e-2 * float(g1.norm())
  for k in m1:
    assert float(m1[k]) == pytest.approx(m2[k], rel=1e-3, abs=1e-6), k


def _worker(rank, world, port, ret):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.trainers.proj.distill import distill as D
  import test_distill_gpu as t
  models, params, _, _, data = t._setup({"student": (t._vit(), 64), "prof": (t._vit(3, "tok"), 96)}, n=8)
  P = params["student"]
  config = t._config(distance_kw=dict(t=2.0))
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=100))
  fn = D.make_update_fn(models, tx, config)
  h = 8 // world
  _, m = fn({"params": params, "opt": tx.init(P)}, None, t._cuda(data, slice(rank * h, (rank + 1) * h)))
  torch.cuda.synchronize()
  if rank == 0:
    ret["grad"] = (P.grad / world).cpu().numpy()
    ret["m"] = {k: float(v) for k, v in m.items()}
  dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_nccl_step_is_the_mean_over_ranks():
  import torch.multiprocessing as mp
  ctx = mp.get_context("spawn")
  ret = ctx.Manager().dict()
  port = 29700 + os.getpid() % 150
  procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  models, params, _, _, data = _setup({"student": (_vit(), 64), "prof": (_vit(3, "tok"), 96)}, n=8)
  g1, m1 = _half_batch_average(models, params, data, 8)
  g1, g2 = g1.cpu().numpy(), ret["grad"]
  assert np.abs(g1 - g2).max() <= 2e-2 * np.abs(g1).max()
  assert np.linalg.norm(g1 - g2) <= 1e-2 * np.linalg.norm(g1)
  for k, v in m1.items():
    assert ret["m"][k] == pytest.approx(v, rel=1e-3, abs=1e-6), k
