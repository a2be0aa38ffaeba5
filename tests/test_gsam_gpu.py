"""GPU: the GSAM / SAM kernels (include/bv_b200_sam.h) element by element against float64, and the GSAM
step (trainers/proj/gsam) against the float64 oracle (tests/gsam_oracle.py on oracle/bv_oracle.py's
models): one gradient on a tiny ViT and a tiny stochastic-depth Mixer, three Adam steps, the per-worker
semantics of the reference's pmap, and a 2-rank NCCL step."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import gsam_oracle
from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24               # fp32 unit roundoff
GSAM = dict(rho_max=0.6, rho_min=0.1, alpha=0.6, lr_max=3e-3, lr_min=3e-5)   # vit_i1k_gsam_no_aug.py
SIZES = [1, 3, 7, 4096 + 5, (3 << 20) + 2]     # n = 1, n % 4 != 0, one block, many blocks


def _vec(n, seed, scale=1.0):
  g = torch.Generator().manual_seed(seed)
  return (torch.randn(n, generator=g, dtype=torch.float64) * scale).float()


# ---- kernels ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("adaptive", [False, True])
@pytest.mark.parametrize("n", SIZES)
def test_sam_perturb_elementwise(n, adaptive):
  """w + (rho g)/(sqrt(s) + eps) (adaptive: ((|w| rho) g)/(...)): every operation one fp32 rounding, so
  |out - exact| <= u |exact| + 6u |shift|; the bf16 shadow is bv_cast of the fp32 output, bit for bit."""
  from big_vision_b200 import ops
  w, g = _vec(n, 1), _vec(n, 2, 1e-2)
  gsq = torch.tensor([float((g.double() ** 2).sum())], dtype=torch.float32)
  rho, eps = np.float32(0.43), np.float32(1e-12)
  out, out16 = ops.sam_perturb(w.cuda(), g.cuda(), gsq.cuda(), float(rho), float(eps), adaptive)
  w64, g64 = w.double(), g.double()
  den = math.sqrt(float(gsq[0])) + float(eps)
  shift = (w64.abs() * float(rho) if adaptive else float(rho)) * g64 / den
  ref = w64 + shift
  err = (out.cpu().double() - ref).abs()
  bound = U * ref.abs() + 6 * U * shift.abs() + 1e-45
  assert bool((err <= bound).all()), float((err / bound).max())
  cast = ops.cast(out, torch.empty(n, dtype=torch.bfloat16, device="cuda"))
  assert torch.equal(out16.view(torch.int16), cast.view(torch.int16))


def _chain(n):
  """Longest fp32 addition chain of bv_sam_dots: per-thread float4 terms, the tail, warp and block
  trees, the finishing pass over <= 1024 partials; plus the product's rounding."""
  blocks = min(max((n // 4 + 255) // 256, 1), 1024)
  per_thread = 4 * math.ceil((n // 4) / (blocks * 256)) + 1
  return per_thread + 5 + 3 + math.ceil(blocks / 256) + 8 + 1


@pytest.mark.parametrize("same", [False, True])
@pytest.mark.parametrize("n", SIZES)
def test_sam_dots_elementwise(n, same):
  """(a.b, b.b) within c u sum|terms| of the float64 sums, c the kernel's longest addition chain."""
  from big_vision_b200 import ops
  a, b = _vec(n, 3), _vec(n, 4)
  ad, bd = a.cuda(), b.cuda()
  out = ops.sam_dots(bd if same else ad, bd).cpu().double()
  a64 = b.double() if same else a.double()
  b64 = b.double()
  c = _chain(n)
  for got, terms in ((out[0], a64 * b64), (out[1], b64 * b64)):
    assert abs(float(got) - float(terms.sum())) <= c * U * float(terms.abs().sum()), (n, float(got))


def test_sam_dots_bit_identical_across_runs():
  from big_vision_b200 import ops
  a, b = _vec((5 << 20) + 3, 5).cuda(), _vec((5 << 20) + 3, 6).cuda()
  vals = {tuple(ops.sam_dots(a, b).cpu().view(torch.int32).tolist()) for _ in range(8)}
  assert len(vals) == 1, vals
  vals = {tuple(ops.sam_dots(b, b).cpu().view(torch.int32).tolist()) for _ in range(4)}
  assert len(vals) == 1, vals


@pytest.mark.parametrize("minimize_fp", [True, False])
@pytest.mark.parametrize("n", SIZES)
def test_gsam_combine_elementwise(n, minimize_fp):
  """The combined gradient against float64 evaluated from the kernel's own fp32 scalars: within 8u of
  the sum of the magnitudes of its terms."""
  from big_vision_b200 import ops
  gc, gr = _vec(n, 7), _vec(n, 8) + 0.3 * _vec(n, 7)
  gcd, grd = gc.cuda(), gr.cuda()
  dots = ops.sam_dots(gcd, grd)                  # (g_c . g_r, ||g_r||^2)
  csq = ops.sam_dots(gcd, gcd)                   # ||g_c||^2
  norm_sq = dots[1:2] if minimize_fp else csq[0:1]
  alpha = np.float32(0.6)
  out = ops.gsam_combine(gcd.clone(), grd, dots[0:1], norm_sq, float(alpha), minimize_fp).cpu().double()
  dot, nsq = float(dots[0]), float(norm_sq[0])
  nrm = math.sqrt(nsq)
  c = dot / nrm
  x, y = (gr.double(), gc.double()) if minimize_fp else (gc.double(), gr.double())
  proj = c * x / nrm
  ref = x - float(alpha) * (y - proj) if minimize_fp else x + float(alpha) * (y - proj)
  bound = 8 * U * (x.abs() + float(alpha) * (y.abs() + proj.abs())) + 1e-45
  err = (out - ref).abs()
  assert bool((err <= bound).all()), float((err / bound).max())


def test_gsam_combine_zero_robust_gradient_is_nan():
  """dual_vector has no eps (gsam.py:24-27): a zero g_r gives 0/0, NaN everywhere, as in the reference
  (likewise a zero g_c without minimize_fp)."""
  from big_vision_b200 import ops
  n = 1027
  gc, zero = _vec(n, 9).cuda(), torch.zeros(n, device="cuda")
  dots = ops.sam_dots(gc, zero)
  assert dots.tolist() == [0.0, 0.0]
  out = ops.gsam_combine(gc.clone(), zero, dots[0:1], dots[1:2], 0.6, True)
  assert bool(torch.isnan(out).all())
  csq = ops.sam_dots(zero, zero)
  out = ops.gsam_combine(zero.clone(), gc, dots[0:1], csq[0:1], 0.6, False)
  assert bool(torch.isnan(out).all())


# ---- the step ------------------------------------------------------------------------------------
def _randomize_zero_inits(tree, seed):
  rng = np.random.default_rng(seed)
  return {k: ((rng.standard_normal(v.shape) * 0.05).astype(np.float32) if not np.any(v) else v)
          for k, v in tree.items()}


def _vit():
  from big_vision_b200.models import vit
  model = vit.Model(16, width=64, depth=2, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type="gap",
                    rep_size=False)
  cfg = dict(depth=2, num_heads=1, pool_type="gap", posemb="learn", rep_size=False, num_classes=16)
  return model, lambda p, img, masks=None: O.vit_forward(p, img, cfg, "float32")


def _mixer():
  from big_vision_b200.models import mlp_mixer
  model = mlp_mixer.Model(16, patch_size=(16, 16), num_blocks=3, hidden_dim=64, tokens_mlp_dim=32,
                          channels_mlp_dim=128, stoch_depth=0.5)
  cfg = dict(num_blocks=3, num_classes=16)
  return model, lambda p, img, masks=None: O.mixer_forward(p, img, cfg, "float32", masks=masks)


def _setup(model, shape, seed=0):
  P = model.init(seed, shape, device="cuda")
  tree = _randomize_zero_inits(P.numpy_tree("f"), seed + 1)
  P.load_tree(tree)
  rng = np.random.default_rng(seed + 2)
  image = rng.uniform(-1, 1, size=shape).astype(np.float32)
  labels = np.eye(16, dtype=np.float32)[rng.integers(0, 16, size=shape[0])]
  return P, tree, image, labels


def _oracle(fwd, tree, image, labels, masks=None, **kw):
  img, lab = torch.from_numpy(image), torch.from_numpy(labels).double()
  return gsam_oracle.gsam_gradient(lambda p: O.sigmoid_xent(fwd(p, img, masks), lab), tree, **kw)


def _assert_close(grads, ref):
  gmax = max(float(np.abs(v).max()) for v in ref.values())
  bad = {}
  for k, g in grads.items():
    err = float(np.abs(g.astype(np.float64) - ref[k]).max())
    tol = 6e-2 * float(np.abs(ref[k]).max()) + 3e-3 * gmax
    if err > tol:
      bad[k] = (err, tol)
  assert not bad, sorted(bad.items(), key=lambda kv: -kv[1][0])[:8]


def _flat(tree):
  return np.concatenate([np.asarray(tree[k], dtype=np.float64).ravel() for k in sorted(tree)])


@pytest.mark.parametrize("arch", ["vit", "mixer"])
def test_gsam_gradient_matches_oracle(arch):
  """One GSAM gradient (config values, lr between lr_min and lr_max) against the float64 oracle; the Mixer
  with stochastic depth and the same given masks in both passes and in the oracle."""
  from big_vision_b200.trainers.proj.gsam import gsam as G
  model, fwd = _vit() if arch == "vit" else _mixer()
  P, tree, image, labels = _setup(model, (4, 64, 64, 3))
  masks = None
  kw = {}
  if arch == "mixer":
    masks = np.array([[[1, 1, 1, 1], [1, 1, 1, 1]], [[1, 0, 1, 1], [0, 1, 1, 0]], [[0, 0, 1, 1], [1, 0, 1, 0]]],
                     dtype=np.float32)
    kw["masks"] = torch.from_numpy(masks).cuda()
  loss = G.gsam_gradient(model, P, torch.from_numpy(image).cuda(), torch.from_numpy(labels).cuda(), lr=2e-3,
                         **GSAM, **kw)
  ref_loss, ref = _oracle(fwd, tree, image, labels, masks, lr=2e-3, **GSAM)
  assert float(loss) == pytest.approx(ref_loss, rel=2e-2)
  _assert_close(P.numpy_tree("g"), ref)
  # the step really is GSAM: far from the plain gradient
  _, plain = _oracle(fwd, tree, image, labels, masks, lr=2e-3, **{**GSAM, "rho_max": 0.0, "rho_min": 0.0,
                                                                 "alpha": 0.0})
  assert np.linalg.norm(_flat(ref) - _flat(plain)) > 0.05 * np.linalg.norm(_flat(plain))


def test_gsam_alpha_zero_is_the_robust_gradient():
  """alpha = 0: P.grad is bit-equal to the robust pass's gradient -- the SAM step.  The robust pass ran on
  weights at distance rho from w, with their bf16 shadow bit-equal to bv_cast of the fp32 weights."""
  from big_vision_b200 import ops
  from big_vision_b200.trainers.proj.gsam import gsam as G
  model, _ = _vit()
  P, _, image, labels = _setup(model, (4, 64, 64, 3))
  T = P.twin()
  G.gsam_gradient(model, P, torch.from_numpy(image).cuda(), torch.from_numpy(labels).cuda(), lr=1.0, P_sam=T,
                  rho_max=0.05, rho_min=0.05, alpha=0.0, lr_max=1.0, lr_min=1.0)
  assert torch.equal(P.grad, T.grad)
  assert bool(torch.isfinite(P.grad).all()) and float(P.grad.abs().max()) > 0
  assert float((T.flat.double() - P.flat.double()).norm()) == pytest.approx(0.05, rel=1e-4)
  cast = ops.cast(T.flat, torch.empty_like(T.half))
  assert torch.equal(cast.view(torch.int16), T.half.view(torch.int16))


def test_update_fn_three_adam_steps_track_oracle():
  """make_update_fn with Adam: three steps follow the oracle's GSAM + Adam trajectory, rho follows the
  optimizer's schedule, and the reported loss is the clean loss."""
  from big_vision_b200 import optax as bv_optax, train
  from big_vision_b200.trainers.proj.gsam import train as gtrain
  model, fwd = _vit()
  P, tree, image, labels = _setup(model, (4, 64, 64, 3))
  lr = 1e-3
  config = dict(optax_name="scale_by_adam", optax=dict(mu_dtype="float32"), lr=lr, wd=0.0, grad_clip_norm=1.0,
                loss="sigmoid_xent", schedule=dict(decay_type="linear", warmup_steps=0, linear_end=0.01),
                gsam=dict(GSAM, lr_max=lr, lr_min=0.01 * lr))
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=10, batch_size=4, data_size=1000))
  state = {"params": P, "opt": tx.init(P)}
  fn = gtrain.make_update_fn(model, tx, config)
  batch = {"image": torch.from_numpy(image).cuda(), "labels": torch.from_numpy(labels).cuda()}
  p_ref = {k: v.astype(np.float64) for k, v in tree.items()}
  m_ref = {k: np.zeros_like(v) for k, v in p_ref.items()}
  v_ref = {k: np.zeros_like(v) for k, v in p_ref.items()}
  for step in range(3):
    clean, _ = train.loss_and_grads(model, P, batch["image"], batch["labels"])
    clean = float(clean)
    state, m = fn(state, None, batch)
    assert float(m["training_loss"]) == pytest.approx(clean, rel=1e-6)
    sched = tx.sched_fns[0](step)
    ref_loss, g = _oracle(fwd, p_ref, image, labels, lr=sched * lr, **config["gsam"])
    assert float(m["training_loss"]) == pytest.approx(ref_loss, rel=2e-2)
    gnorm = math.sqrt(sum(float((v ** 2).sum()) for v in g.values()))
    assert float(m["l2_grads"]) == pytest.approx(gnorm, rel=5e-2)
    for k in p_ref:
      p_ref[k], m_ref[k], v_ref[k] = O.adam_reference(p_ref[k], g[k], m_ref[k], v_ref[k], step + 1, lr=lr, b1=0.9,
                                                      b2=0.999, eps=1e-8, wd=0.0, sched=sched, clip=1.0, gnorm=gnorm)
  got = P.numpy_tree("f")
  d_got, d_ref = _flat(got) - _flat(tree), _flat(p_ref) - _flat(tree)
  cos = float(d_got @ d_ref / (np.linalg.norm(d_got) * np.linalg.norm(d_ref)))
  assert cos > 0.95, cos
  assert np.linalg.norm(d_got) == pytest.approx(np.linalg.norm(d_ref), rel=0.1)
  assert np.abs(_flat(got) - _flat(p_ref)).max() <= 10 * lr


def _half_batch_average(model, P, image, labels, kw):
  from big_vision_b200.trainers.proj.gsam import gsam as G
  acc = torch.zeros_like(P.grad)
  h = image.shape[0] // 2
  for r in range(2):
    G.gsam_gradient(model, P, torch.from_numpy(image[r * h:(r + 1) * h]).cuda(),
                    torch.from_numpy(labels[r * h:(r + 1) * h]).cuda(), **kw)
    acc += P.grad
  P.grad.copy_(acc / 2)
  return P.numpy_tree("g")


def test_per_worker_gsam_then_mean():
  """gsam.py:63-64 / train.py:209-211: each worker perturbs by its OWN clean gradient and the combined
  gradients are averaged.  Two half-batch gradients, averaged, match the oracle's per-worker average and
  differ from the whole-batch GSAM gradient."""
  model, fwd = _vit()
  P, tree, image, labels = _setup(model, (8, 64, 64, 3))
  kw = dict(lr=2e-3, **GSAM)
  got = _half_batch_average(model, P, image, labels, kw)
  halves = [_oracle(fwd, tree, image[r * 4:(r + 1) * 4], labels[r * 4:(r + 1) * 4], **kw)[1] for r in range(2)]
  ref = {k: 0.5 * (halves[0][k] + halves[1][k]) for k in halves[0]}
  _assert_close(got, ref)
  _, whole = _oracle(fwd, tree, image, labels, **kw)
  err = np.linalg.norm(_flat(got) - _flat(ref))
  assert np.linalg.norm(_flat(whole) - _flat(ref)) > 5 * err


def _worker(rank, world, port, ret):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.trainers.proj.gsam import train as gtrain
  import test_gsam_gpu as t
  model, _ = t._vit()
  P, _, image, labels = t._setup(model, (8, 64, 64, 3))
  config = dict(optax_name="scale_by_adam", lr=2e-3, schedule=dict(decay_type="cosine", warmup_steps=0),
                gsam=dict(t.GSAM))
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=100))
  fn = gtrain.make_update_fn(model, tx, config)
  h = image.shape[0] // world
  fn({"params": P, "opt": tx.init(P)}, None, {"image": torch.from_numpy(image[rank * h:(rank + 1) * h]).cuda(),
                                              "labels": torch.from_numpy(labels[rank * h:(rank + 1) * h]).cuda()})
  torch.cuda.synchronize()
  if rank == 0:
    ret["grad"] = (P.grad / world).cpu().numpy()
    ret["lr"] = tx.sched_fns[0](0) * 2e-3
  dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_nccl_step_is_the_per_worker_average():
  import torch.multiprocessing as mp
  ctx = mp.get_context("spawn")
  ret = ctx.Manager().dict()
  port = 29500 + os.getpid() % 150
  procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  model, _ = _vit()
  P, _, image, labels = _setup(model, (8, 64, 64, 3))
  _half_batch_average(model, P, image, labels, dict(lr=ret["lr"], **GSAM))
  g1, g2 = P.grad.cpu().numpy(), ret["grad"]
  # the same kernels on the same rows; only the order of fp32 atomics differs
  assert np.abs(g1 - g2).max() <= 2e-2 * np.abs(g1).max()
  assert np.linalg.norm(g1 - g2) <= 1e-2 * np.linalg.norm(g1)
