"""CPU: the GSAM / SAM step (trainers/proj/gsam) -- its float64 oracle against a direct transcription of
the reference's tree-map formulas, the rho schedule, config parsing, the refusal of frozen parameters, and the
refusal of CPU tensors by the SAM ops."""
import os

import numpy as np
import pytest
import torch

import gsam_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- a random tree and a loss with a closed-form gradient ----------------------------------------
def _tree(seed):
  rng = np.random.default_rng(seed)
  shapes = {"a/kernel": (5, 7), "a/bias": (7,), "b/scale": (3,), "c": (2, 3, 4)}
  params = {k: rng.standard_normal(s) for k, s in shapes.items()}
  coef = {k: rng.uniform(0.5, 2.0, s) for k, s in shapes.items()}
  return params, coef


def _loss_fn(coef):
  """sum_k sum(c_k * p_k^2 / 2 + sin(p_k)) in torch, for the oracle's autograd."""
  return lambda p: sum(torch.sum(torch.as_tensor(coef[k]) * p[k] ** 2 / 2 + torch.sin(p[k])) for k in p)


def _grad_np(coef):
  return lambda p: {k: coef[k] * p[k] + np.cos(p[k]) for k in p}


def _transcription(grad, params, rho_max, rho_min, alpha, lr, lr_max, lr_min, eps=1e-12,
                   adaptive_perturbation=False, minimize_fp=True):
  """gsam.py:69-119 written with numpy tree maps, independently of the oracle."""
  tree_map = lambda f, *ts: {k: f(*(t[k] for t in ts)) for k in ts[0]}
  leaves = lambda t: [t[k] for k in sorted(t)]

  def dual_vector(y):
    n = np.sqrt(sum(np.sum(np.square(e)) for e in leaves(y)))
    return tree_map(lambda x: x / n, y), n

  g_clean = grad(params)
  _, g_clean_length = dual_vector(g_clean)
  sam_rho = rho_max if lr_max == lr_min else rho_min + (rho_max - rho_min) * (lr - lr_min) / (lr_max - lr_min)
  if adaptive_perturbation:
    param_sam = tree_map(lambda a, b: a + np.abs(a) * sam_rho * b / (g_clean_length + eps), params, g_clean)
  else:
    param_sam = tree_map(lambda a, b: a + sam_rho * b / (g_clean_length + eps), params, g_clean)
  g_robust = grad(param_sam)
  if minimize_fp:
    g_robust_normalized, _ = dual_vector(g_robust)
    proj = sum(np.vdot(p, q) for p, q in zip(leaves(g_robust_normalized), leaves(g_clean)))
    residual = tree_map(lambda a, b: a - proj * b, g_clean, g_robust_normalized)
    return tree_map(lambda a, b: a - b * alpha, g_robust, residual)
  g_clean_normalized, _ = dual_vector(g_clean)
  proj = sum(np.vdot(p, q) for p, q in zip(leaves(g_clean_normalized), leaves(g_robust)))
  residual = tree_map(lambda a, b: a - proj * b, g_robust, g_clean_normalized)
  return tree_map(lambda a, b: a + b * alpha, g_clean, residual)


@pytest.mark.parametrize("adaptive", [False, True])
@pytest.mark.parametrize("minimize_fp", [True, False])
def test_oracle_equals_the_reference_formulas(adaptive, minimize_fp):
  params, coef = _tree(1)
  kw = dict(rho_max=0.6, rho_min=0.1, alpha=0.6, lr=2e-3, lr_max=3e-3, lr_min=3e-5,
            adaptive_perturbation=adaptive, minimize_fp=minimize_fp)
  loss, g = gsam_oracle.gsam_gradient(_loss_fn(coef), params, **kw)
  ref = _transcription(_grad_np(coef), params, **kw)
  assert loss == pytest.approx(float(_loss_fn(coef)({k: torch.as_tensor(v) for k, v in params.items()})), rel=1e-14)
  for k in params:
    np.testing.assert_allclose(g[k], ref[k], rtol=1e-12, atol=1e-13)
  # the four variants are different functions of the same inputs
  other = _transcription(_grad_np(coef), params, **{**kw, "minimize_fp": not minimize_fp})
  assert max(np.abs(g[k] - other[k]).max() for k in params) > 1e-3


def test_alpha_zero_with_constant_rho_is_sam():
  """gsam.py:67 note: rho_max == rho_min, alpha = 0 -> the SAM gradient grad(L)(w + rho g / ||g||)."""
  params, coef = _tree(2)
  grad = _grad_np(coef)
  _, g = gsam_oracle.gsam_gradient(_loss_fn(coef), params, rho_max=0.05, rho_min=0.05, alpha=0.0, lr=1.0,
                                   lr_max=2.0, lr_min=0.5)
  gc = grad(params)
  norm = np.sqrt(sum(np.sum(v ** 2) for v in gc.values()))
  sam = grad({k: params[k] + 0.05 * gc[k] / (norm + 1e-12) for k in params})
  for k in params:
    np.testing.assert_allclose(g[k], sam[k], rtol=1e-13, atol=1e-14)


def test_rho_schedule():
  from big_vision_b200.trainers.proj.gsam import gsam as G
  kw = dict(rho_max=0.6, rho_min=0.1, lr_max=3e-3, lr_min=3e-5)
  assert G.sam_rho(3e-3, **kw) == pytest.approx(0.6, rel=1e-12)
  assert G.sam_rho(3e-5, **kw) == pytest.approx(0.1, rel=1e-12)
  assert G.sam_rho(0.5 * (3e-3 + 3e-5), **kw) == pytest.approx(0.35, rel=1e-12)
  # lr_max == lr_min: rho_max whatever the learning rate
  assert G.sam_rho(7.0, rho_max=0.6, rho_min=0.1, lr_max=1e-3, lr_min=1e-3) == 0.6


def test_config_gsam_is_parsed():
  """configs/proj/gsam/vit_i1k_gsam_no_aug.py's dict (lr_max = lr, lr_min = linear_end * lr) and the defaults
  of gsam.py:29-31; anything gsam_gradient does not take is an error, as `**config.gsam` would be."""
  from big_vision_b200.trainers.proj.gsam import gsam as G
  kw = G.parse_config(dict(rho_max=0.6, rho_min=0.1, alpha=0.6, lr_max=0.003, lr_min=0.01 * 0.003))
  assert kw == dict(rho_max=0.6, rho_min=0.1, alpha=0.6, lr_max=0.003, lr_min=3e-5, eps=1e-12,
                    adaptive_perturbation=False, minimize_fp=True)
  kw = G.parse_config(dict(rho_max=1, rho_min=1, alpha=0, lr_max=1, lr_min=1, eps=1e-6,
                           adaptive_perturbation=True, minimize_fp=False))
  assert kw["adaptive_perturbation"] and not kw["minimize_fp"] and kw["eps"] == 1e-6
  with pytest.raises(TypeError, match="unknown"):
    G.parse_config(dict(rho_max=0.6, rho_min=0.1, alpha=0.6, lr_max=1, lr_min=0, rho=0.1))
  with pytest.raises(TypeError, match="missing"):
    G.parse_config(dict(rho_max=0.6))


def _tiny_vit_tx(schedule):
  from big_vision_b200 import engine as E
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.models import vit
  model = vit.Model(10, width=64, depth=2, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type="gap")
  specs, aliases = model.specs((32, 32), 3)
  P = E.FlatParams(specs, aliases, "cpu")
  tx, _ = bv_optax.make(dict(lr=1e-3, schedule=schedule), P, sched_kw=dict(total_steps=10))
  return model, P, tx


def test_frozen_schedule_is_refused():
  from big_vision_b200.trainers.proj.gsam import train as gtrain
  gsam = dict(rho_max=0.6, rho_min=0.1, alpha=0.6, lr_max=1e-3, lr_min=1e-5)
  model, _, tx = _tiny_vit_tx([("head/.*", dict(decay_type="cosine")), (".*", None)])
  with pytest.raises(NotImplementedError, match="frozen"):
    gtrain.make_update_fn(model, tx, dict(gsam=gsam))
  model, _, tx = _tiny_vit_tx(dict(decay_type="cosine"))
  assert callable(gtrain.make_update_fn(model, tx, dict(gsam=gsam)))


def test_twin_params_share_the_layout():
  _, P, _ = _tiny_vit_tx(dict(decay_type="cosine"))
  T = P.twin()
  assert T.offsets is P.offsets and T.total == P.total and T.n_decay == P.n_decay
  assert T.flat.data_ptr() != P.flat.data_ptr() and T.grad.data_ptr() != P.grad.data_ptr()
  assert T.half.dtype == torch.bfloat16 and T.half.numel() == P.total
  P.flat.fill_(1.0)
  assert float(T.flat.abs().sum()) == 0.0
  assert set(T.tree("f")) == set(P.tree("f"))


def test_sam_ops_refuse_cpu_tensors():
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  x = torch.zeros(8)
  with pytest.raises(L.BvError):
    ops.sam_dots(x, x, out=torch.zeros(2), ws=torch.zeros(L.SAM_WS_FLOATS))
  with pytest.raises(L.BvError):
    ops.sam_perturb(x, x, torch.ones(1), 0.1, out=x.clone(), out_bf16=torch.zeros(8, dtype=torch.bfloat16))
  with pytest.raises(L.BvError):
    ops.gsam_combine(x, x, torch.ones(1), torch.ones(1), 0.5)
