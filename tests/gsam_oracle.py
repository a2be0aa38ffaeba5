"""TEST INFRASTRUCTURE: the GSAM gradient (big_vision/trainers/proj/gsam/gsam.py:19-122) in float64 on
torch-CPU autograd, over any loss of a parameter tree -- with oracle/bv_oracle.py's model restatements it
is the reference for tests/test_gsam_gpu.py.  Each statement cites the reference line it restates."""
import numpy as np
import torch

F64 = torch.float64


def _grad(loss_fn, params):
  p = {k: torch.tensor(np.asarray(v), dtype=F64, requires_grad=True) for k, v in params.items()}
  loss = loss_fn(p)
  loss.backward()
  return float(loss.detach()), {k: (v.grad.detach() if v.grad is not None else torch.zeros_like(v.detach()))
                                for k, v in p.items()}


def dual_vector(y):
  """gsam.py:19-27: (y / ||y||, ||y||) over the whole tree, no eps."""
  gradient_norm = torch.sqrt(sum(torch.sum(torch.square(e)) for e in y.values()))      # :24-25
  return {k: x / gradient_norm for k, x in y.items()}, gradient_norm                   # :26-27


def gsam_gradient(loss_fn, params, rho_max, rho_min, alpha, lr, lr_max, lr_min, eps=1e-12,
                  adaptive_perturbation=False, minimize_fp=True):
  """gsam.py:29-122.  `loss_fn(tree of float64 tensors) -> scalar`; `params` {name: array}.
  Returns (clean loss, {name: float64 numpy GSAM gradient})."""
  l_clean, g_clean = _grad(loss_fn, params)                                             # :69
  _, g_clean_length = dual_vector(g_clean)                                              # :70
  if lr_max == lr_min:                                                                  # :72-75
    sam_rho = rho_max
  else:
    sam_rho = rho_min + (rho_max - rho_min) * (lr - lr_min) / (lr_max - lr_min)
  w = {k: torch.as_tensor(np.asarray(v), dtype=F64) for k, v in params.items()}
  if adaptive_perturbation:                                                             # :78-80
    param_sam = {k: w[k] + torch.abs(w[k]) * sam_rho * g_clean[k] / (g_clean_length + eps) for k in w}
  else:                                                                                 # :81-83
    param_sam = {k: w[k] + sam_rho * g_clean[k] / (g_clean_length + eps) for k in w}
  _, g_robust = _grad(loss_fn, param_sam)                                               # :86
  if minimize_fp:
    g_robust_normalized, _ = dual_vector(g_robust)                                      # :94
    g_clean_projection_norm = sum(torch.sum(g_robust_normalized[k] * g_clean[k]) for k in w)   # :98-99
    g_clean_residual = {k: g_clean[k] - g_clean_projection_norm * g_robust_normalized[k] for k in w}  # :100-101
    g_gsam = {k: g_robust[k] - g_clean_residual[k] * alpha for k in w}                  # :104-105
  else:
    g_clean_normalized, _ = dual_vector(g_clean)                                        # :108
    g_robust_projection_norm = sum(torch.sum(g_clean_normalized[k] * g_robust[k]) for k in w)  # :112-113
    g_robust_residual = {k: g_robust[k] - g_robust_projection_norm * g_clean_normalized[k] for k in w}  # :114-115
    g_gsam = {k: g_clean[k] + g_robust_residual[k] * alpha for k in w}                  # :118-119
  return l_clean, {k: v.numpy() for k, v in g_gsam.items()}                             # :122
