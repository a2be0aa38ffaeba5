"""Surrogate-gap sharpness-aware minimisation (GSAM, arXiv 2203.08065) -- mirror of
big_vision/trainers/proj/gsam/gsam.py:19-122 on the flat parameter buffers.

  g_c      = grad(loss)(w)                         pass 1, this worker's shard, no all-reduce
  rho      = rho_max, or linear in lr between (lr_min, rho_min) and (lr_max, rho_max)
  w_sam    = w + rho * g_c / (||g_c|| + eps)       (* |w| with adaptive_perturbation)
  g_r      = grad(loss)(w_sam)                     pass 2, same batch, same stochastic-depth masks
  g        = g_r - alpha * (g_c - c * g_r/||g_r||),  c = (g_r/||g_r||) . g_c       (minimize_fp)
           = g_c + alpha * (g_r - c * g_c/||g_c||),  c = (g_c/||g_c||) . g_r       (otherwise)

The vector algebra is three kinds of bandwidth-bound kernels (include/bv_b200_sam.h): bv_sam_dots for
||g_c||^2 and for (g_c . g_r, ||g_r||^2), bv_sam_perturb for w_sam and its bf16 shadow, and
bv_gsam_combine in place over g_c.  The norms and the dot product stay on the device: the step never
waits for the host.  rho_max == rho_min and alpha = 0 is plain SAM.
"""
import torch

from big_vision_b200 import ops

GSAM_KEYS = ("rho_max", "rho_min", "alpha", "lr_max", "lr_min", "eps", "adaptive_perturbation", "minimize_fp")


def sam_rho(lr, rho_max, rho_min, lr_max, lr_min):
  """gsam.py:72-75: the perturbation radius at learning rate `lr`."""
  if lr_max == lr_min:
    return rho_max
  return rho_min + (rho_max - rho_min) * (lr - lr_min) / (lr_max - lr_min)


def parse_config(gsam):
  """`config.gsam` -> keyword arguments of gsam_gradient (without `lr`).  The reference passes the dict
  through as `**config.gsam` (train.py:209-210), so a key gsam_gradient does not take is an error."""
  kw = dict(gsam or {})
  unknown = sorted(set(kw) - set(GSAM_KEYS))
  if unknown:
    raise TypeError(f"config.gsam: unknown keys {unknown}")
  missing = [k for k in ("rho_max", "rho_min", "alpha", "lr_max", "lr_min") if k not in kw]
  if missing:
    raise TypeError(f"config.gsam: missing {missing}")
  out = {k: float(kw[k]) for k in ("rho_max", "rho_min", "alpha", "lr_max", "lr_min")}
  out["eps"] = float(kw.get("eps", 1e-12))
  out["adaptive_perturbation"] = bool(kw.get("adaptive_perturbation", False))
  out["minimize_fp"] = bool(kw.get("minimize_fp", True))
  return out


def gsam_gradient(model, P, images, labels, *, rho_max, rho_min, alpha, lr, lr_max, lr_min, eps=1e-12,
                  adaptive_perturbation=False, minimize_fp=True, loss_name="sigmoid_xent", P_sam=None, **fwd_kw):
  """gsam.py:29-122 on this worker's shard: leaves the (local, not averaged) GSAM gradient in P.grad and
  returns the clean loss, a device tensor [1].  `P_sam` (P.twin(), allocated here if None) receives the
  perturbed weights and the robust gradient g_r.  `fwd_kw` goes to both forwards: give explicit
  stochastic-depth `masks`, so that both passes drop the same residual branches."""
  from big_vision_b200 import train
  if P_sam is None:
    P_sam = P.twin()
  sc = torch.empty(4, dtype=torch.float32, device=P.grad.device)   # ||g_c||^2 (twice), g_c . g_r, ||g_r||^2
  ws = torch.empty(ops.L.SAM_WS_FLOATS, dtype=torch.float32, device=P.grad.device)
  # gsam.py:69-70: value and gradient at w, and the gradient's norm
  loss, _ = train.loss_and_grads(model, P, images, labels, loss_name, **fwd_kw)
  ops.sam_dots(P.grad, P.grad, out=sc[0:2], ws=ws)
  # gsam.py:72-83: the perturbed weights and their bf16 shadow
  rho = sam_rho(lr, rho_max, rho_min, lr_max, lr_min)
  ops.sam_perturb(P.flat, P.grad, sc[0:1], rho, eps, adaptive_perturbation, out=P_sam.flat, out_bf16=P_sam.half)
  # gsam.py:86: the gradient at w_sam (pass 1's saved activations are gone: loss_and_grads kept none)
  train.loss_and_grads(model, P_sam, images, labels, loss_name, **fwd_kw)
  # gsam.py:92-119
  ops.sam_dots(P.grad, P_sam.grad, out=sc[2:4], ws=ws)
  ops.gsam_combine(P.grad, P_sam.grad, sc[2:3], sc[3:4] if minimize_fp else sc[0:1], alpha, minimize_fp)
  return loss
