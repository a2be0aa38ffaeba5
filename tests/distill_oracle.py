"""TEST INFRASTRUCTURE: distillation in float64 on torch-CPU autograd -- `dist()`
(big_vision/evaluators/proj/distill/distance.py:35-67), the distill `loss_fn`
(big_vision/trainers/proj/distill/distill.py:217-248) and the gradient of one update step (:270-272).  With
oracle/bv_oracle.py's model restatements it is the reference for tests/test_distill_gpu.py.  Each statement
cites the reference line it restates."""
import numpy as np
import torch

F64 = torch.float64


def softmax_xent(logits, labels, kl=False):
  """utils.py:276-281 with reduction=False, axis=-1."""
  log_p = torch.log_softmax(logits, -1)                                                   # :277
  nll = -torch.sum(labels * log_p, -1)                                                    # :278
  if kl:
    nll = nll + torch.sum(labels * torch.log(torch.clamp(labels, min=1e-8)), -1)          # :279-280
  return nll


def top_k_indices(x, k):
  """jax.lax.top_k's indices: descending values, the lower index first among equal values."""
  return torch.sort(x, dim=-1, descending=True, stable=True).indices[..., :k]


def dist(student, teacher, kind, epsilon=1e-12, t=1, ls=0.0, k=1):
  """distance.py:35-67 over the last axis of float64 tensors."""
  student, teacher = torch.as_tensor(student, dtype=F64), torch.as_tensor(teacher, dtype=F64)
  diff = student - teacher                                                                # :38
  if kind == "euclidean":
    return torch.sqrt(torch.sum(diff * diff, -1) + epsilon)                               # :40
  if kind == "l2":
    return torch.sum(diff * diff, -1)                                                     # :42
  if kind == "hard":
    # :44-45; torch.argmax does not promise the first maximum, so take it from a stable sort
    pseudolabels = top_k_indices(teacher, 1)[..., 0]
    pl = torch.nn.functional.one_hot(pseudolabels, teacher.shape[-1]).to(F64)
    if ls:
      pl = (1.0 - ls) * pl + (ls / (pl.shape[-1] - 1)) * (1.0 - pl)                       # :46-47
    return softmax_xent(student, pl, kl=True)                                             # :48-49
  if kind == "kl":
    return t ** 2 * softmax_xent(student / t, torch.softmax(teacher / t, -1), kl=True)    # :51-54
  if kind == "logsoftmax_euclidean":
    d = torch.log_softmax(student, -1) - torch.log_softmax(teacher, -1)                   # :56-58
    return torch.sqrt(torch.sum(d * d, -1) + epsilon)                                     # :59-60
  if kind == "agree":
    return (top_k_indices(student, k) == top_k_indices(teacher, 1)).sum(-1)               # :62-65
  raise AssertionError(f"Unknown kind of distance {kind}.")                               # :67


def loss_fn(logits, teachers, labels=None, distance="kl", distance_kw=None):
  """distill.py:230-248 from the models' logits {name: [n, C]} (with "student"): (distill_loss,
  measurements), every entry a batch mean."""
  measurements = {}
  for name, lg in logits.items():
    measurements[f"entropy_{name}"] = -torch.sum(torch.log_softmax(lg, -1) * torch.softmax(lg, -1), -1)   # :232-233
    if labels is not None:
      measurements[f"task_loss_{name}"] = softmax_xent(lg, labels)                        # :235-236
  measurements["distill_loss"] = 0.0                                                      # :240
  for name in teachers:
    l = dist(logits["student"], logits[name], distance, **(distance_kw or {}))            # :242-243
    measurements[f"distill_loss_{name}"] = l
    measurements["distill_loss"] = measurements["distill_loss"] + l                       # :245
  measurements = {k: v.mean() for k, v in measurements.items()}                           # :248
  return measurements["distill_loss"], measurements


def value_and_grad(fwds, trees, data, teachers, **kw):
  """distill.py:270-272: the gradient of the mean distill_loss with respect to the student's parameters.
  fwds {name: fn(tree of float64 tensors, image) -> logits}, trees {name: {param: array}}; every model
  sees data[name] if present, else data["image"] (:225).
  Returns (measurements as floats, {param: float64 numpy gradient})."""
  p = {n: {k: torch.tensor(np.asarray(v), dtype=F64, requires_grad=n == "student") for k, v in tree.items()}
       for n, tree in trees.items()}
  logits = {n: fwds[n](p[n], torch.as_tensor(data.get(n, data["image"]))) for n in ("student",) + tuple(teachers)}
  labels = torch.as_tensor(data["labels"], dtype=F64) if "labels" in data else None
  loss, m = loss_fn(logits, teachers, labels, **kw)
  loss.backward()
  grads = {k: (v.grad.numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in p["student"].items()}
  return {k: float(v.detach()) for k, v in m.items()}, grads
