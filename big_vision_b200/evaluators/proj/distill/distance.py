"""Distance between a student's and a teacher's outputs -- the device arithmetic of
big_vision/evaluators/proj/distill/distance.py: `dist()` (:35-67) over `bv_distance`, the flattening of
:86-88 and the summary of :146-151.  The tf.data loop around it is the caller's."""
import numpy as np
import torch

from big_vision_b200 import ops


def dist(student, teacher, kind, feat_axis=-1, epsilon=1e-12, t=1, ls=0.0, k=1):
  """Distance function used for distillation (distance.py:35-67): reduces `feat_axis` of two fp32 CUDA
  tensors of equal shape.  fp32, int32 for `agree`."""
  if student.shape != teacher.shape:
    raise ValueError(f"student {tuple(student.shape)} and teacher {tuple(teacher.shape)} differ in shape")
  s, u = student.movedim(feat_axis, -1), teacher.movedim(feat_axis, -1)
  lead = s.shape[:-1]
  rows = lambda x: x.reshape(-1, x.shape[-1]).float()
  return ops.distance(rows(s), rows(u), kind, epsilon=epsilon, t=t, ls=ls, k=k).view(lead)


def flatten(x):
  """'b ... -> b (...)' (distance.py:86-88): any non-vector, e.g. a feature map, becomes one."""
  return x.reshape(x.shape[0], -1)


def batch_distances(repr_s, repr_t, distances):
  """The body of _eval_fn (distance.py:86-96): one [b] tensor per entry of `distances`, each a dict of
  dist()'s keyword arguments such as dict(kind="kl", t=2)."""
  repr_s, repr_t = flatten(repr_s), flatten(repr_t)
  return [dist(repr_s, repr_t, **kw) for kw in distances]


def dist_name(kw):
  return "_".join(f"{k}={v}" for k, v in kw.items())           # distance.py:127-129


def summarize(name, batches, masks):
  """distance.py:143-151: the values of the examples whose mask is 1, over all batches, as
  `name/all`, `name/avg`, `name/min`, `name/max`."""
  ds = np.concatenate([np.asarray(torch.as_tensor(d).cpu())[np.asarray(torch.as_tensor(m).cpu()) == 1]
                       for d, m in zip(batches, masks)])
  return {f"{name}/all": ds, f"{name}/avg": np.mean(ds), f"{name}/min": np.min(ds), f"{name}/max": np.max(ds)}
