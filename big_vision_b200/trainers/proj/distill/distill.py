"""Distillation training step -- mirror of `loss_fn` / `update_fn` in
big_vision/trainers/proj/distill/distill.py:217-285 ("Knowledge distillation: a good teacher is patient and
consistent"; configs/proj/distill/*.py, configs/proj/flexivit/i1k_deit3_distill.py):

  mixup of image, labels and every model-named input with ONE coefficient (per rank, as train.py)
  ->  each teacher's forward, frozen: nothing is saved, and its activations are gone before the student runs
  ->  student forward  ->  bv_distill_loss once per teacher (distance, gradient, measurements)
  ->  student backward with train.py's gradient all-reduce  ->  tx.update

Only the student's parameters are optimised (`tx` is made from them, distill.py:206-211); a teacher is
never written and needs no gradient buffer (FlatParams.drop_grad).  `train_state["params"]` is
{"student": P, <teacher>: P, ...}.  Built distances: `kl` (every shipped config) and `hard`.
"""
import torch

from big_vision_b200 import lib as L
from big_vision_b200 import ops
from big_vision_b200 import train
from big_vision_b200.trainers.proj.image_text.siglip import Dist

TRAINED_KINDS = ("kl", "hard")


def getfirst(d, *keys):
  """d[k] of the first k in d (distill.py:62-66): a model's own input under its name, else "image"."""
  for k in keys:
    if k in d:
      return d[k]
  raise KeyError(f"none of {keys} in {sorted(d)}")


def parse_config(config, models):
  """-> (teachers, kind, distance_kw) of distill.py:241-243, checked against `models`."""
  teachers = tuple(config["teachers"])
  if not teachers:
    raise ValueError("config.teachers is empty")
  missing = [n for n in ("student",) + teachers if n not in models]
  if missing or "student" in teachers:
    raise ValueError(f"models must hold 'student' and every teacher of {teachers}; missing {missing}")
  kind = config.get("distance", "kl")
  if kind not in L.DIST_KINDS:
    raise ValueError(f"Unknown kind of distance {kind}.")
  if kind not in TRAINED_KINDS:
    raise NotImplementedError(f"training with distance '{kind}': the fused loss / gradient kernel is built for "
                              f"{' and '.join(TRAINED_KINDS)}")
  kw = dict(config.get("distance_kw") or {})
  unknown = sorted(set(kw) - {"t", "ls"})
  if unknown:
    raise TypeError(f"distance_kw: '{kind}' takes t and ls, got unknown {unknown}")
  return teachers, kind, kw


def loss_and_grads(models, params, data, teachers, kind="kl", distance_kw=None, dist_view=None, frozen=None,
                   **student_kw):
  """value_and_grad(loss_fn)(student params) of distill.py:217-248, 270-272 on this rank's shard.
  params["student"].grad holds the LOCAL gradient of the LOCAL-mean distill_loss (the sum over teachers).
  Returns the measurements of :230-248 as 0-d device tensors (local means)."""
  logits, outs = {}, {}
  for name in teachers:
    # frozen=True: forward only, every activation freed once consumed, nothing kept for a backward
    logits[name], saved = models[name].fwd(params[name], getfirst(data, name, "image"), frozen=True)
    del saved
  labels = data.get("labels")

  def loss_grad(flat, ld):
    dl = None
    lab = labels.reshape(flat.shape) if labels is not None else None
    for name in teachers:          # distill_loss is the sum over teachers (:240-245): gradients add up
      outs[name], _, dl = ops.distill_loss(flat, logits[name].reshape(flat.shape), lab, kind, dlogits=dl,
                                           dlogits_cols=ld, **(distance_kw or {}))
    return dl

  train.fwd_loss_bwd(models["student"], params["student"], getfirst(data, "student", "image"), loss_grad,
                     dist_view, frozen, **student_kw)
  idx = {k: i for i, k in enumerate(L.DISTILL_OUTPUTS)}
  m = {"entropy_student": outs[teachers[0]][idx["entropy_student"]]}
  for name in teachers:
    m[f"distill_loss_{name}"] = outs[name][idx["distance"]]
    m[f"entropy_{name}"] = outs[name][idx["entropy_teacher"]]
  if labels is not None:
    m["task_loss_student"] = outs[teachers[0]][idx["task_loss_student"]]
    for name in teachers:
      m[f"task_loss_{name}"] = outs[name][idx["task_loss_teacher"]]
  m["distill_loss"] = torch.stack([m[f"distill_loss_{name}"] for name in teachers]).sum()
  return m


def make_update_fn(models, tx, config):
  """models: {"student": model, <teacher>: model, ...}; tx: the optimizer of the student's parameters."""
  teachers, kind, distance_kw = parse_config(config, models)
  mixup_p = (config.get("mixup") or {}).get("p")
  d = Dist()
  frozen = tx.frozen() if hasattr(tx, "frozen") else frozenset()
  student = models["student"]

  def update_fn(train_state, rng, batch):
    params, opt = train_state["params"], train_state["opt"]
    P = params["student"]
    data = dict(batch)
    if mixup_p:                                               # distill.py:256-261
      from big_vision_b200 import utils as u
      if rng is None:
        raise ValueError("mixup needs an rng (numpy Generator)")
      to_mix = {name: data[name] for name in ("image", "labels") + tuple(models) if name in data}
      rng, _, to_mix = u.get_mixup(rng, mixup_p)(**to_mix)
      data.update(to_mix)
    # stochastic depth for the student only (`train=name == "student"`, distill.py:226)
    kw = dict(train=True, rng=rng) if getattr(student, "stoch_depth", 0.0) else {}
    m = loss_and_grads(models, params, data, teachers, kind, distance_kw, dist_view=d, frozen=frozen, **kw)
    # every measurement is the mean over the GLOBAL batch: sum the per-rank means and divide by world
    names = sorted(m)
    vals = torch.stack([m[k] for k in names])
    d.all_reduce_sum(vals)
    vals = vals / d.world
    sc = tx.update(P, opt, grad_mult=1.0 / d.world)
    measurements = dict(zip(names, vals.unbind()))
    measurements.update({
        "training_loss": measurements["distill_loss"],
        "l2_grads": sc[0].sqrt() / d.world,
        "l2_params": sc[2].sqrt(),
        "l2_updates": sc[1].sqrt(),
    })
    return train_state, measurements

  return update_fn


def make_predict_fns(models, config):
  """The predict functions of distill.py:338-359, over train_state["params"] = {name: P}:
  `<name>_fwd` per model, `teacher_ensemble_fwd` (the mean of the teachers' softmaxes) and
  `student_<teacher>_fwd` / `student_teacher_ensemble_fwd` pairs for the distance evaluator."""
  teachers = tuple(config["teachers"])
  fns = {}
  for name, model in models.items():
    def fwd(train_state, batch, n=name, m=model):
      return m.apply({"params": train_state["params"][n]}, batch["image"])
    fns[f"{name}_fwd"] = fwd

  def teacher_ensemble_fwd(train_state, batch):
    # [n, classes] bookkeeping of an evaluation, not a step's hot path: torch's softmax
    probs = [torch.softmax(fns[f"{n}_fwd"](train_state, batch)[0], dim=-1) for n in teachers]
    return torch.stack(probs).mean(0), {}
  fns["teacher_ensemble_fwd"] = teacher_ensemble_fwd

  for name in teachers + ("teacher_ensemble",):
    def pair(train_state, batch, n=name):
      return fns["student_fwd"](train_state, batch), fns[f"{n}_fwd"](train_state, batch)
    fns[f"student_{name}_fwd"] = pair
  return fns
