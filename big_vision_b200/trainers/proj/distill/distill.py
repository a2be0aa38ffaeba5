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
import importlib

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
  seed = int(config.get("seed", 0))

  def update_fn(train_state, rng, batch, **student_kw):
    """`student_kw`: extra keyword arguments of the student's forward only (a FlexiViT student's seqhw)."""
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
    if getattr(student, "dropout", 0.0):      # the teachers run train=False: no dropout
      kw["dropout"] = train.dropout_key(seed, opt, d, getfirst(data, "student", "image").shape[0])
    m = loss_and_grads(models, params, data, teachers, kind, distance_kw, dist_view=d, frozen=frozen, **kw,
                       **student_kw)
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


def _model_module(config, name):
  return importlib.import_module(f"big_vision_b200.models.{config[f'{name}_name']}")


def init_params(params, config):
  """Initialises params {name: FlatParams} in place after model.init, as flexi/distill.py:273-314 does:
    - `init_head_bias` first fills every model's head bias, as the distillation trainer's init does
      (distill/distill.py:186-189): the i21k config's -10, so the loss starts small.  A loaded head
      replaces it;
    - each teacher loads `<name>_init` through its model module's `load` (config["<name>_name"]), with
      config[name] as the model config and config["<name>_load"] as keyword arguments.  Teachers are
      never checkpointed, so each must have one;
    - then the student loads `student_init` the same way, if the config has one.  For a FlexiViT student
      that is models/proj/flexi/vit.py:load, which takes a plain ViT checkpoint of any grid and patch
      size: it resizes the position embedding and resamples the patch-embedding kernel; for a BiT model
      (`bit_paper`) models/bit_paper.py:load, which also converts TF-dumped BiT checkpoints.
  Shared by this trainer and trainers/proj/flexi/distill.py."""
  if "init_head_bias" in config:
    for P in params.values():
      views = P.tree("f")
      if "head/bias" in views:
        views["head/bias"].fill_(config["init_head_bias"])
        P.sync_half()
  teachers = tuple(config["teachers"])
  for name in teachers + ("student",):
    init = config.get(f"{name}_init")
    if not init:
      if name != "student":
        raise ValueError(f"teacher '{name}' has no {name}_init: teachers are never trained or checkpointed")
      continue
    from big_vision_b200 import utils as u
    P = params[name]
    tree = u.recover_tree(*zip(*P.numpy_tree("f").items()))
    tree = _model_module(config, name).load(tree, init, dict(config.get(name) or {}),
                                            **config.get(f"{name}_load", {}))
    P.load_tree(dict(u.tree_flatten_with_names(tree)[0]))
  return params
