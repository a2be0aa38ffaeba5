"""FlexiViT distillation -- mirror of big_vision/trainers/proj/flexi/distill.py (configs
configs/proj/flexivit/i1k_deit3_distill.py and i21k_distill.py, how the published FlexiViT checkpoints were
trained):

  each step draws every flexible argument of the student on the host (flexi_args, the same draw on every
  rank), then runs the distillation step of trainers/proj/distill -- mixup of image, labels and every
  teacher-named input with one coefficient, each teacher's forward frozen at its own input, bv_distill_loss,
  the student's backward and all-reduce, tx.update, the same measurements -- with those arguments passed to
  the student's forward only.

`config` holds the distillation keys (`teachers`, `distance`, `distance_kw`, `mixup`, the optimizer) and
`flexi`, {argument name: {"v": values, "p": weights}}.  `train_state["params"]` is {"student": P, <teacher>:
P, ...}; only the student is trained.
"""
import functools

from big_vision_b200.trainers.proj.distill import distill
from big_vision_b200.trainers.proj.flexi import common as flexi
from big_vision_b200.trainers.proj.flexi.train import demand_flexi_args, flexi_args  # pylint: disable=unused-import


def make_update_fn(models, tx, config):
  """-> update_fn(train_state, rng, batch, **flexi_kw): distill.make_update_fn's step with `flexi_kw`
  (flexi_args of the step) passed to the student.  Every flexible argument must be given."""
  return demand_flexi_args(distill.make_update_fn(models, tx, config), config)


def make_predict_fns(models, config):
  """The predict functions of flexi/distill.py:325-348, each fn(train_state, batch) over
  train_state["params"] = {name: P}, a model reading batch[name] if present, else batch["image"]:
    "student_seqhw=5", ...: the student at each combination of the flexible arguments;
    "<teacher>": each teacher;
    "student_seqhw=5_<teacher>", ...: (student output, teacher output) for the distance evaluator."""
  def predict_fn(train_state, batch, *, name, **kw):
    return models[name].apply({"params": train_state["params"][name]}, distill.getfirst(batch, name, "image"), **kw)

  student_fns = flexi.mkpredictfns(functools.partial(predict_fn, name="student"), config["flexi"], "student_{x}")
  teacher_fns = {name: functools.partial(predict_fn, name=name) for name in config["teachers"]}
  pairs = {f"{sn}_{tn}": lambda ts, batch, sfn=sfn, tfn=tfn: (sfn(ts, batch), tfn(ts, batch))
           for sn, sfn in student_fns.items() for tn, tfn in teacher_fns.items()}
  return {**student_fns, **teacher_fns, **pairs}


# the config-driven initialisation is the plain distillation trainer's (trainers/proj/distill)
_model_module = distill._model_module
init_params = distill.init_params
