"""FlexiViT classification training -- mirror of big_vision/trainers/proj/flexi/train.py
(config: configs/proj/flexivit/i21k_sup.py):

  each step draws every flexible model argument on the host (flexi_args), then runs the classification
  step of train.py -- mixup, the loss, frozen parameters, the gradient all-reduce, the optimizer and the
  measurements unchanged -- with those arguments passed to the model's forward.

`config["flexi"]` is {argument name: {"v": values, "p": weights}}, e.g. seqhw = {"v": (5, ..., 30),
"p": (1, ..., 1)}.
"""
from big_vision_b200 import train
from big_vision_b200.trainers.proj.flexi import common as flexi


def flexi_args(config, step, xid=-1, wid=-1):
  """The step's values of the flexible arguments: one draw per argument in sorted name order from the
  step's Generator (flexi/train.py:284-288), so every host draws the same."""
  rng = flexi.mkrng(xid, wid, step)
  return {name: flexi.choice(config["flexi"][name]["v"], config["flexi"][name].get("p"), rng).item()
          for name in sorted(config["flexi"])}


def demand_flexi_args(step, config):
  """-> update_fn(train_state, rng, batch, **flexi_kw) = step(...) that refuses a call which does not pass
  exactly the flexible arguments of `config`."""
  names = sorted(config["flexi"])

  def update_fn(train_state, rng, batch, **flexi_kw):
    if sorted(flexi_kw) != names:
      raise TypeError(f"update_fn takes the flexible arguments {names}, got {sorted(flexi_kw)}")
    return step(train_state, rng, batch, **flexi_kw)

  return update_fn


def make_update_fn(model, tx, config):
  """-> update_fn(train_state, rng, batch, **flexi_kw): train.py's step with `flexi_kw` (flexi_args of
  the step) passed to the model.  Every flexible argument must be given."""
  return demand_flexi_args(train.make_update_fn(model, tx, config), config)


def make_predict_fns(model, config):
  """{"predict_seqhw=5": fn(params, image) -> (logits, out), ...}: one per combination of the flexible
  arguments' values (flexi/train.py:206-209, 253-256)."""
  def predict_fn(params, image, **flexi_kw):
    return model.apply({"params": params}, image, **flexi_kw)
  return flexi.mkpredictfns(predict_fn, config["flexi"], "predict_{x}")
