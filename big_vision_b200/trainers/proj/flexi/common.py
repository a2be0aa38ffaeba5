"""Helpers of the flexible-setting trainers (reference trainers/proj/flexi/common.py): the per-step random
draw of each flexible model argument, and one predict function per combination of their values.

`config` here is the trainer config's `flexi` section: {argument name: {"v": values, "p": weights}}.
"""
import functools
import itertools

import numpy as np


def mkrng(xid, wid, step):
  """The numpy Generator of one step, seeded by (experiment id, work-unit id, step), each capped below at 0
  (local runs use -1).  Every host makes the same draw."""
  return np.random.default_rng((max(xid, 0), max(wid, 0), max(step, 0)))


def mkprob(x):
  """Weights -> probabilities (None stays None: uniform)."""
  if x is None:
    return None
  return np.array(x) / np.sum(x)


def choice(values, ratios, rng=None):
  """One of `values`, drawn with probabilities proportional to `ratios`."""
  if rng is None:
    rng = np.random.default_rng()
  return rng.choice(values, p=mkprob(ratios))


def mkpredictfns(predict_fn, config, template="predict_{x}"):
  """{template.format(x="a=1_b=10"): predict_fn with a=1, b=10 bound, ...} over every combination of the
  flexible arguments' values, arguments in the config's order."""
  combos = itertools.product(*[[(arg, val) for val in config[arg]["v"]] for arg in config])
  return {template.format(x="_".join(f"{k}={v}" for k, v in combo)): functools.partial(predict_fn, **dict(combo))
          for combo in combos}
