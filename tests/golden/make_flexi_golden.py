"""Generates tests/golden/flexi_choices.json by RUNNING THE REFERENCE's own (numpy-only) flexi helpers
(big_vision/trainers/proj/flexi/common.py, imported by path, so neither jax nor tensorflow is needed): the
per-step draws of the flexible arguments and the predict-function names.  The outputs are committed, so the
test that checks them needs no reference checkout.

  python tests/golden/make_flexi_golden.py <big_vision checkout>
"""
import importlib.util
import json
import os
import sys

import numpy as np

spec = importlib.util.spec_from_file_location(
    "flexi_common", os.path.join(sys.argv[1], "big_vision", "trainers", "proj", "flexi", "common.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

# i21k_sup.py's seqhw values, under its uniform weights and under uneven ones; a second argument so the
# sorted-name draw order is exercised
FLEXI = {
    "uniform": {"seqhw": {"v": [5, 6, 8, 10, 12, 15, 16, 20, 24, 30], "p": [1] * 10}},
    "weighted": {"seqhw": {"v": [5, 6, 8, 10, 12, 15, 16, 20, 24, 30], "p": [1, 2, 3, 4, 5, 5, 4, 3, 2, 1]},
                 "alpha": {"v": [0.5, 1.0, 2.0], "p": [0.2, 0.3, 0.5]}},
}
out = {"flexi": FLEXI, "draws": {}}
for name, cfg in FLEXI.items():
  for xid in (-1, 0, 3):
    for wid in (-1, 0, 3):
      rows = []
      for step in range(1, 201):
        rng = ref.mkrng(xid, wid, step)     # the draw of flexi/train.py:284-288
        rows.append([ref.choice(cfg[n]["v"], cfg[n]["p"], rng).item() for n in sorted(cfg)])
      out["draws"][f"{name}/{xid}/{wid}"] = rows


class _Arg:
  def __init__(self, v):
    self.v = v


names = ref.mkpredictfns(lambda **kw: kw, {"seqhw": _Arg([5, 30]), "alpha": _Arg([0.5, 2.0])}, "predict_{x}")
out["predict_names"] = list(names)
out["predict_kw"] = [names[k]() for k in names]
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "flexi_choices.json"), "w") as f:
  json.dump(out, f, indent=None, separators=(",", ":"))
  f.write("\n")
