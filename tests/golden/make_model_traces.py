"""Generates tests/golden/model_traces.json.gz: the C-ABI call trace of the ViT and two-tower models.

The models run on CPU tensors with `lib.call` replaced by a recorder, so no kernel runs and no GPU is
needed.  For each configuration and freezing schedule the trace holds every call (entry point, scalar
arguments, the fields of its argument struct), every pointer resolved to `f|g|h:<storage>+<element>`
inside the FlatParams buffers or else `act` / `null`, the `P.on_ready` calls of the backward, and the
bytes the forward keeps for the backward beyond its inputs.  tests/test_model_traces.py compares a fresh trace with it;
a change that alters what the models launch, where they accumulate or what they keep shows there.
  python tests/golden/make_model_traces.py
"""
import bisect
import ctypes
import gzip
import json
import os
import re
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "model_traces.json.gz")
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

# ViT: every pool, with and without scan and pre_logits, a padded 37-class head; sin-cos posemb with scan
VIT_MODELS = [dict(pool_type=pool, scan=scan, rep_size=rep, posemb="sincos2d" if scan else "learn")
              for pool in ("gap", "map", "tok", "0", "none") for scan in (False, True) for rep in (False, 32)]
# name -> regex of the TRAINED storage names (everything else is frozen); None: nothing frozen
VIT_SCHEDULES = {
    "all": None,
    "head": r"head/.*",
    "head+map": r"head/.*|MAPHead_0/.*",
    "pre_logits+head": r"head/.*|pre_logits/.*",
    "above_block0": r"(?!embedding/|pos_embedding|cls|Transformer/encoderblock_0/).*",
    "above_encoder": r"(?!embedding/|pos_embedding|cls|Transformer/encoderblock).*",
    "middle_block": r"(?!Transformer/encoderblock_1/).*",
}
TEXT_POOLS = ("last", "first", "mean", "max", "map")
TWO_TOWER_SCHEDULES = {
    "all": None,
    "siglit": r"(?!img/).*",
    "txt_frozen": r"(?!txt/).*",
    "txt_head": r"txt/head/.*",
}


class Recorder:
  """Stands in for `lib.call`: appends one line per call, pointers resolved against `P`."""

  def __init__(self, P):
    self.P, self.lines = P, []
    self.names = sorted((off, name, int(np.prod(shape))) for name, (off, shape) in P.offsets.items())
    self.starts = [o for o, _, _ in self.names]

  def ptr(self, p):
    if p is None:
      return "null"
    for kind, buf in (("f", self.P.flat), ("g", self.P.grad), ("h", self.P.half)):
      base = buf.data_ptr()
      if base <= p < base + buf.numel() * buf.element_size():
        e = (p - base) // buf.element_size()
        off, name, n = self.names[bisect.bisect_right(self.starts, e) - 1]
        return f"{kind}:{name}+{e - off}" if e < off + n else f"{kind}:<pad>+{e}"
    return "act"

  def struct(self, s):
    out = []
    for name, typ in s._fields_:   # pylint: disable=protected-access
      v = getattr(s, name)
      if typ is ctypes.c_void_p:
        out.append(f"{name}={self.ptr(v)}")
      elif isinstance(v, ctypes.Structure):
        out.append(f"{name}={{{' '.join(self.struct(v))}}}")
      else:
        out.append(f"{name}={v!r}")
    return out

  def arg(self, a):
    if a is None:
      return "null"
    if isinstance(a, ctypes.c_void_p):
      return self.ptr(a.value)
    if type(a).__name__ == "CArgObject":           # ctypes.byref(struct)
      return "{" + " ".join(self.struct(a._obj)) + "}"   # pylint: disable=protected-access
    return repr(a)

  def call(self, name, *args, tag=None):
    del tag
    self.lines.append(" ".join([name] + [self.arg(a) for a in args]))


def saved_bytes(saved, P, *inputs):
  """Bytes of the distinct storages reachable from `saved`, except the parameter buffers and the
  model's inputs (the caller holds those anyway)."""
  skip = {t.untyped_storage().data_ptr() for t in (P.flat, P.grad, P.half) + inputs}
  seen, stack = {}, [saved]
  while stack:
    x = stack.pop()
    if isinstance(x, torch.Tensor):
      st = x.untyped_storage()
      if st.data_ptr() not in skip:
        seen[st.data_ptr()] = st.nbytes()
    elif isinstance(x, dict):
      stack.extend(x.values())
    elif isinstance(x, (list, tuple)):
      stack.extend(x)
  return sum(seen.values())


def _frozen(P, trained):
  if trained is None:
    return None
  return frozenset(k for k in P.offsets if not re.fullmatch(trained, k))


def _run(P, patch, fn):
  """fn() under the recorder; returns (trace lines, fn's result)."""
  from big_vision_b200 import lib, ops
  rec = Recorder(P)
  patch(lib, "call", rec.call)
  patch(ops, "_stream", lambda: "stream")
  patch(torch.Tensor, "is_cuda", property(lambda self: True))
  P.on_ready = lambda name: rec.lines.append("on_ready " + name)
  out = fn()
  return rec.lines, out


def vit_traces(patch):
  from big_vision_b200 import engine as E
  from big_vision_b200.models import vit
  image = torch.zeros((2, 32, 32, 3))
  out = {}
  for kw in VIT_MODELS:
    model = vit.Model(37, width=64, depth=3, mlp_dim=128, num_heads=1, patch_size=(16, 16), **kw)
    P = E.FlatParams(*model.specs((32, 32), 3), "cpu")
    tag = "vit " + " ".join(f"{k}={v}" for k, v in kw.items())
    for sched, trained in VIT_SCHEDULES.items():
      frozen = _frozen(P, trained)

      def step():
        y, saved = model.fwd(P, image, frozen=frozen)
        nbytes = saved_bytes(saved, P, image)
        rows = y.shape[:-1]
        model.bwd(P, torch.zeros(rows + (model.head.Cp,)), saved)
        return nbytes
      lines, nbytes = _run(P, patch, step)
      out[f"{tag} / {sched}"] = {"calls": lines, "saved_bytes": nbytes}
    lines, _ = _run(P, patch, lambda: model.apply({"params": P}, image))
    out[f"{tag} / apply"] = {"calls": lines, "saved_bytes": 0}
  return out


def two_tower_traces(patch):
  import common
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.image_text import two_towers
  image, text = torch.zeros(common.TINY_IMAGE_SHAPE), torch.ones(common.TINY_TEXT_SHAPE, dtype=torch.int32)
  n, D = common.TINY_IMAGE_SHAPE[0], common.TINY["out_dim"][1]
  out = {}
  for pool in TEXT_POOLS:
    for scan in (False, True):
      kw = dict(common.TINY, image=dict(common.TINY["image"], scan=scan),
                text=dict(common.TINY["text"], scan=scan, pool_type=pool))
      model = two_towers.Model(**kw)
      P = E.FlatParams(*model.specs(common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE), "cpu")
      for sched, trained in TWO_TOWER_SCHEDULES.items():
        frozen = _frozen(P, trained)

        def step():
          _, _, saved = model.fwd(P, image, text, frozen=frozen)
          nbytes = saved_bytes(saved, P, image, text)
          model.bwd(P, torch.zeros((n, D)), torch.zeros((n, D)), saved)
          return nbytes
        lines, nbytes = _run(P, patch, step)
        out[f"two_towers text_pool={pool} scan={scan} / {sched}"] = {"calls": lines, "saved_bytes": nbytes}
  return out


def traces(patch):
  """Every configuration's trace; `patch(obj, name, value)` installs the recorder (and must undo it)."""
  return {**vit_traces(patch), **two_tower_traces(patch)}


def load():
  with gzip.open(GOLDEN, "rt") as f:
    return json.load(f)


def main():
  undo = []

  def patch(obj, name, value):
    undo.append((obj, name, obj.__dict__.get(name)))
    setattr(obj, name, value)
  try:
    out = traces(patch)
  finally:
    for obj, name, old in reversed(undo):
      if old is None:
        delattr(obj, name)
      else:
        setattr(obj, name, old)
  path = sys.argv[1] if len(sys.argv) > 1 else GOLDEN
  with gzip.GzipFile(path, "wb", mtime=0) as f:
    f.write(json.dumps(out, indent=0, sort_keys=True).encode())
  print(f"{path}: {len(out)} configurations, {sum(len(v['calls']) for v in out.values())} calls")


if __name__ == "__main__":
  main()
