"""Generates tests/golden/model_traces.json.gz: the C-ABI call trace of the ViT, two-tower and MLP-Mixer
models, and their parameter layouts.

The models run on CPU tensors with `lib.call` replaced by a recorder, so no kernel runs and no GPU is
needed.  For each configuration and freezing schedule the trace holds every call (entry point, scalar
arguments, the fields of its argument struct), every pointer resolved to `f|g|h:<storage>+<element>`
inside the FlatParams buffers or else `act` / `null`, the `P.on_ready` calls of the backward, and the
bytes the forward keeps for the backward beyond its inputs.  For each configuration it also holds the
FlatParams layout (storage name, offset, shape) and a checksum of `FlatParams.init(0)`, which fix the
spec order that checkpoints and the init's random stream rest on.  tests/test_model_traces.py compares
a fresh trace with it; a change that alters what the models launch, where they accumulate, what they
keep or how their parameters are laid out shows there.
  python tests/golden/make_model_traces.py
"""
import bisect
import ctypes
import gzip
import hashlib
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

# ViT: every pool, with and without scan and pre_logits, a padded 37-class head; sin-cos posemb with scan.
# Then every pool without a class head: pre_logits or the pooled encoder output is the model's output.
VIT_MODELS = ([dict(pool_type=pool, scan=scan, rep_size=rep, posemb="sincos2d" if scan else "learn")
               for pool in ("gap", "map", "tok", "0", "none") for scan in (False, True) for rep in (False, 32)]
              + [dict(pool_type=pool, rep_size=rep, num_classes=None)
                 for pool in ("gap", "map", "tok", "0", "none") for rep in (False, 32)])
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
# MLP-Mixer: a padded (6 -> 8) and an unpadded token count, a padded 37-class head and a 16-class one
MIXER_MODELS = [(hw, C) for hw in ((32, 48), (32, 64)) for C in (37, 16)]
MIXER_SCHEDULES = {
    "all": None,
    "head": r"head/.*",
    "pre_head+head": r"head/.*|pre_head_layer_norm/.*",
    "above_block0": r"(?!stem/|MixerBlock_0/).*",
    "middle_block": r"(?!MixerBlock_1/).*",
}
# stochastic-depth masks [num_blocks, 2 branches, n]: blocks 1 and 2 drop a sample in both branches
MIXER_MASKS = [[[1, 1], [1, 1]], [[1, 0], [0, 1]], [[0, 1], [1, 0]]]


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


def vit_models():
  from big_vision_b200 import engine as E
  from big_vision_b200.models import vit
  for kw in VIT_MODELS:
    model = vit.Model(**{"num_classes": 37, "width": 64, "depth": 3, "mlp_dim": 128, "num_heads": 1,
                         "patch_size": (16, 16), **kw})
    P = E.FlatParams(*model.specs((32, 32), 3), "cpu")
    yield "vit " + " ".join(f"{k}={v}" for k, v in kw.items()), model, P


def two_tower_models():
  import common
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.image_text import two_towers
  for pool in TEXT_POOLS:
    for scan in (False, True):
      kw = dict(common.TINY, image=dict(common.TINY["image"], scan=scan),
                text=dict(common.TINY["text"], scan=scan, pool_type=pool))
      model = two_towers.Model(**kw)
      P = E.FlatParams(*model.specs(common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE), "cpu")
      yield f"two_towers text_pool={pool} scan={scan}", model, P


def mixer_models():
  from big_vision_b200 import engine as E
  from big_vision_b200.models import mlp_mixer
  for hw, C in MIXER_MODELS:
    model = mlp_mixer.Model(C, patch_size=(16, 16), num_blocks=3, hidden_dim=64, tokens_mlp_dim=32,
                            channels_mlp_dim=128)
    yield f"mixer image={hw[0]}x{hw[1]} classes={C}", model, E.FlatParams(*model.specs(hw, 3), "cpu"), hw


def param_layouts():
  """Every configuration's storage names, offsets and shapes, and a checksum of its seed-0 init."""
  out = {}
  for tag, _, P, *_ in (*vit_models(), *two_tower_models(), *mixer_models()):
    P.init(0)
    out[f"{tag} / params"] = {
        "layout": [f"{name} {off} {list(shape)}" for name, (off, shape) in P.offsets.items()],
        "init_sha256": hashlib.sha256(P.flat.numpy().tobytes()).hexdigest()}
  return out


def vit_traces(patch):
  image = torch.zeros((2, 32, 32, 3))
  out = {}
  for tag, model, P in vit_models():
    for sched, trained in VIT_SCHEDULES.items():
      frozen = _frozen(P, trained)

      def step():
        y, saved = model.fwd(P, image, frozen=frozen)
        nbytes = saved_bytes(saved, P, image)
        cols = y.shape[-1] if model.head is None else model.head.Cp
        model.bwd(P, torch.zeros(y.shape[:-1] + (cols,)), saved)
        return nbytes
      lines, nbytes = _run(P, patch, step)
      out[f"{tag} / {sched}"] = {"calls": lines, "saved_bytes": nbytes}
    lines, _ = _run(P, patch, lambda: model.apply({"params": P}, image))
    out[f"{tag} / apply"] = {"calls": lines, "saved_bytes": 0}
  return out


def two_tower_traces(patch):
  import common
  image, text = torch.zeros(common.TINY_IMAGE_SHAPE), torch.ones(common.TINY_TEXT_SHAPE, dtype=torch.int32)
  n, D = common.TINY_IMAGE_SHAPE[0], common.TINY["out_dim"][1]
  out = {}
  for tag, model, P in two_tower_models():
    for sched, trained in TWO_TOWER_SCHEDULES.items():
      frozen = _frozen(P, trained)

      def step():
        _, _, saved = model.fwd(P, image, text, frozen=frozen)
        nbytes = saved_bytes(saved, P, image, text)
        model.bwd(P, torch.zeros((n, D)), torch.zeros((n, D)), saved)
        return nbytes
      lines, nbytes = _run(P, patch, step)
      out[f"{tag} / {sched}"] = {"calls": lines, "saved_bytes": nbytes}
  return out


def mixer_traces(patch):
  out = {}
  for tag, model, P, hw in mixer_models():
    image = torch.zeros((2,) + hw + (3,))
    for masks in (None, torch.tensor(MIXER_MASKS, dtype=torch.float32)):
      inputs = (image,) if masks is None else (image, masks)
      for sched, trained in MIXER_SCHEDULES.items():
        frozen = _frozen(P, trained)

        def step():
          _, saved = model.fwd(P, image, masks=masks, frozen=frozen)
          nbytes = saved_bytes(saved, P, *inputs)
          model.bwd(P, torch.zeros((2, model.head.Cp)), saved)
          return nbytes
        lines, nbytes = _run(P, patch, step)
        out[f"{tag} masks={masks is not None} / {sched}"] = {"calls": lines, "saved_bytes": nbytes}
    lines, _ = _run(P, patch, lambda: model.apply({"params": P}, image))
    out[f"{tag} / apply"] = {"calls": lines, "saved_bytes": 0}
  return out


def traces(patch):
  """Every configuration's trace and parameter layout; `patch(obj, name, value)` installs the recorder
  (and must undo it)."""
  out = param_layouts()         # first: FlatParams.init takes the CPU path only while nothing is patched
  for fn in (vit_traces, two_tower_traces, mixer_traces):
    out.update(fn(patch))
  return out


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
  print(f"{path}: {len(out)} entries, {sum(len(v.get('calls', ())) for v in out.values())} calls")


if __name__ == "__main__":
  main()
