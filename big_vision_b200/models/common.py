"""Host-side helpers shared by the model modules.

`merge_params` has the contract of big_vision/models/common.py:24-92: the result has the structure
of the freshly initialised tree and the checkpoint's values, except for names matched by a
`dont_load` regex (those keep their init value and may be absent on either side); any other
structural difference is an error that lists both sides.

`ClassifierHead` is the `head` Dense of the ViT and MLP-Mixer classifiers, the one place that knows
how its parameters are stored.
"""
import numpy as np
import torch

from big_vision_b200 import engine as E
from big_vision_b200 import ops
from big_vision_b200 import utils as u


def to16(x):
  """bf16 operand of a GEMM: x itself if it is bf16, else a bf16 copy."""
  if x.dtype == torch.bfloat16:
    return x
  return ops.cast(x, torch.empty_like(x, dtype=torch.bfloat16))


class ClassifierHead(E.Stage):
  """The `head` Dense (kernel [rep, C], bias [C]) of a classifier, logits in fp32; a backward stage
  (engine.Staged) of the ViT.

  The kernel is the MN-major B operand of the head GEMM, and TMA needs its row stride to be a multiple
  of 16 bytes.  So with C % 8 != 0 (21843 classes for ImageNet-21k, 37 for Oxford pets, ...) it is
  stored as `head/kernel_pad` [rep, Cp] and `head/bias_pad` [Cp], Cp = round_up(C, 8), and exposed
  under the reference names as the views [:, :C] and [:C].  The padding starts at zero and stays
  exactly zero: the logit gradient is zero in its padding columns (the xent kernels write it so), so
  the padding's gradient is zero, and an Adam / scale update and the weight decay of zero are zero;
  Adafactor updates the reference-shaped views only.  With C % 8 == 0 nothing is padded or aliased.
  """

  def __init__(self, prefix, rep, num_classes, kernel_init):
    self.rep, self.C, self.kernel_init = rep, num_classes, kernel_init
    self.Cp = (num_classes + 7) // 8 * 8
    pad = "_pad" if self.Cp != self.C else ""
    self.p, self.kernel, self.bias = prefix + "head/", prefix + "head/kernel" + pad, prefix + "head/bias" + pad
    self.prefixes = (self.p,)

  def specs(self):
    rep, C, Cp, init = self.rep, self.C, self.Cp, self.kernel_init
    if Cp == C:
      return [E.ParamSpec(self.kernel, (rep, C), init), E.ParamSpec(self.bias, (C,), E.zeros)], []
    specs = [E.ParamSpec(self.kernel, (rep, Cp),
                         lambda rng, shape: np.concatenate([init(rng, (rep, C)), np.zeros((rep, Cp - C))], 1)),
             E.ParamSpec(self.bias, (Cp,), E.zeros)]
    aliases = [E.Alias(self.p + "kernel", self.kernel, lambda t: t[:, :C]),
               E.Alias(self.p + "bias", self.bias, lambda t: t[:C])]
    return specs, aliases

  def fwd(self, P, x, geom=None, save=True):
    """x [rows, rep] -> (logits fp32 [rows, C], x if save): a view of the [rows, Cp] GEMM output when
    padded."""
    out = ops.gemm(to16(x), P.h(self.kernel), b_mn=True, bias=P.f(self.bias), out_dtype=torch.float32)
    return (out if self.Cp == self.C else out[:, :self.C]), (x if save else None)

  def bwd(self, P, dlogits, x, geom=None, sink=None, need_dx=True):
    """dlogits fp32 [rows, Cp], zero in the columns past C; x the forward's input.  Accumulates the
    head's gradients and returns d x (fp32 [rows, rep]), or None with need_dx=False."""
    if tuple(dlogits.shape[1:]) != (self.Cp,):
      raise ValueError(f"head backward: the logit gradient must be [rows, {self.Cp}] (padded to "
                       f"{self.Cp} zero-filled columns), got {tuple(dlogits.shape)}")
    d16 = to16(dlogits)
    ops.colsum(dlogits, P.g(self.bias))
    ops.gemm(to16(x), d16, a_mn=True, b_mn=True, out=P.g(self.kernel), reduce_out=True)
    return ops.gemm(d16, P.h(self.kernel), out_dtype=torch.float32) if need_dx else None


def _report(ckpt_names, model_names, only_model, only_ckpt):
  def block(title, names, bullet="  "):
    return [f"{title}:"] + [f"{bullet}{n}" for n in sorted(names)] if names else []
  lines = (block("Params in checkpoint", ckpt_names) + block("Params in model (code)", model_names) +
           block("Params in model (code) but not in checkpoint and not `dont_load`ed", only_model, " - ") +
           block("Params in checkpoint but not in model (code) and not `dont_load`ed", only_ckpt, " + "))
  return "\n".join(lines)


def merge_params(loaded, inited, dont_load=(), match_dtype=False):
  if inited is None:                 # nothing to match against (interactive use)
    return loaded
  patterns = u.check_and_compile_patterns(dont_load)
  exempt = lambda name: any(p.fullmatch(name) for p in patterns)
  ckpt = dict(u.tree_flatten_with_names(loaded)[0])
  model = dict(u.tree_flatten_with_names(inited)[0])

  out = {}
  for name, init_val in model.items():
    if name in ckpt and not exempt(name):
      out[name] = ckpt[name].astype(init_val.dtype) if match_dtype else ckpt[name]
    else:
      out[name] = init_val           # dont_load, or (checked below) missing from the checkpoint

  only_model = [n for n in model if n not in ckpt and not exempt(n)]
  only_ckpt = [n for n in ckpt if n not in model and not exempt(n)]
  if only_model or only_ckpt:
    raise ValueError(_report(ckpt.keys(), model.keys(), only_model, only_ckpt))
  return u.recover_tree(list(out.keys()), list(out.values()))
