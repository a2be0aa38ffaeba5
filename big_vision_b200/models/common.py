"""Host-side helpers shared by the model modules.

`merge_params` has the contract of big_vision/models/common.py:24-92: the result has the structure
of the freshly initialised tree and the checkpoint's values, except for names matched by a
`dont_load` regex (those keep their init value and may be absent on either side); any other
structural difference is an error that lists both sides.

`Dense` is the Dense stage of every model's heads (pre_logits, the class heads), and `dense_specs` the
one place that knows how a Dense with padded columns is stored.
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


def dense_specs(prefix, fan_in, fan_out, init, store_cols=None):
  """(specs, aliases) of a Dense: kernel [fan_in, fan_out] from `init`, zero bias [fan_out].

  A kernel that is the MN-major B operand of a GEMM needs a row stride of a multiple of 16 bytes (TMA).
  With `store_cols` > fan_out the kernel and bias are stored as `kernel_pad` [fan_in, store_cols] and
  `bias_pad` [store_cols], zero past column fan_out, and exposed under the reference names as the views
  [:, :fan_out] and [:fan_out].  The first spec is always the kernel, the second the bias."""
  sc = store_cols or fan_out
  if sc == fan_out:
    return [E.ParamSpec(prefix + "kernel", (fan_in, fan_out), init),
            E.ParamSpec(prefix + "bias", (fan_out,), E.zeros)], []
  pad = np.zeros((fan_in, sc - fan_out))
  specs = [E.ParamSpec(prefix + "kernel_pad", (fan_in, sc),
                       lambda rng, shape: np.concatenate([init(rng, (fan_in, fan_out)), pad], 1)),
           E.ParamSpec(prefix + "bias_pad", (sc,), E.zeros)]
  aliases = [E.Alias(prefix + "kernel", prefix + "kernel_pad", lambda t: t[:, :fan_out]),
             E.Alias(prefix + "bias", prefix + "bias_pad", lambda t: t[:fan_out])]
  return specs, aliases


class Dense(E.Stage):
  """A Dense stored under `prefix` (kernel [fan_in, fan_out], bias [fan_out]) as a backward stage
  (engine.Staged): bf16 GEMM operands, fp32 output, tanh(x W + b) with `tanh` (the ViT's pre_logits),
  the input gradient in `dx_dtype`.  `rep` is the input width (a head's representation size), `C` the
  output width.

  pad=True is for class heads: when the class count C = fan_out is not a multiple of 8 (21843 for
  ImageNet-21k, 37 for Oxford pets, ...) the kernel and bias are stored with Cp = round_up(C, 8)
  columns (dense_specs), the output is the [rows, C] view of the [rows, Cp] GEMM output, and the
  backward takes the output gradient as [rows, Cp].  The padding starts at zero and stays exactly zero:
  the logit gradient is zero in its padding columns (the xent kernels write it so), so the padding's
  gradient is zero, and an Adam / scale update and the weight decay of zero are zero; Adafactor
  updates the reference-shaped views only."""

  def __init__(self, prefix, fan_in, fan_out, kernel_init, *, tanh=False, dx_dtype=torch.float32, pad=False):
    self.p, self.rep, self.C, self.tanh, self.dx_dtype = prefix, fan_in, fan_out, tanh, dx_dtype
    self.Cp = (fan_out + 7) // 8 * 8 if pad else fan_out
    self._specs = dense_specs(prefix, fan_in, fan_out, kernel_init, self.Cp)
    self.kernel, self.bias = (s.name for s in self._specs[0])
    self.prefixes = (prefix,)

  def specs(self):
    return self._specs

  def fwd(self, P, x, geom=None, save=True):
    """x [rows, fan_in] -> (y fp32 [rows, C], saved)."""
    y = ops.gemm(to16(x), P.h(self.kernel), b_mn=True, bias=P.f(self.bias), out_dtype=torch.float32)
    if self.tanh:
      y = ops.tanh_fwd(y)
    saved = (x, y if self.tanh else None) if save else None
    return (y if self.Cp == self.C else y[:, :self.C]), saved

  def bwd(self, P, dy, saved, geom=None, sink=None, need_dx=True):
    """dy fp32 [rows, Cp], zero in the columns past C.  Accumulates the Dense's gradients and returns
    d x ([rows, fan_in] in dx_dtype), or None with need_dx=False."""
    if tuple(dy.shape[1:]) != (self.Cp,):
      raise ValueError(f"{self.p} backward: the output gradient must be [rows, {self.Cp}] (the stored "
                       f"columns, zero past column {self.C}), got {tuple(dy.shape)}")
    x, y = saved
    if self.tanh:
      dy = ops.tanh_bwd(dy, y)
    d16 = to16(dy)
    ops.colsum(dy, P.g(self.bias))
    ops.gemm(to16(x), d16, a_mn=True, b_mn=True, out=P.g(self.kernel), reduce_out=True)
    return ops.gemm(d16, P.h(self.kernel), out_dtype=self.dx_dtype) if need_dx else None


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
