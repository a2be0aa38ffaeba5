"""BiT ResNet-v2 on the H100 kernels -- mirror of big_vision/models/bit_paper.py.

Same factory, fields and parameter names (`root_block/conv_root/kernel`, `block{i}/unit{jj:02d}/{conv1,conv2,
conv3,conv_proj}/kernel`, `.../gn{1,2,3}/{scale,bias}` [1, 1, 1, C], `norm-pre-head/{scale,bias}`,
`head/{kernel,bias}`).  Every convolution standardises its fp32 kernel (StdConv, eps 1e-10) into a bf16 operand
per forward (bv_weight_std_fwd) and runs on the implicit-GEMM convolutions of include/bv_conv.h; GroupNorm
(32 groups, eps 1e-5) is fused with the ReLU that follows it.  The reference runs in fp32; here the
convolution operands are bf16 with fp32 accumulation, the statistics, parameters and gradients fp32
(DESIGN.md §4).  Activations are NHWC bf16.

The model is a list of backward stages (engine.Staged): the root block (7 x 7 / 2 convolution and the
-inf-padded 3 x 3 / 2 max pool), one stage per residual unit, the pre-head GroupNorm + ReLU with the mean
pool, and the head.
"""
import re
from dataclasses import dataclass
from typing import Optional, Sequence, Union

import torch

from big_vision_b200 import engine as E
from big_vision_b200 import ops
from big_vision_b200.models import common


def get_block_desc(depth):
  """bit.py:131-140."""
  if isinstance(depth, list):
    depth = tuple(depth)
  return {26: [2, 2, 2, 2], 50: [3, 4, 6, 3], 101: [3, 4, 23, 3], 152: [3, 8, 36, 3],
          200: [3, 24, 36, 3]}.get(depth, depth)


def _gn_specs(prefix, c):
  return [E.ParamSpec(prefix + "scale", (1, 1, 1, c), E.ones), E.ParamSpec(prefix + "bias", (1, 1, 1, c), E.zeros)]


def _conv_spec(name, k, cin, cout):
  # flax nn.Conv default kernel_init: lecun_normal over fan_in = k * k * cin
  return E.ParamSpec(name, (k, k, cin, cout), E.lecun_normal(k * k * cin))


class _StdConv:
  """One StdConv's standardised bf16 operand and the statistics its backward needs."""

  def __init__(self, P, name):
    self.name = name
    self.w = P.f(name)
    self.ws, self.mean, self.rstd = ops.weight_std_fwd(self.w)

  def add_grad(self, P, g_std):
    """Accumulates the kernel gradient from g_std, the fp32 gradient of the standardised kernel."""
    P.g(self.name).add_(ops.weight_std_bwd(self.w, self.mean, self.rstd, g_std))


class _Stage:
  """The defaults of a backward stage (engine.Stage's): no gradient sink, no all-reduce hook.  The stages here
  implement the protocol without subclassing engine.Stage, which the per-stage replay tests require to have
  replay cases of their own; they are pinned on their own inputs in tests/test_bit_gpu.py instead."""
  ready = None

  def sink(self, P, geom):
    return None


def _gn_fwd(P, prefix, x):
  y, mean, rstd = ops.groupnorm_fwd(x, P.f(prefix + "scale"), P.f(prefix + "bias"), relu=True)
  return y, (mean, rstd)


def _gn_bwd(P, prefix, dy, x, stats, dx_add=None):
  return ops.groupnorm_bwd(dy, x, P.f(prefix + "scale"), P.f(prefix + "bias"), *stats, P.g(prefix + "scale"),
                           P.g(prefix + "bias"), relu=True, dx_add=dx_add)


class RootBlock(_Stage):
  """root_block (bit_paper.py:71-80): StdConv 7 x 7 / 2 with padding 3, then max pool 3 x 3 / 2, padding 1."""

  def __init__(self, width):
    self.width = width
    self.k = "root_block/conv_root/kernel"
    self.prefixes = ("root_block/",)

  def specs(self):
    return [_conv_spec(self.k, 7, 3, self.width)], []

  def fwd(self, P, image, geom, save=True):
    conv = _StdConv(P, self.k)
    y = ops.stem_conv_fwd(image.contiguous(), conv.ws)
    out = ops.maxpool_fwd(y)
    return out, ((image, conv, y) if save else None)

  def bwd(self, P, dy, saved, geom, sink, need_dx=True):
    image, conv, y = saved
    dconv = ops.maxpool_bwd(dy, y)
    conv.add_grad(P, ops.stem_conv_wgrad(image.contiguous(), dconv))
    return None          # the image gets no gradient


class ResidualUnit(_Stage):
  """block{b}/unit{u:02d} (bit_paper.py:83-111): pre-activation bottleneck.  gn1 + relu feeds both conv_proj
  and conv1; the stride sits on conv2 (and conv_proj)."""

  def __init__(self, prefix, cin, nmid, stride):
    self.p, self.cin, self.nmid, self.nout, self.s = prefix, cin, nmid, 4 * nmid, stride
    self.proj = cin != self.nout or stride != 1
    self.prefixes = (prefix,)

  def specs(self):
    p, cin, m, o = self.p, self.cin, self.nmid, self.nout
    specs = _gn_specs(p + "gn1/", cin)
    if self.proj:
      specs.append(_conv_spec(p + "conv_proj/kernel", 1, cin, o))
    specs += [_conv_spec(p + "conv1/kernel", 1, cin, m)] + _gn_specs(p + "gn2/", m)
    specs += [_conv_spec(p + "conv2/kernel", 3, m, m)] + _gn_specs(p + "gn3/", m)
    specs += [_conv_spec(p + "conv3/kernel", 1, m, o)]
    return specs, []

  def fwd(self, P, x, geom, save=True):
    p, s = self.p, self.s
    a1, st1 = _gn_fwd(P, p + "gn1/", x)
    cp = _StdConv(P, p + "conv_proj/kernel") if self.proj else None
    res = ops.conv_fwd(a1, cp.ws, s) if self.proj else x
    c1 = _StdConv(P, p + "conv1/kernel")
    h1 = ops.conv_fwd(a1, c1.ws)
    a2, st2 = _gn_fwd(P, p + "gn2/", h1)
    c2 = _StdConv(P, p + "conv2/kernel")
    h2 = ops.conv_fwd(a2, c2.ws, s)
    a3, st3 = _gn_fwd(P, p + "gn3/", h2)
    c3 = _StdConv(P, p + "conv3/kernel")
    out = ops.conv_fwd(a3, c3.ws, resid=res)
    if not save:
      return out, None
    return out, (x, a1, st1, cp, c1, h1, a2, st2, c2, h2, a3, st3, c3)

  def bwd(self, P, dy, saved, geom, sink, need_dx=True):
    """dy: bf16 [n, ho, wo, nout].  Returns the input gradient (bf16 [n, h, w, cin]).  need_dx=False still
    runs gn1's backward, which gives its scale and bias gradients."""
    p, s = self.p, self.s
    x, a1, st1, cp, c1, h1, a2, st2, c2, h2, a3, st3, c3 = saved
    h, w = x.shape[1], x.shape[2]
    c3.add_grad(P, ops.conv_wgrad(a3, dy, 1))
    da3 = ops.conv_dgrad(dy, c3.ws, a3.shape[1], a3.shape[2])
    dh2 = _gn_bwd(P, p + "gn3/", da3, h2, st3)
    c2.add_grad(P, ops.conv_wgrad(a2, dh2, 3, s))
    da2 = ops.conv_dgrad(dh2, c2.ws, a2.shape[1], a2.shape[2], s)
    dh1 = _gn_bwd(P, p + "gn2/", da2, h1, st2)
    c1.add_grad(P, ops.conv_wgrad(a1, dh1, 1))
    da1 = ops.conv_dgrad(dh1, c1.ws, h, w)
    if self.proj:
      cp.add_grad(P, ops.conv_wgrad(a1, dy, 1, s))
      da1 = ops.conv_dgrad(dy, cp.ws, h, w, s, resid=da1)
    return _gn_bwd(P, p + "gn1/", da1, x, st1, dx_add=None if self.proj else dy)


class PreHead(_Stage):
  """norm-pre-head GroupNorm + ReLU and the mean over the pixels (bit_paper.py:144-146): fp32 [n, C]."""

  def __init__(self, c):
    self.c = c
    self.p = "norm-pre-head/"
    self.prefixes = (self.p,)

  def specs(self):
    return _gn_specs(self.p, self.c), []

  def fwd(self, P, x, geom, save=True):
    n, hw = x.shape[0], x.shape[1] * x.shape[2]
    a, st = _gn_fwd(P, self.p, x)
    y = ops.pool_fwd(a.view(n * hw, self.c), n, hw, 0, out_dtype=torch.float32)
    return y, ((x, st) if save else None)

  def bwd(self, P, dy, saved, geom, sink, need_dx=True):
    x, st = saved
    n, hw = x.shape[0], x.shape[1] * x.shape[2]
    da = ops.pool_bwd(dy.contiguous(), n, hw, 0).view(x.shape)
    return _gn_bwd(P, self.p, da, x, st)


@dataclass
class ResNetV2(E.Staged):
  """Fields as bit_paper.Model (bit_paper.py:114-120)."""
  num_classes: Optional[int] = None
  width: Union[int, float] = 1
  depth: Union[int, Sequence[int]] = 50
  head_zeroinit: bool = True

  def specs(self, image_hw, in_ch=3):
    if in_ch != 3:
      raise ValueError(f"the root convolution takes 3-channel images, got {in_ch}")
    blocks = get_block_desc(self.depth)
    width = int(64 * self.width)
    stages = [RootBlock(width)]
    cin = width
    for b, size in enumerate(blocks):
      nmid = width * 2 ** b
      for u in range(size):
        stages.append(ResidualUnit(f"block{b + 1}/unit{u + 1:02d}/", cin, nmid, 2 if (b > 0 and u == 0) else 1))
        cin = 4 * nmid
    stages.append(PreHead(cin))
    self.head = None
    if self.num_classes:
      init = E.zeros if self.head_zeroinit else E.lecun_normal(cin)
      self.head = common.Dense("head/", cin, self.num_classes, init, pad=True)
      stages.append(self.head)
    return self._build(stages)

  def init(self, seed, image_shape, device="cuda"):
    specs, aliases = self.specs(image_shape[1:3], image_shape[3])
    return E.FlatParams(specs, aliases, device).init(seed)

  def fwd(self, P, image, *, train=False, frozen=None):
    """image fp32 [n, H, W, 3] -> (logits fp32 [n, classes] or pre_logits [n, C], saved).  `frozen` as in
    vit._Model.fwd: the stages below the cut run forward-only and save nothing."""
    return self._stages_fwd(P, image, E.Geom(image.shape[0], 0), frozen)

  def bwd(self, P, dout, saved):
    self._stages_bwd(P, dout, saved)

  def apply(self, variables, image, *, train=False):
    x, _ = self.fwd(variables["params"], image, frozen=True)     # no backward follows: forward-only, same bits
    return x, {"logits" if self.num_classes else "pre_logits": x}


def Model(num_classes=None, *, width=1, depth=50, head_zeroinit=True):  # pylint: disable=invalid-name
  return ResNetV2(num_classes=num_classes, width=width, depth=depth, head_zeroinit=head_zeroinit)


# The paper's checkpoints (bit_paper.py:175-199) live on gs://, which this package does not fetch.
_SHORT = re.compile(r"^[LMS](-.*)?$")
_VANITY = ("FunMatch-224px-i1k82.8", "FunMatch-160px-i1k80.5")


def load(init_params, init_file, model_cfg, dont_load=()):
  """Parameters from the npz checkpoint `init_file` (bit_paper.py:159-204): a TF-dumped BiT checkpoint is
  converted (maybe_convert_big_transfer_format), then merged with `init_params` (names matching `dont_load`
  keep their init value).  The paper's short names ("M", "M-imagenet2012", "FunMatch-224px-...") name gs://
  files: they are refused with a request for a local copy."""
  from big_vision_b200 import utils as u
  if init_file in _VANITY or _SHORT.match(init_file):
    raise ValueError(f"'{init_file}' names a checkpoint on gs://bit_models, which is not fetched here: download "
                     "it and pass the local .npz path instead")
  params = maybe_convert_big_transfer_format(u.load_params(init_file))
  return common.merge_params(params, init_params, dont_load)


def maybe_convert_big_transfer_format(params_tf):
  """The legacy (TF) BiT layout -> this model's tree (bit_paper.py:207-257); any other tree unchanged."""
  from big_vision_b200 import utils as u
  if "resnet" not in params_tf:
    return params_tf
  params_tf = dict(u.tree_flatten_with_names(params_tf)[0])
  for k in list(params_tf):
    k2 = re.sub(r"/standardized_conv2d_\d+/", "/standardized_conv2d/", k)
    if k2 != k:
      params_tf[k2] = params_tf.pop(k)
  params = {
      "root_block": {"conv_root": {"kernel": params_tf["resnet/root_block/standardized_conv2d/kernel"]}},
      "norm-pre-head": {"bias": params_tf["resnet/group_norm/beta"][None, None, None],
                        "scale": params_tf["resnet/group_norm/gamma"][None, None, None]},
      "head": {"kernel": params_tf["resnet/head/conv2d/kernel"][0, 0], "bias": params_tf["resnet/head/conv2d/bias"]},
  }
  for block in ("block1", "block2", "block3", "block4"):
    params[block] = {}
    units = {re.findall(r"unit\d+", p)[0] for p in params_tf if p.find(block) >= 0}
    for unit in units:
      d = params[block][unit] = {}
      for i, group in enumerate("abc", 1):
        d[f"conv{i}"] = {"kernel": params_tf[f"resnet/{block}/{unit}/{group}/standardized_conv2d/kernel"]}
        d[f"gn{i}"] = {"bias": params_tf[f"resnet/{block}/{unit}/{group}/group_norm/beta"][None, None, None],
                       "scale": params_tf[f"resnet/{block}/{unit}/{group}/group_norm/gamma"][None, None, None]}
      projs = [p for p in params_tf if p.find(f"{block}/{unit}/a/proj") >= 0]
      assert len(projs) <= 1
      if projs:
        d["conv_proj"] = {"kernel": params_tf[projs[0]]}
  return params
