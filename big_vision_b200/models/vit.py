"""ViT on the H100 kernels -- host-side mirror of big_vision/models/vit.py.

Same factory (`Model(num_classes, variant=..., **kw)`), same fields, same parameter-tree
names/shapes as the reference (models/vit.py:186-281, param names SURVEY.md 8b); the
computation is an explicit forward + hand-written backward over the C-ABI kernels
(bv_gemm / bv_attention_* / bv_layernorm_* ...) instead of flax modules under jax.grad.

dtype flow (reference with dtype_mm="bfloat16", SURVEY.md 8a): residual stream bf16,
LayerNorm statistics fp32, every matmul bf16 x bf16 -> fp32 accumulate, parameters and
their gradients fp32.  Unlike the reference, the MAP head / heads also run their matmuls
in bf16 (fp32 accumulate, fp32 outputs); see DESIGN.md "numerics".
"""
import math
from dataclasses import dataclass, field
from typing import Optional, Sequence, Tuple, Union

import numpy as np
import torch

from big_vision_b200 import engine as E
from big_vision_b200 import lib as L
from big_vision_b200 import ops
from big_vision_b200.models import common


def posemb_sincos_2d(h, w, width, temperature=10_000.0):
  """Fixed 2-D sine/cosine position table [h*w, width] in the MoCo-v3 channel layout the reference
  uses (models/vit.py:34-44): the width is cut into four equal bands holding sin(x w_k), cos(x w_k),
  sin(y w_k), cos(y w_k) for the token at column x, row y (row-major token order), with frequencies
  w_k = temperature^(-k/(width/4 - 1))."""
  if width % 4:
    raise AssertionError("Width must be mult of 4 for sincos posemb")
  bands = width // 4
  freq = 1.0 / temperature ** (np.arange(bands) / (bands - 1))
  col = np.tile(np.arange(w), h)          # x of token t = t % w
  row = np.repeat(np.arange(h), w)        # y of token t = t // w
  ax, ay = np.outer(col, freq), np.outer(row, freq)
  return np.concatenate([np.sin(ax), np.cos(ax), np.sin(ay), np.cos(ay)], axis=1).astype(np.float32)


# name: (width, depth, mlp_dim, num_heads) -- the size table of models/vit.py:284-303
_VARIANTS = {
    "mu": (32, 1, 128, 2), "Ti": (192, 12, 768, 3), "S": (384, 12, 1536, 6), "M": (512, 12, 2048, 8),
    "B": (768, 12, 3072, 12), "L": (1024, 24, 4096, 16), "So400m": (1152, 27, 4304, 16),
    "H": (1280, 32, 5120, 16), "g": (1408, 40, 6144, 16), "g-opt": (1536, 40, 6144, 16),
    "G": (1664, 48, 8192, 16), "G-opt": (1536, 48, 8192, 16), "e": (1792, 56, 15360, 16),
}


def check_head_dim(width, num_heads):
  """Raises NotImplementedError unless width / num_heads is a head dim the attention kernels have."""
  if width % num_heads or width // num_heads not in ops.ATTN_HEAD_DIMS:
    raise NotImplementedError(
        f"width {width} / {num_heads} heads: the attention kernels are built for head dims "
        f"{', '.join(map(str, ops.ATTN_HEAD_DIMS))}")


def decode_variant(variant):
  """"B" / "B/16" -> dict(width, depth, mlp_dim, num_heads[, patch_size]); None -> {}."""
  if variant is None:
    return {}
  name, _, patch = variant.partition("/")
  width, depth, mlp_dim, num_heads = _VARIANTS[name]
  out = dict(width=width, depth=depth, mlp_dim=mlp_dim, num_heads=num_heads)
  if patch:
    out["patch_size"] = (int(patch), int(patch))
  return out


# ------------------------------------------------------------------------------------------
# building blocks (each: specs(), fwd(), bwd()); `P` is an engine.FlatParams
# ------------------------------------------------------------------------------------------
def _stacked(init, stack):
  """Initialiser of a scan-stacked parameter: `stack` independent draws along a new leading axis."""
  if not stack:
    return init
  return lambda rng, shape: np.stack([np.asarray(init(rng, tuple(shape[1:]))) for _ in range(shape[0])])


def _shape(shape, stack):
  return ((stack,) + tuple(shape)) if stack else tuple(shape)


def ln_specs(p, d, stack=0):
  return [E.ParamSpec(p + "scale", _shape((d,), stack), _stacked(E.ones, stack)),
          E.ParamSpec(p + "bias", _shape((d,), stack), _stacked(E.zeros, stack))]


def mlp_specs(p, d, m, stack=0):
  """MlpBlock (models/vit.py:57-78): xavier_uniform kernels, normal(1e-6) biases."""
  return [
      E.ParamSpec(p + "Dense_0/kernel", _shape((d, m), stack), _stacked(E.xavier_uniform(d, m), stack)),
      E.ParamSpec(p + "Dense_0/bias", _shape((m,), stack), _stacked(E.normal(1e-6), stack)),
      E.ParamSpec(p + "Dense_1/kernel", _shape((m, d), stack), _stacked(E.xavier_uniform(m, d), stack)),
      E.ParamSpec(p + "Dense_1/bias", _shape((d,), stack), _stacked(E.normal(1e-6), stack)),
  ]


class Scope:
  """A parameter sub-tree of a FlatParams: `S.f("Dense_0/kernel")` is the fp32 master of
  `prefix + "Dense_0/kernel"` (g: gradient, h: bf16 shadow).  With `index` the stored tensors carry
  a leading stack axis (the reference's scan=True layout, models/vit.py:129-148: one `encoderblock`
  sub-tree whose leaves have a leading `depth` axis) and the scope addresses slice `index` of it."""

  def __init__(self, P, prefix, index=None):
    self.P, self.prefix, self.index = P, prefix, index

  def _get(self, kind, name):
    full = self.prefix + name
    if self.index is None:
      return getattr(self.P, kind)(full)
    key = (kind, full, self.index)
    v = self.P._views.get(key)   # pylint: disable=protected-access
    if v is None:
      v = getattr(self.P, kind)(full)[self.index]
      self.P._views[key] = v     # pylint: disable=protected-access
    return v

  def f(self, name):
    return self._get("f", name)

  def g(self, name):
    return self._get("g", name)

  def h(self, name):
    return self._get("h", name)

  def sub(self, rel):
    return Scope(self.P, self.prefix + rel, self.index)


def mlp_fwd(S, y, resid, out_dtype=torch.bfloat16, save=True, drop=None):
  """resid + Dense_1(gelu(Dense_0(y))) with S the MlpBlock's Scope.  Returns (out, saved).
  save=False (forward only): GELU's pre-activation is not written at all, saved is None.
  drop: None, or the lib.DropoutKeys (GELU output, MLP output) of the encoder block's dropouts
  (models/vit.py:76,109): the GELU output is dropped in place, so the saved activation is the dropped one,
  and the residual add follows the dropped Dense_1 output.  A GELU key of None leaves the GELU output as it
  is (BERT drops the MLP output only)."""
  if save:
    act, pre = ops.gemm(y, S.h("Dense_0/kernel"), b_mn=True, bias=S.f("Dense_0/bias"),
                        epilogue=L.EPI_BIAS_GELU)
  else:
    act = ops.gemm(y, S.h("Dense_0/kernel"), b_mn=True, bias=S.f("Dense_0/bias"),
                   epilogue=L.EPI_BIAS_GELU_ACT)
  if drop is not None:
    if drop[0] is not None:
      ops.dropout(act, drop[0], out=act)
    out = ops.gemm(act, S.h("Dense_1/kernel"), b_mn=True, bias=S.f("Dense_1/bias"))
    out = ops.dropout_add(resid, out, drop[1], out=out)
  else:
    out = ops.gemm(act, S.h("Dense_1/kernel"), b_mn=True, bias=S.f("Dense_1/bias"),
                   aux=resid, epilogue=L.EPI_BIAS_RESID if resid is not None else L.EPI_BIAS,
                   out_dtype=out_dtype)
  return out, ((y, act, pre) if save else None)


def mlp_bwd(S, dout, saved, want_bias2_grad=True, gelu_drop=None):
  """dout: bf16 [M,d] gradient of the block output.  Returns d(y) (bf16).

  The bias gradient of Dense_1 is colsum(dout); callers that already have that column sum
  from the LayerNorm-backward kernel pass want_bias2_grad=False.  gelu_drop: the lib.DropoutKey of the
  forward's GELU-output dropout, or None; its mask is applied to d(GELU pre-activation), which equals
  masking the GELU output's gradient since both are element-wise products."""
  y, act, pre = saved
  if want_bias2_grad:
    ops.colsum(dout, S.g("Dense_1/bias"))
  ops.gemm(act, dout, a_mn=True, b_mn=True, out=S.g("Dense_1/kernel"), reduce_out=True)
  if gelu_drop is not None:
    dpre = ops.gemm(dout, S.h("Dense_1/kernel"), aux=pre, epilogue=L.EPI_DGELU)
    ops.dropout(dpre, gelu_drop, out=dpre, colsum_into=S.g("Dense_0/bias"))
  else:
    # the Dense_0 bias gradient (column sums of dpre) is accumulated by the same GEMM's epilogue
    dpre = ops.gemm(dout, S.h("Dense_1/kernel"), aux=pre, epilogue=L.EPI_DGELU,
                    colsum=S.g("Dense_0/bias"))
  ops.gemm(y, dpre, a_mn=True, b_mn=True, out=S.g("Dense_0/kernel"), reduce_out=True)
  return ops.gemm(dpre, S.h("Dense_0/kernel"))


def mha_specs(p, d, heads, fuse_qkv=True, stack=0):
  """flax MultiHeadDotProductAttention params: query/key/value kernels [d,h,dh] + bias [h,dh],
  out kernel [h,dh,d] + bias [d]; kernel_init xavier_uniform (models/vit.py:95,177), zero biases.
  Stored fused ([d,3d] or q:[d,d] + kv:[d,2d]) and aliased to the reference names.  `stack` > 0
  adds the leading scan axis to every stored tensor and every alias."""
  dh = d // heads
  xav = E.xavier_uniform(d, d)
  ax = 1 if stack else 0          # axis of the `d` input features in the stored kernels

  def fused_init(k):
    return _stacked(lambda rng, shape: np.concatenate([xav(rng, (d, d)) for _ in range(k)], axis=1), stack)

  specs, aliases = [], []

  def alias_cols(store, names):
    for i, nm in enumerate(names):
      aliases.append(E.Alias(p + nm + "/kernel", p + store + "/kernel",
                             lambda t, i=i: t.narrow(ax + 1, i * d, d).unflatten(ax + 1, (heads, dh))))
      aliases.append(E.Alias(p + nm + "/bias", p + store + "/bias",
                             lambda t, i=i: t.narrow(ax, i * d, d).unflatten(ax, (heads, dh))))

  if fuse_qkv:
    specs += [E.ParamSpec(p + "qkv/kernel", _shape((d, 3 * d), stack), fused_init(3)),
              E.ParamSpec(p + "qkv/bias", _shape((3 * d,), stack), _stacked(E.zeros, stack))]
    alias_cols("qkv", ["query", "key", "value"])
  else:
    specs += [E.ParamSpec(p + "q/kernel", _shape((d, d), stack), _stacked(xav, stack)),
              E.ParamSpec(p + "q/bias", _shape((d,), stack), _stacked(E.zeros, stack)),
              E.ParamSpec(p + "kv/kernel", _shape((d, 2 * d), stack), fused_init(2)),
              E.ParamSpec(p + "kv/bias", _shape((2 * d,), stack), _stacked(E.zeros, stack))]
    alias_cols("q", ["query"])
    alias_cols("kv", ["key", "value"])
  specs += [E.ParamSpec(p + "out_proj/kernel", _shape((d, d), stack), _stacked(xav, stack)),
            E.ParamSpec(p + "out/bias", _shape((d,), stack), _stacked(E.zeros, stack))]
  aliases.append(E.Alias(p + "out/kernel", p + "out_proj/kernel",
                         lambda t: t.unflatten(ax, (heads, dh))))
  return specs, aliases


class EncoderBlock(E.Stage):
  """Encoder1DBlock (models/vit.py:81-112): x + MHSA(LN(x)); x + MLP(LN(x)).
  `index` = position in the scan-stacked `encoderblock` sub-tree (None: own `encoderblock_{i}`); `layer` = the
  block's depth in its encoder, which selects its dropout masks (default: index)."""

  def __init__(self, prefix, d, m, heads, index=None, layer=None):
    self.p, self.d, self.m, self.heads, self.index = prefix, d, m, heads, index
    self.layer = index if layer is None else layer
    self.prefixes = (prefix,)
    # every parameter from this block on (in spec order) has its final gradient after its backward: a
    # data-parallel trainer can start reducing them while the earlier blocks are still running
    self.ready = prefix + "LayerNorm_0/scale" if index is None else None

  def specs(self, stack=0):
    att = self.p + "MultiHeadDotProductAttention_0/"
    s, a = mha_specs(att, self.d, self.heads, stack=stack)
    return (ln_specs(self.p + "LayerNorm_0/", self.d, stack) + s + ln_specs(self.p + "LayerNorm_1/", self.d, stack)
            + mlp_specs(self.p + "MlpBlock_0/", self.d, self.m, stack)), a

  def scope(self, P):
    return Scope(P, self.p, self.index)

  def fwd(self, P, x, geom, save=True):
    """save=False (forward only): same output bits; every intermediate is released as soon as the
    next op has consumed it and saved is None."""
    n, N = geom.n, geom.N
    d = self.d
    S = self.scope(P)
    A = S.sub("MultiHeadDotProductAttention_0/")
    ln1, mean1, rstd1 = ops.layernorm_fwd(x, S.f("LayerNorm_0/scale"), S.f("LayerNorm_0/bias"))
    qkv = ops.gemm(ln1, A.h("qkv/kernel"), b_mn=True, bias=A.f("qkv/bias"))
    qkv3 = qkv.view(n, N, 3 * d)
    o, lse = ops.attention_fwd(qkv3[:, :, 0:d], qkv3[:, :, d:2 * d], qkv3[:, :, 2 * d:], self.heads)
    if not save:
      del ln1, mean1, rstd1, qkv, qkv3, lse
    dr = geom.dropout
    if dr is None:
      x1 = ops.gemm(o.view(n * N, d), A.h("out_proj/kernel"), b_mn=True,
                    bias=A.f("out/bias"), aux=x, epilogue=L.EPI_BIAS_RESID)
    else:    # models/vit.py:100: the attention output is dropped before the residual add
      x1 = ops.gemm(o.view(n * N, d), A.h("out_proj/kernel"), b_mn=True, bias=A.f("out/bias"))
      x1 = ops.dropout_add(x, x1, dr.mask(self.layer, E.DROP_ATTN), out=x1)
    if not save:
      del o
    ln2, mean2, rstd2 = ops.layernorm_fwd(x1, S.f("LayerNorm_1/scale"), S.f("LayerNorm_1/bias"))
    drop = None if dr is None else (dr.mask(self.layer, E.DROP_GELU), dr.mask(self.layer, E.DROP_MLP))
    if not save:
      del mean2, rstd2
      x2, _ = mlp_fwd(S.sub("MlpBlock_0/"), ln2, x1, save=False, drop=drop)
      return x2, None
    x2, mlp_saved = mlp_fwd(S.sub("MlpBlock_0/"), ln2, x1, drop=drop)
    return x2, (x, ln1, mean1, rstd1, qkv, o, lse, x1, mean2, rstd2, mlp_saved)

  def sink(self, P, geom):
    """colsum(d block-output) is the gradient of this block's MlpBlock Dense_1 bias.  Under dropout that
    bias sees the masked gradient, so the block offers no sink and sums it itself (bwd)."""
    return None if geom.dropout else self.scope(P).g("MlpBlock_0/Dense_1/bias")

  def bwd(self, P, dx2, saved, geom, sink, need_dx=True):
    """dx2: bf16 [M,d] grad of block output; without dropout colsum(dx2) has ALREADY been accumulated
    into this block's Dense_1 bias grad by whoever produced dx2 (sink).  Returns dx (grad of block input);
    colsum(dx) is accumulated into `sink` (the bias gradient of the stage below).  Under dropout the
    gradients entering the MLP and the attention output projection are masked as in the forward; the
    residual stream's gradient is not."""
    n, N = geom.n, geom.N
    d = self.d
    S = self.scope(P)
    A = S.sub("MultiHeadDotProductAttention_0/")
    x, ln1, mean1, rstd1, qkv, o, lse, x1, mean2, rstd2, mlp_saved = saved
    dr = geom.dropout
    if dr is None:
      dln2 = mlp_bwd(S.sub("MlpBlock_0/"), dx2, mlp_saved, want_bias2_grad=False)
    else:
      dm = ops.dropout(dx2, dr.mask(self.layer, E.DROP_MLP), colsum_into=S.g("MlpBlock_0/Dense_1/bias"))
      dln2 = mlp_bwd(S.sub("MlpBlock_0/"), dm, mlp_saved, want_bias2_grad=False,
                     gelu_drop=dr.mask(self.layer, E.DROP_GELU))
      del dm
    dx1 = ops.layernorm_bwd(dln2, x1, S.f("LayerNorm_1/scale"), mean2, rstd2, dres=dx2,
                            dscale=S.g("LayerNorm_1/scale"), dbias=S.g("LayerNorm_1/bias"),
                            dx_colsum=A.g("out/bias") if dr is None else None)
    del dln2
    da = dx1 if dr is None else ops.dropout(dx1, dr.mask(self.layer, E.DROP_ATTN), colsum_into=A.g("out/bias"))
    o2 = o.view(n * N, d)
    ops.gemm(o2, da, a_mn=True, b_mn=True, out=A.g("out_proj/kernel"), reduce_out=True)
    do = ops.gemm(da, A.h("out_proj/kernel"))
    del da
    qkv3 = qkv.view(n, N, 3 * d)
    dqkv = torch.empty_like(qkv)
    dqkv3 = dqkv.view(n, N, 3 * d)
    gb = A.g("qkv/bias")     # q|k|v bias gradients come out of the attention backward
    ops.attention_bwd(do.view(n, N, d), qkv3[:, :, 0:d], qkv3[:, :, d:2 * d], qkv3[:, :, 2 * d:],
                      o, lse, self.heads, dq=dqkv3[:, :, 0:d], dk=dqkv3[:, :, d:2 * d],
                      dv=dqkv3[:, :, 2 * d:], dq_colsum=gb[0:d], dk_colsum=gb[d:2 * d],
                      dv_colsum=gb[2 * d:])
    del do
    ops.gemm(ln1, dqkv, a_mn=True, b_mn=True, out=A.g("qkv/kernel"), reduce_out=True)
    dln1 = ops.gemm(dqkv, A.h("qkv/kernel"))
    del dqkv
    dx = ops.layernorm_bwd(dln1, x, S.f("LayerNorm_0/scale"), mean1, rstd1, dres=dx1,
                           dscale=S.g("LayerNorm_0/scale"), dbias=S.g("LayerNorm_0/bias"),
                           dx_colsum=sink)
    return dx


class ScanEncoder(E.Stage):
  """The encoder blocks as the reference's nn.scan over ONE `encoderblock` whose parameters carry a
  leading depth axis, each iteration wrapped in nn.remat with policy `nothing_saveable`
  (models/vit.py:129-148): only the block INPUT survives the forward and the block is recomputed in
  the backward, which is what makes L/14@336 at 2048 pairs per GPU fit in HBM.  One backward stage:
  a single storage holds every block."""

  def __init__(self, prefix, depth, d, m, heads, remat_policy="nothing_saveable"):
    if remat_policy not in ("nothing_saveable", None):
      raise NotImplementedError(f"remat_policy={remat_policy!r}: only nothing_saveable (recompute the "
                                "whole block) is built")
    self.blocks = [EncoderBlock(f"{prefix}encoderblock/", d, m, heads, index=i) for i in range(depth)]
    self.prefixes = (self.blocks[0].p,)

  def specs(self):
    return self.blocks[0].specs(stack=len(self.blocks))

  def fwd(self, P, x, geom, save=True):
    saved = [] if save else None
    for b in self.blocks:
      if save:
        saved.append(x)                           # remat: keep the block input only
      x, _ = b.fwd(P, x, geom, save)
    return x, saved

  def sink(self, P, geom):
    return self.blocks[-1].sink(P, geom)

  def bwd(self, P, dx, saved, geom, sink, need_dx=True):
    for i in reversed(range(len(self.blocks))):
      x_out, s = self.blocks[i].fwd(P, saved[i], geom)    # recompute the block from its input
      del x_out
      dx = self.blocks[i].bwd(P, dx, s, geom, self.blocks[i - 1].sink(P, geom) if i else sink)
      saved[i] = s = None
    return dx


def encoder_stages(prefix, depth, d, m, heads, scan=False, remat_policy="nothing_saveable"):
  """The blocks of vit.Encoder (models/vit.py:115-160) as backward stages: one per `encoderblock_{i}`
  (models/vit.py:151-158), or one ScanEncoder with scan=True."""
  if scan:
    return [ScanEncoder(prefix, depth, d, m, heads, remat_policy)]
  return [EncoderBlock(f"{prefix}encoderblock_{i}/", d, m, heads, layer=i) for i in range(depth)]


class NormPool(E.Stage):
  """encoder_norm (models/vit.py:160) and the pooling that follows it.  `pool`: "mean"; "first" or
  "last" (one token); "max"; None (no pooling: LN only, for the MAP head and pool_type "none").  A
  pooled output has dtype `out_dtype`; an unpooled one is bf16."""

  def __init__(self, prefix, d, pool, out_dtype):
    self.p, self.d, self.pool = prefix, d, pool
    self.out_dtype = out_dtype if pool else torch.bfloat16
    self.prefixes = (prefix,)

  def specs(self):
    return ln_specs(self.p, self.d), []

  def _tok(self, N):
    return 0 if self.pool == "first" else N - 1

  def fwd(self, P, x, geom, save=True):
    n, N = geom.n, geom.N
    scale, bias = P.f(self.p + "scale"), P.f(self.p + "bias")
    if self.pool in ("first", "last"):
      # LayerNorm is per token: LN(x)[:, t] == LN(x[:, t]) -- select first, normalise one row
      x = ops.pool_fwd(x, n, N, 1, tok=self._tok(N))
      y, mean, rstd = ops.layernorm_fwd(x, scale, bias, out_dtype=self.out_dtype)
      return y, ((x, mean, rstd, None) if save else None)
    encd, mean, rstd = ops.layernorm_fwd(x, scale, bias)
    saved = (x, mean, rstd, encd if self.pool == "max" else None) if save else None
    if self.pool == "mean":
      return ops.pool_fwd(encd, n, N, 0, out_dtype=self.out_dtype), saved
    if self.pool == "max":
      return ops.pool_fwd(encd, n, N, 2, out_dtype=self.out_dtype), saved
    return encd, saved

  def bwd(self, P, dy, saved, geom, sink, need_dx=True):
    n, N = geom.n, geom.N
    x, mean, rstd, encd = saved
    if dy.dtype != self.out_dtype:
      dy = ops.cast(dy, torch.empty_like(dy, dtype=self.out_dtype))
    grads = dict(dscale=P.g(self.p + "scale"), dbias=P.g(self.p + "bias"), dx_colsum=sink)
    if self.pool in ("first", "last"):
      dx = ops.layernorm_bwd(dy, x, P.f(self.p + "scale"), mean, rstd, **grads)
      return ops.pool_bwd(dx, n, N, 1, tok=self._tok(N)) if need_dx else None
    if self.pool == "mean":
      dy = ops.pool_bwd(dy, n, N, 0)
    elif self.pool == "max":
      dy = ops.pool_max_bwd(dy, encd, n, N)
    return ops.layernorm_bwd(dy, x, P.f(self.p + "scale"), mean, rstd, **grads)


class MAPHead(E.Stage):
  """Multihead attention pooling (models/vit.py:163-183).  Its MLP writes fp32; with out_dtype bf16 (the
  text tower's) the output is cast to bf16, and the backward casts the bf16 output gradient to fp32
  before it proceeds as for an fp32 output."""

  def __init__(self, prefix, d, m, heads, out_dtype=torch.float32):
    self.p, self.d, self.m, self.heads, self.out_dtype = prefix, d, m, heads, out_dtype
    self.att = prefix + "MultiHeadDotProductAttention_0/"
    self.prefixes = (prefix,)

  def specs(self):
    d = self.d
    s, a = mha_specs(self.att, d, self.heads, fuse_qkv=False)
    probe = E.ParamSpec(self.p + "probe", (1, 1, d), E.xavier_uniform(1, d))
    return ([probe] + s + ln_specs(self.p + "LayerNorm_0/", d)
            + mlp_specs(self.p + "MlpBlock_0/", d, self.m)), a

  def fwd(self, P, enc, geom, save=True):
    n, N = geom.n, geom.N
    d = self.d
    q1 = ops.gemm(P.h(self.p + "probe").view(1, d), P.h(self.att + "q/kernel"), b_mn=True,
                  bias=P.f(self.att + "q/bias"))
    qn = ops.broadcast_row(q1, n)
    kv = ops.gemm(enc, P.h(self.att + "kv/kernel"), b_mn=True, bias=P.f(self.att + "kv/bias"))
    kv3 = kv.view(n, N, 2 * d)
    o, lse = ops.attention_fwd(qn.view(n, 1, d), kv3[:, :, 0:d], kv3[:, :, d:], self.heads)
    if not save:
      del kv, kv3, lse
    a = ops.gemm(o.view(n, d), P.h(self.att + "out_proj/kernel"), b_mn=True, bias=P.f(self.att + "out/bias"))
    y, mean, rstd = ops.layernorm_fwd(a, P.f(self.p + "LayerNorm_0/scale"), P.f(self.p + "LayerNorm_0/bias"))
    out, mlp_saved = mlp_fwd(Scope(P, self.p + "MlpBlock_0/"), y, a, out_dtype=torch.float32, save=save)
    if self.out_dtype != torch.float32:
      out = ops.cast(out, torch.empty_like(out, dtype=self.out_dtype))
    if not save:
      return out, None
    return out, (enc, qn, kv, o, lse, a, mean, rstd, mlp_saved)

  def bwd(self, P, dout, saved, geom, sink=None, need_dx=True):
    """dout [n,d] in out_dtype -> d(enc) bf16 [n*N, d] (None with need_dx=False)."""
    n, N = geom.n, geom.N
    d = self.d
    enc, qn, kv, o, lse, a, mean, rstd, mlp_saved = saved
    if self.out_dtype != torch.float32:
      dout = ops.cast(dout, torch.empty_like(dout, dtype=torch.float32))
    dout16 = ops.cast(dout, torch.empty_like(dout, dtype=torch.bfloat16))
    dy = mlp_bwd(Scope(P, self.p + "MlpBlock_0/"), dout16, mlp_saved, want_bias2_grad=True)
    da = ops.layernorm_bwd(dy, a, P.f(self.p + "LayerNorm_0/scale"), mean, rstd, dres=dout16,
                           dscale=P.g(self.p + "LayerNorm_0/scale"), dbias=P.g(self.p + "LayerNorm_0/bias"),
                           dx_colsum=P.g(self.att + "out/bias"))
    ops.gemm(o.view(n, d), da, a_mn=True, b_mn=True, out=P.g(self.att + "out_proj/kernel"), reduce_out=True)
    do = ops.gemm(da, P.h(self.att + "out_proj/kernel"))
    kv3 = kv.view(n, N, 2 * d)
    dkv = torch.empty_like(kv)
    dkv3 = dkv.view(n, N, 2 * d)
    dq = torch.empty_like(qn)
    ops.attention_bwd(do.view(n, 1, d), qn.view(n, 1, d), kv3[:, :, 0:d], kv3[:, :, d:], o, lse,
                      self.heads, dq=dq.view(n, 1, d), dk=dkv3[:, :, 0:d], dv=dkv3[:, :, d:])
    ops.colsum(dkv, P.g(self.att + "kv/bias"))
    ops.gemm(enc, dkv, a_mn=True, b_mn=True, out=P.g(self.att + "kv/kernel"), reduce_out=True)
    denc = ops.gemm(dkv, P.h(self.att + "kv/kernel")) if need_dx else None
    # the single probe query is shared by the batch: its gradient is the batch sum of dq
    dq1 = torch.zeros(d, dtype=torch.float32, device=dq.device)
    ops.colsum(dq, dq1)
    ops.axpby(P.g(self.att + "q/bias"), dq1, 1.0, 1.0, out=P.g(self.att + "q/bias"))
    dq1h = ops.cast(dq1, torch.empty(d, dtype=torch.bfloat16, device=dq.device)).view(1, d)
    ops.gemm(P.h(self.p + "probe").view(1, d), dq1h, a_mn=True, b_mn=True,
             out=P.g(self.att + "q/kernel"), reduce_out=True)
    ops.gemm(dq1h, P.h(self.att + "q/kernel"), out=P.g(self.p + "probe").view(1, d), reduce_out=True)
    return denc


class PatchEmbedding(E.Stage):
  """The patch embedding (models/vit.py:212-225) of [n, *image_hw, in_ch] images: a Dense over flattened
  patches, stored under `prefix + name`, with the position embedding added in its epilogue, then [cls]
  prepended when `cls`.  posemb=None adds no position embedding: the MLP-Mixer's stem
  (models/mlp_mixer.py:72).  `tokens`: the output's tokens per image."""

  def __init__(self, prefix, name, image_hw, patch_size, in_ch, d, posemb, cls):
    self.p, self.patch_size, self.in_ch, self.d, self.posemb, self.cls = prefix, patch_size, in_ch, d, posemb, cls
    self.grid = (image_hw[0] // patch_size[0], image_hw[1] // patch_size[1])
    self.tokens = self.grid[0] * self.grid[1] + cls
    self.w = prefix + name + "/"
    self.prefixes = ((self.w,) + ((prefix + "pos_embedding",) if posemb == "learn" else ())
                     + ((prefix + "cls",) if cls else ()))
    self._sincos = None

  def specs(self):
    """The kernel is stored flattened [ph*pw*in_ch, d] (the im2col column order), padded to a multiple
    of 8 rows, and exposed under `kernel` as [ph, pw, in_ch, d]."""
    (ph, pw), (gh, gw), d, w, in_ch = self.patch_size, self.grid, self.d, self.w, self.in_ch
    K = ph * pw * in_ch
    Kp = (K + 7) // 8 * 8
    lec = E.lecun_normal(K)   # flax Conv default kernel_init, fan_in = ph*pw*C
    specs = [E.ParamSpec(w + "kernel_flat", (Kp, d),
                         lambda rng, shape: np.concatenate([lec(rng, (K, d)), np.zeros((Kp - K, d))], 0)),
             E.ParamSpec(w + "bias", (d,), E.zeros)]
    aliases = [E.Alias(w + "kernel", w + "kernel_flat", lambda t: t[:K].unflatten(0, (ph, pw, in_ch)))]
    if self.posemb == "learn":
      specs.append(E.ParamSpec(self.p + "pos_embedding", (1, gh * gw, d), E.normal(1 / math.sqrt(d))))
    if self.cls:
      specs.append(E.ParamSpec(self.p + "cls", (1, 1, d), E.zeros))
    return specs, aliases

  def _posemb16(self, P):
    if self.posemb == "learn":
      return P.h(self.p + "pos_embedding").view(-1, self.d)
    if self._sincos is None or self._sincos.device != P.device:
      self._sincos = torch.from_numpy(posemb_sincos_2d(*self.grid, self.d)).to(P.device).bfloat16()
    return self._sincos

  def fwd(self, P, image, geom, save=True):
    n, N = geom.n, geom.N
    N0, w = N - self.cls, self.w
    patches = ops.patchify(image, self.patch_size[0])
    if self.posemb:
      x = ops.gemm(patches, P.h(w + "kernel_flat"), b_mn=True, bias=P.f(w + "bias"),
                   aux=self._posemb16(P), aux_row_mod=N0, epilogue=L.EPI_BIAS_RESID)
    else:
      x = ops.gemm(patches, P.h(w + "kernel_flat"), b_mn=True, bias=P.f(w + "bias"))
    saved = patches if save else None
    del patches
    if self.cls:
      # cls token is prepended AFTER the position embedding was added (models/vit.py:223-225)
      x = ops.concat_cls(x, P.f(self.p + "cls").view(self.d), n, N0)
    if geom.dropout is not None:     # models/vit.py:228
      ops.dropout(x, geom.dropout.mask(0, E.DROP_EMBED), out=x)
    return x, saved

  def sink(self, P, geom):
    # the column sum of the gradient reaching the embedding output is the patch-embed bias gradient
    # (models/vit.py:212-214); with [cls] it is summed over the patch tokens only, and under dropout over
    # the masked gradient (bwd)
    return None if self.cls or geom.dropout else P.g(self.w + "bias")

  def bwd(self, P, dx, patches, geom, sink=None, need_dx=False):
    n, N = geom.n, geom.N
    d, p = self.d, self.p
    if geom.dropout is not None:
      dx = ops.dropout(dx, geom.dropout.mask(0, E.DROP_EMBED), colsum_into=None if self.cls else P.g(self.w + "bias"))
    if self.cls:
      # batch-sum of the gradient at every token position: row 0 is d cls, the rest d pos_embedding;
      # the patch-embed bias gradient is the sum of the latter over positions
      N0 = N - 1
      tmp = torch.zeros(N * d, dtype=torch.float32, device=dx.device)
      ops.colsum(dx.view(n, N * d), tmp)
      gcls = P.g(p + "cls").view(d)
      ops.axpby(gcls, tmp[:d], 1.0, 1.0, out=gcls)
      if self.posemb == "learn":
        gpos = P.g(p + "pos_embedding").view(N0 * d)
        ops.axpby(gpos, tmp[d:], 1.0, 1.0, out=gpos)
      ops.colsum(tmp[d:].view(N0, d), P.g(self.w + "bias"))
      dx = ops.drop_cls(dx, n, N0)
    elif self.posemb == "learn":
      ops.colsum(dx.view(n, N * d), P.g(p + "pos_embedding").view(N * d))
    ops.gemm(patches, dx, a_mn=True, b_mn=True, out=P.g(self.w + "kernel_flat"), reduce_out=True)


# ------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------
_POOLS = {"gap": "mean", "0": "first", "tok": "first", "map": None, "none": None}   # -> NormPool's pool


@dataclass
class _Model(E.Staged):
  """ViT model; fields as in models/vit.py:186-204."""
  num_classes: Optional[int] = None
  patch_size: Sequence[int] = (16, 16)
  width: int = 768
  depth: int = 12
  mlp_dim: Optional[int] = None
  num_heads: int = 12
  posemb: str = "learn"
  rep_size: Union[int, bool] = False
  dropout: float = 0.0
  pool_type: str = "gap"
  head_zeroinit: bool = True
  scan: bool = False
  remat_policy: str = "nothing_saveable"
  dtype_mm: str = "bfloat16"
  name: str = ""

  def __post_init__(self):
    E.check_dropout_rate(self.dropout)
    if self.pool_type not in _POOLS:
      raise ValueError(f"Unknown pool type: '{self.pool_type}'")
    check_head_dim(self.width, self.num_heads)
    self.mlp = self.mlp_dim or 4 * self.width
    self.prefix = (self.name + "/") if self.name else ""

  # ---- parameters ------------------------------------------------------------------------
  def specs(self, image_hw, in_ch=3):
    """Builds the backward stages for [n, *image_hw, in_ch] images -> (specs, aliases)."""
    p, d, enc = self.prefix, self.width, self.prefix + "Transformer/"
    rep = (d if self.rep_size is True else self.rep_size) if self.rep_size else d
    head_init = E.zeros if self.head_zeroinit else E.lecun_normal(rep)
    self.head = common.Dense(p + "head/", rep, self.num_classes, head_init, pad=True) if self.num_classes else None
    # bottom-up; parameterless pools belong to no stage of their own
    embed = PatchEmbedding(p, "embedding", image_hw, self.patch_size, in_ch, d, self.posemb, self.pool_type == "tok")
    stages = ([embed] + encoder_stages(enc, self.depth, d, self.mlp, self.num_heads, self.scan, self.remat_policy)
              + [NormPool(enc + "encoder_norm/", d, _POOLS[self.pool_type], torch.float32)])
    if self.pool_type == "map":
      stages.append(MAPHead(p + "MAPHead_0/", d, self.mlp, self.num_heads))
    if self.rep_size:   # models/vit.py:258-265
      stages.append(common.Dense(p + "pre_logits/", d, rep, E.lecun_normal(d), tanh=True))
    if self.head is not None:
      stages.append(self.head)
    return self._build(stages)

  def init(self, seed, image_shape, device="cuda"):
    """Counterpart of model.init(rng, zeros_image)["params"] (train.py:195-205)."""
    specs, aliases = self.specs(image_shape[1:3], image_shape[3])
    return E.FlatParams(specs, aliases, device).init(seed)

  # ---- forward / backward ----------------------------------------------------------------
  def fwd(self, P, image, frozen=None, dropout=None):
    """image [n,H,W,C] fp32 in [-1,1] (the shape given to specs()) -> (x fp32 [n, out], saved).  With a
    class head whose storage is padded (common.Dense) x is the [n, num_classes] view of the padded logits.

    `frozen`: storage names that receive no gradient (optax.Chain.frozen()), or True for all of them
    (inference).  Stages below the cut (see cut()) run forward-only and save nothing; the output is
    bit-identical either way.  `dropout`: the engine.DropoutKey of a training forward; without one (or at
    rate 0) no dropout is applied, as with train=False.  Frozen stages drop too."""
    n, N = image.shape[0], self._stages[0].tokens
    geom = E.Geom(n, N, dropout=E.dropout(self.dropout, dropout, N))
    out, saved = self._stages_fwd(P, image, geom, frozen)
    if self.pool_type == "none":
      # no pooling (models/vit.py:252-253): pre_logits / head run on every token, out is [n, N, .]
      if out.dtype != torch.float32:
        out = ops.cast(out, torch.empty_like(out, dtype=torch.float32))
      out = out.view(n, N, -1)
    return out, saved

  def bwd(self, P, dout, saved):
    """dout: fp32 [n, out] ([n, N, out] without pooling).  Accumulates parameter gradients into P.grad.
    With a padded class head, out is the padded class count (common.Dense.bwd)."""
    if self.pool_type == "none":
      geom = saved["geom"]
      dout = dout.reshape(geom.n * geom.N, -1)
    self._stages_bwd(P, dout, saved)

  # ---- reference-style entry points --------------------------------------------------------
  def apply(self, variables, image, *, train=False):
    """(x, out) like flax apply (models/vit.py:206-276); `out` holds what this path keeps.  train=True
    with dropout needs a key, which apply() has no argument for: use fwd(..., dropout=key)."""
    if train and self.dropout:
      raise ValueError("apply(train=True) with dropout > 0 has no dropout key; call fwd(..., dropout=key)")
    P = variables["params"]
    x, _ = self.fwd(P, image, frozen=True)     # no backward follows: forward-only, same bits
    out = {"head_input": x} if not (self.rep_size or self.num_classes) else {}
    out["pre_logits" if not self.num_classes else "logits"] = x
    return x, out


def Model(num_classes=None, *, variant=None, **kw):  # pylint: disable=invalid-name
  """Factory, same signature as big_vision.models.vit.Model (models/vit.py:279-281)."""
  return _Model(num_classes, **{**decode_variant(variant), **kw})


# ----------------------------------------------------------------------------------------------
# Checkpoint interchange (host side; nested dicts of numpy arrays under the reference's names).
# Contract of models/vit.py:306-433: accept every on-disk generation of ViT checkpoints the
# reference accepts and deliver a tree shaped like the model's freshly initialised parameters.
# ----------------------------------------------------------------------------------------------
def resample_posemb(old, new):
  """Position embeddings for a different input resolution ("high-res finetuning"): the square
  [1, g*g, d] grid `old` is bilinearly resized (order-1 spline, scipy.ndimage.zoom) to the grid size
  of `new`; returned unchanged when the shapes already agree."""
  old = np.asarray(old)
  want = tuple(new.shape)
  if old.shape == want:
    return old
  import scipy.ndimage
  side_from, side_to = (int(np.sqrt(shape[1])) for shape in (old.shape, want))
  ratio = side_to / side_from
  resized = scipy.ndimage.zoom(old.reshape(side_from, side_from, -1), (ratio, ratio, 1), order=1)
  return resized.reshape(1, side_to * side_to, -1)


# Older checkpoint generations, oldest quirk first; each entry rewrites the top-level tree in place.
def _posemb_out_of_encoder(tree):
  """The position embedding used to be a parameter of the encoder ("Transformer/pos_embedding", and
  before that of a "posembed_input" sub-module); today it is a top-level parameter."""
  enc = tree.get("Transformer")
  if not isinstance(enc, dict):
    return
  enc = tree["Transformer"] = dict(enc)
  if "posembed_input" in enc:
    tree["pos_embedding"] = enc.pop("posembed_input")["pos_embedding"]
  if "pos_embedding" in enc:
    tree["pos_embedding"] = enc.pop("pos_embedding")


def _cls_out_of_posemb(tree):
  """[cls] used to be concatenated BEFORE the position embedding was added, so old tables have
  g*g + 1 rows; the extra first row is folded into the cls parameter."""
  table = tree.get("pos_embedding")
  if table is None:
    return
  rows = int(table.shape[1])
  grid = int(np.sqrt(rows))
  if grid * grid + 1 != rows:
    return
  tree["pos_embedding"] = table[:, 1:]
  if "cls" in tree:
    tree["cls"] = tree["cls"] + table[:, :1]


def _map_head_into_module(tree):
  """The MAP head was written inline at first; its four parameter groups now live in "MAPHead_0"."""
  if "probe" not in tree:
    return
  moved = ("probe", "MlpBlock_0", "MultiHeadDotProductAttention_0", "LayerNorm_0")
  tree["MAPHead_0"] = {name: tree.pop(name) for name in moved}


_CHECKPOINT_FIXES = (_posemb_out_of_encoder, _cls_out_of_posemb, _map_head_into_module)


def fix_old_checkpoints(params):
  """Brings a ViT parameter tree of any older generation to today's layout (a new top-level dict;
  the input is not modified).  Pre-linen checkpoints cannot occur in .npz files written by
  linen-era code and are not handled."""
  tree = dict(params)
  for fix in _CHECKPOINT_FIXES:
    fix(tree)
  return tree


def _block_names(encoder_tree):
  names = [k for k in encoder_tree if k.startswith("encoderblock_")]
  return sorted(names, key=lambda k: int(k.rsplit("_", 1)[1]))


def _zip_trees(fn, trees):
  """fn over corresponding leaves of identically shaped dict trees."""
  first = trees[0]
  if isinstance(first, dict):
    return {k: _zip_trees(fn, [t[k] for t in trees]) for k in first}
  return fn(trees)


def pyloop_to_scan(params_pyloop, encoder="Transformer"):
  """Per-layer sub-trees "encoderblock_0..L-1" of the Python-loop encoder -> the single
  "encoderblock" of the scanned encoder, every leaf stacked along a new leading layer axis."""
  out = dict(params_pyloop)
  enc = dict(out[encoder])
  layers = _block_names(enc)
  if [int(k.rsplit("_", 1)[1]) for k in layers] != list(range(len(layers))):
    raise ValueError(f"encoder blocks are not numbered 0..{len(layers) - 1}: {layers}")
  enc["encoderblock"] = _zip_trees(np.stack, [enc.pop(k) for k in layers])
  out[encoder] = enc
  return out


def scan_to_pyloop(params_scan, encoder="Transformer"):
  """The inverse: slice l of every stacked leaf becomes layer "encoderblock_l"."""
  out = dict(params_scan)
  enc = dict(out[encoder])
  stacked = enc.pop("encoderblock")
  depth = len(stacked["LayerNorm_0"]["bias"])
  for layer in range(depth):
    enc[f"encoderblock_{layer}"] = _zip_trees(lambda leaves, layer=layer: leaves[0][layer], [stacked])
  out[encoder] = enc
  return out


def load(init_params, init_file, model_cfg, dont_load=()):
  """Parameters for `model_cfg` initialised from checkpoint `init_file` ("path.npz[:sub/tree]"):
  older layouts are modernised, the encoder is (un)stacked to match `model_cfg["scan"]`, names
  matching `dont_load` keep their fresh value from `init_params`, and the position embedding is
  resampled when the checkpoint was trained at another resolution.  Trees are nested dicts under the
  reference names (`utils.recover_tree(*zip(*P.numpy_tree().items()))` / `P.load_tree(dict(flat))`
  convert from and to a FlatParams)."""
  from big_vision_b200 import utils
  from big_vision_b200.models import common
  tree = fix_old_checkpoints(utils.load_params(init_file))
  stored_scanned = "encoderblock" in tree["Transformer"]
  if bool(model_cfg.get("scan")) != stored_scanned:
    tree = scan_to_pyloop(tree) if stored_scanned else pyloop_to_scan(tree)
  tree = common.merge_params(tree, init_params, dont_load)
  if init_params and "pos_embedding" in init_params:
    tree["pos_embedding"] = resample_posemb(old=tree["pos_embedding"], new=init_params["pos_embedding"])
  return tree
