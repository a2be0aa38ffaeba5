"""Jet -- host-side mirror of big_vision/models/proj/jet/jet.py (arXiv 2412.15129), a normalizing flow built
from ViT blocks.

The image [n, H, W, C] is cut into T tokens of 2c = ps*ps*C values (jet.py:236-237), and `depth` affine
couplings map it to z.  Each coupling permutes the n * D values of an image with a fixed 0/1 matrix, over the
values of a token ("channels") or over the tokens ("spatial", followed by `n (s c) -> (n s) c` with s = 2,
jet.py:96-120), splits the result into halves x1 and x2 of [T, c] each, runs the DNN -- Dense c -> emb_dim
plus a position embedding, `block_depth` ViT encoder blocks, encoder_norm, Dense emb_dim -> 2c (jet.py:34-65)
-- on x1 and maps x2 to (x2 + bias) * s with s = sigmoid(raw) * scale_factor (jet.py:126-147).

The masks are parameters (`*_coupling_masks-FREEZE_ME`) that the reference applies with einsum.  Because they
are permutations, every split and merge here is a gather: the index table of each coupling is derived on the
host from the masks, once per parameter set (init / load_tree of the parameters, see _Params), and the
device kernels of include/bv_b200_jet.h gather through it.  The flow state is fp32 throughout; the DNN runs
on the library's bf16 GEMM / attention / LayerNorm path.

As the reference wraps each coupling in nn.remat(nothing_saveable), the forward keeps each coupling's fp32
input only, and the backward recomputes the coupling's DNN from it.
"""
import itertools
import math
from dataclasses import dataclass
from typing import Sequence

import numpy as np
import torch

from big_vision_b200 import engine as E
from big_vision_b200 import lib as L
from big_vision_b200 import ops
from big_vision_b200 import utils as u
from big_vision_b200.models import common
from big_vision_b200.models import vit

CHANNEL_MASKS = "channel_coupling_masks-FREEZE_ME"
SPATIAL_MASKS = "spatial_coupling_masks-FREEZE_ME"
MASKS = frozenset((CHANNEL_MASKS, SPATIAL_MASKS))
DNN = "couplings/dnn/"


def interleave_couplings(depth, kinds, channels_coupling_projs, spatial_coupling_projs):
  """[(kind, channel proj kind, spatial proj kind)] of the `depth` couplings (jet.py:168-186): the kinds cycle
  through `kinds`, and each kind's projections cycle independently; "zero" marks the unused one.  kind is 1 for
  a channel coupling and 0 for a spatial one, as in the reference."""
  ks = itertools.cycle(kinds)
  cc = itertools.cycle(channels_coupling_projs)
  sc = itertools.cycle(spatial_coupling_projs)
  out = []
  for _ in range(depth):
    k = next(ks)
    if k == "channels":
      out.append((1, next(cc), "zero"))
    elif k == "spatial":
      out.append((0, "zero", next(sc)))
    else:
      raise ValueError(f"Unknown coupling kind: {k}")
  return out


def channel_masks_init(depth, dt, proj_kinds):
  """Initialiser of `channel_coupling_masks-FREEZE_ME` [depth, dt, dt] (jet.py:265-283): for a "random"
  coupling i, M[i, p[j], j] = 1 for a random permutation p, drawn from the numpy Generator (the reference's
  JAX draw cannot be reproduced); zeros for a placeholder."""
  def init(rng, shape):
    w = np.zeros(shape, dtype=np.float32)
    for i, kind in enumerate(proj_kinds):
      if kind == "random":
        w[i, rng.permutation(dt), np.arange(dt)] = 1.0
      elif kind != "zero":
        raise ValueError(f"Unknown coupling kind: {kind}")
    return w
  return init


def spatial_masks(depth, nh, nw, proj_kinds):
  """`spatial_coupling_masks-FREEZE_ME` [depth, n, n], n = nh * nw tokens (jet.py:286-318): M[i, idx1[m], m] = 1
  for the first n/2 columns and M[i, idx2[m], n/2 + m] = 1 for the rest, where idx1 / idx2 are the even / odd
  tokens, rows or checkerboard squares, swapped for a "-inv" kind; zeros for a placeholder."""
  n = nh * nw
  w = np.zeros((depth, n, n), dtype=np.float32)
  t = np.arange(n)

  def where(cond):           # jnp.where(cond, size=n // 2)[0]: the first n/2 hits, padded with index 0
    hits = np.nonzero(cond)[0][:n // 2]
    return np.concatenate([hits, np.zeros(n // 2 - len(hits), dtype=hits.dtype)])

  for i, kind in enumerate(proj_kinds):
    if kind == "zero":
      continue
    if kind.startswith("vstripes"):
      idx1, idx2 = t[::2], t[1:][::2]
    elif kind.startswith("hstripes"):
      idx1, idx2 = where((t // nw) % 2 == 0), where((t // nw) % 2 == 1)
    elif kind.startswith("checkerboard"):
      vals = t + t // nw     # arange(n).reshape(nh, nw) + arange(nh)[:, None], flattened
      idx1, idx2 = where(vals % 2 == 0), where(vals % 2 == 1)
    else:
      raise ValueError(f"Unknown coupling kind: {kind}")
    if kind.endswith("-inv"):
      idx1, idx2 = idx2, idx1
    w[i, idx1, np.arange(n // 2)] = 1.0
    w[i, idx2, np.arange(n // 2, n)] = 1.0
  return w


def permutation_of(mask, what):
  """p with mask[p[j], j] = 1 for a 0/1 permutation matrix; raises ValueError for anything else."""
  m = np.asarray(mask)
  ok = (np.all((m == 0) | (m == 1)) and np.all(m.sum(0) == 1) and np.all(m.sum(1) == 1))
  if not ok:
    raise ValueError(f"{what} is not a 0/1 permutation matrix")
  return np.argmax(m, axis=0)


def index_table(kind, channel_mask, spatial_mask, T, dt):
  """The gather table idx[0:D] (D = T * dt) of one coupling: x1 = x[idx[:D/2]] and x2 = x[idx[D/2:]] read as
  [T, dt/2] matrices, for x the flow state [T, dt] flattened.
    channels: x @ M permutes the dt values of each token, then splits them (jet.py:97-100);
    spatial: M^T x permutes the T tokens, splits them in halves of T/2 tokens, and cuts each row of dt values
      into two rows of dt/2 (jet.py:109-114), so row 2r + s of x1 is half s of permuted token r."""
  c = dt // 2
  if kind == 1:
    p = permutation_of(channel_mask, "a channel coupling mask")
    t = np.arange(T)[:, None]
    return np.concatenate([(t * dt + p[None, :c]).reshape(-1), (t * dt + p[None, c:]).reshape(-1)])
  q = permutation_of(spatial_mask, "a spatial coupling mask")
  return (q[:, None] * dt + np.arange(dt)[None, :]).reshape(-1)     # permuted token r, value k at r * dt + k


class _Params(E.FlatParams):
  """FlatParams of a Jet model: also holds the couplings' index tables (int32 [depth, D] on the device),
  derived from the mask parameters whenever the parameters are set through init() or load_tree(), so no
  forward can run on tables of other masks."""
  model = None

  def init(self, seed=0):
    super().init(seed)
    self.model._derive_tables(self)
    return self

  def load_tree(self, tree):
    if any(isinstance(v, dict) for v in tree.values()):
      tree = dict(u.tree_flatten_with_names(tree)[0])
    super().load_tree(tree)
    self.model._derive_tables(self)
    return self


# The two stages below follow engine.Staged's stage protocol (prefixes, specs, fwd, bwd, sink, ready) but are not
# engine.Stage subclasses: that base marks the stages replayed one by one on [rows, d] bf16 activation gradients by
# tests/test_stage_replay_gpu.py, and these pass fp32 flow states and a (dz, dlogdet) pair instead.  They are
# checked as a whole against the float64 oracle (tests/test_jet_gpu.py).
class Dequantize:
  """The bottom stage: it holds the two mask storages and turns the image into the flow state, adding the
  dequantization noise.  It never runs a backward (the masks are always frozen)."""
  ready = None

  def __init__(self, depth, dt, T, grid, c_kinds, s_kinds, ps):
    self.depth, self.dt, self.T, self.grid, self.c_kinds, self.s_kinds, self.ps = depth, dt, T, grid, c_kinds, s_kinds, ps
    self.prefixes = (CHANNEL_MASKS, SPATIAL_MASKS)

  def specs(self):
    s_init = spatial_masks(self.depth, *self.grid, self.s_kinds)
    return [E.ParamSpec(CHANNEL_MASKS, (self.depth, self.dt, self.dt), channel_masks_init(self.depth, self.dt, self.c_kinds)),
            E.ParamSpec(SPATIAL_MASKS, (self.depth, self.T, self.T), lambda rng, shape: s_init)], []

  def fwd(self, P, inp, geom, save=True):
    image, noise = inp
    if noise is None:
      return ops.jet_dequantize_patchify(image, self.ps, noise_scale=0.0), None
    seed, counter, offset = noise
    return ops.jet_dequantize_patchify(image, self.ps, seed, counter, offset), None

  def sink(self, P, geom):
    return None

  def bwd(self, P, dy, saved, geom, sink=None, need_dx=False):
    return None


class Couplings:
  """Every coupling of the flow, as the reference's nn.scan over one remat'd `couplings` module whose
  parameters carry a leading depth axis: one backward stage that holds all `couplings/` storage."""
  ready = None

  def __init__(self, depth, block_depth, d, heads, T, c, scale_factor):
    self.depth, self.d, self.heads, self.T, self.c, self.scale_factor = depth, d, heads, T, c, scale_factor
    self.prefixes = ("couplings/",)
    self.blocks = [[vit.EncoderBlock(f"{DNN}vit/encoderblock_{j}/", d, 4 * d, heads, index=i)
                    for j in range(block_depth)] for i in range(depth)]

  def sink(self, P, geom):
    return None

  def specs(self):
    D, d, c, T, st = self.depth, self.d, self.c, self.T, self.depth
    specs = [E.ParamSpec(DNN + "init_proj/kernel", (D, c, d), vit._stacked(E.lecun_normal(c), st)),
             E.ParamSpec(DNN + "init_proj/bias", (D, d), vit._stacked(E.zeros, st)),
             E.ParamSpec(DNN + "posemb", (D, 1, T, d), vit._stacked(E.normal(1 / math.sqrt(d)), st))]
    aliases = []
    for blk in self.blocks[0]:
      s, a = blk.specs(stack=D)
      specs += s
      aliases += a
    specs += vit.ln_specs(DNN + "vit/encoder_norm/", d, stack=D)
    specs += [E.ParamSpec(DNN + "final_proj/kernel", (D, d, 2 * c), vit._stacked(E.zeros, st)),
              E.ParamSpec(DNN + "final_proj/bias", (D, 2 * c), vit._stacked(E.zeros, st))]
    return specs, aliases

  # ---- the DNN of coupling i (jet.py:34-65) --------------------------------------------------------------
  def dnn_fwd(self, P, i, x1, n, save=True):
    """x1 bf16 [n * T, c] -> (br fp32 [n * T, 2c], saved or None)."""
    S = vit.Scope(P, DNN, i)
    geom = E.Geom(n, self.T)
    h = ops.gemm(x1, S.h("init_proj/kernel"), b_mn=True, bias=S.f("init_proj/bias"),
                 aux=S.h("posemb").view(self.T, self.d), aux_row_mod=self.T, epilogue=L.EPI_BIAS_RESID)
    blocks = []
    for blk in self.blocks[i]:
      h, s = blk.fwd(P, h, geom, save)
      blocks.append(s)
    enc, mean, rstd = ops.layernorm_fwd(h, S.f("vit/encoder_norm/scale"), S.f("vit/encoder_norm/bias"))
    br = ops.gemm(enc, S.h("final_proj/kernel"), b_mn=True, bias=S.f("final_proj/bias"), out_dtype=torch.float32)
    return br, ((x1, blocks, h, mean, rstd, enc) if save else None)

  def dnn_bwd(self, P, i, dbr, saved, n):
    """dbr bf16 [n * T, 2c] -> dx1 fp32 [n * T, c]; accumulates coupling i's parameter gradients."""
    S = vit.Scope(P, DNN, i)
    geom = E.Geom(n, self.T)
    x1, blocks, h, mean, rstd, enc = saved
    ops.colsum(dbr, S.g("final_proj/bias"))
    ops.gemm(enc, dbr, a_mn=True, b_mn=True, out=S.g("final_proj/kernel"), reduce_out=True)
    denc = ops.gemm(dbr, S.h("final_proj/kernel"))
    del enc
    top = self.blocks[i][-1].sink(P, geom) if self.blocks[i] else S.g("init_proj/bias")
    dh = ops.layernorm_bwd(denc, h, S.f("vit/encoder_norm/scale"), mean, rstd, dscale=S.g("vit/encoder_norm/scale"),
                           dbias=S.g("vit/encoder_norm/bias"), dx_colsum=top)
    del denc
    for j in reversed(range(len(self.blocks[i]))):
      sink = self.blocks[i][j - 1].sink(P, geom) if j else S.g("init_proj/bias")
      dh = self.blocks[i][j].bwd(P, dh, blocks[j], geom, sink)
      blocks[j] = None
    # the position embedding is shared by the batch: its gradient is the batch sum (init_proj's bias gradient,
    # the sum over rows too, came with dh as the column sum of the stage above)
    ops.colsum(dh.view(n, self.T * self.d), S.g("posemb").view(self.T * self.d))
    ops.gemm(x1, dh, a_mn=True, b_mn=True, out=S.g("init_proj/kernel"), reduce_out=True)
    return ops.gemm(dh, S.h("init_proj/kernel"), out_dtype=torch.float32)

  # ---- the stage ----------------------------------------------------------------------------------------
  def fwd(self, P, z, geom, save=True):
    """z fp32 [n, T, 2c] -> ((z', logdet fp32 [n]), saved).  Without save every coupling runs in place."""
    n, T, c = geom.n, self.T, self.c
    idx = P.jet_tables
    logdet = torch.zeros(n, dtype=torch.float32, device=z.device)
    inputs = [] if save else None
    for i in range(self.depth):
      x1 = ops.jet_split(z, idx[i], T, c)
      br, _ = self.dnn_fwd(P, i, x1, n, save=False)
      del x1
      if save:
        inputs.append(z)                       # remat: keep the coupling input only
        z = ops.jet_coupling_fwd(z, idx[i], br, logdet, T, c, self.scale_factor)
      else:
        ops.jet_coupling_fwd(z, idx[i], br, logdet, T, c, self.scale_factor, out=z)
    return (z, logdet), inputs

  def inverse(self, P, x, n, logdet):
    """The couplings in reverse order, each inverted, in place on x fp32 [n, T, 2c]; subtracts the logdets."""
    idx = P.jet_tables
    for i in reversed(range(self.depth)):
      br, _ = self.dnn_fwd(P, i, ops.jet_split(x, idx[i], self.T, self.c), n, save=False)
      ops.jet_coupling_fwd(x, idx[i], br, logdet, self.T, self.c, self.scale_factor, inverse=True, out=x)
    return x

  def bwd(self, P, dy, saved, geom, sink=None, need_dx=True):
    """dy = (dz fp32 [n, T, 2c], dlogdet: the constant gradient of the loss with respect to each image's
    logdet).  Returns the gradient of the flow input (dz's buffer, overwritten)."""
    dz, dlogdet = dy
    n, T, c, idx = geom.n, self.T, self.c, P.jet_tables
    for i in reversed(range(self.depth)):
      x = saved[i]
      x1 = ops.jet_split(x, idx[i], T, c)
      br, s = self.dnn_fwd(P, i, x1, n)         # recompute the DNN from the saved input
      _, dbr = ops.jet_coupling_bwd(dz, x, idx[i], br, dlogdet, T, c, self.scale_factor, dx=dz)
      del br
      dx1 = self.dnn_bwd(P, i, dbr, s, n)
      del dbr, s
      ops.jet_merge_grad(dz, dx1, idx[i], T, c, dx=dz)
      saved[i] = None
    return dz


@dataclass
class _Model(E.Staged):
  """Jet; fields and defaults as in jet.py:150-161."""
  depth: int = 2
  block_depth: int = 1
  emb_dim: int = 256
  num_heads: int = 4
  scale_factor: float = 2.0
  ps: int = 4
  channels_coupling_projs: Sequence[str] = ("random",)
  spatial_coupling_projs: Sequence[str] = ("checkerboard", "checkerboard-inv")
  kinds: Sequence[str] = ("channels", "channels", "spatial")

  def __post_init__(self):
    vit.check_head_dim(self.emb_dim, self.num_heads)
    self.couplings = interleave_couplings(self.depth, self.kinds, self.channels_coupling_projs,
                                          self.spatial_coupling_projs)

  # ---- parameters ------------------------------------------------------------------------
  def specs(self, image_hw, in_ch=3):
    """Builds the two stages for [n, *image_hw, in_ch] images -> (specs, aliases)."""
    H, W = image_hw
    if H % self.ps or W % self.ps:
      raise ValueError(f"image {H}x{W} is not a multiple of the patch size {self.ps}")
    self.image_hw, self.in_ch = (H, W), in_ch
    self.grid = (H // self.ps, W // self.ps)
    self.T, self.dt = self.grid[0] * self.grid[1], self.ps * self.ps * in_ch
    self.c = self.dt // 2
    if self.dt % 2 or self.c % 8:
      raise NotImplementedError(
          f"ps={self.ps}, {in_ch} channels: half a token, c = ps*ps*C/2 = {self.dt / 2}, must be a multiple of 8 "
          "(the rows of the DNN's first GEMM operand need 16-byte strides for TMA)")
    if any(k == 0 for k, _, _ in self.couplings) and self.T % 2:
      raise ValueError(f"spatial couplings need an even token count, got {self.T}")
    kinds, c_kinds, s_kinds = zip(*self.couplings)
    return self._build([Dequantize(self.depth, self.dt, self.T, self.grid, c_kinds, s_kinds, self.ps),
                        Couplings(self.depth, self.block_depth, self.emb_dim, self.num_heads, self.T, self.c,
                                  self.scale_factor)])

  def init(self, seed, image_shape, device="cuda"):
    """Counterpart of model.init(rng, image, method=model.forward)["params"] (trainers/proj/jet/train.py:196-201).
    The index tables are derived from the masks here, and again on every P.load_tree()."""
    specs, aliases = self.specs(image_shape[1:3], image_shape[3])
    P = _Params(specs, aliases, device)
    P.model = self
    return P.init(seed)

  def _derive_tables(self, P):
    """P.jet_tables int32 [depth, D] on P's device, from P's masks; raises ValueError if the mask of a
    coupling's kind is not a 0/1 permutation matrix."""
    cm = P.f(CHANNEL_MASKS).detach().cpu().numpy()
    sm = P.f(SPATIAL_MASKS).detach().cpu().numpy()
    tables = [index_table(k, cm[i], sm[i], self.T, self.dt) for i, (k, _, _) in enumerate(self.couplings)]
    P.jet_tables = torch.from_numpy(np.stack(tables).astype(np.int32)).to(P.device)

  # ---- forward / backward ----------------------------------------------------------------
  def fwd(self, P, image, frozen=None, noise=None):
    """image fp32 [n, H, W, C] in [-1, 1] -> ((z fp32 [n, T, 2c] in the flow layout, logdet fp32 [n]), saved).
    noise: None, or (seed, counter, offset) to add the dequantization noise of bv_jet_dequantize_patchify
    (offset: this batch's first element in the global batch).  `frozen` as in vit.Model.fwd; the masks are
    always frozen."""
    frozen = True if frozen is True else MASKS | frozenset(frozen or ())
    return self._stages_fwd(P, (image, noise), E.Geom(image.shape[0], self.T), frozen)

  def bwd(self, P, dz, dlogdet, saved):
    """dz fp32 [n, T, 2c] (consumed), dlogdet the constant d loss / d logdet[b].  Accumulates into P.grad."""
    self._stages_bwd(P, (dz, dlogdet), saved)

  # ---- reference-style entry points (forward-only, in place in the flow layout) --------------
  def forward(self, P, image):
    """(z [n, H, W, C], logdet [n]) of jet.py:232-246, without noise."""
    (z, logdet), _ = self.fwd(P, image, frozen=True)
    return ops.jet_unpatchify(z, image.shape, self.ps), logdet

  def inverse(self, P, z):
    """(image [n, H, W, C], logdet [n]) of jet.py:248-262: every coupling inverted, in reverse order;
    logdet is minus the forward's."""
    x = ops.jet_dequantize_patchify(z, self.ps, noise_scale=0.0)
    logdet = torch.zeros(z.shape[0], dtype=torch.float32, device=z.device)
    self._stages[1].inverse(P, x, z.shape[0], logdet)
    return ops.jet_unpatchify(x, z.shape, self.ps), logdet


def Model(**kw):  # pylint: disable=invalid-name
  """Factory, same fields as big_vision.models.proj.jet.jet.Model."""
  return _Model(**kw)


def load(init_params, init_file, model_cfg=None, dont_load=()):
  """Parameters from checkpoint `init_file` ("path.npz[:sub/tree]") merged into `init_params` (jet.py:321-332):
  names matching `dont_load` keep their value from init_params.  P.load_tree(tree) then sets them, masks and
  index tables together."""
  del model_cfg
  tree = u.load_params(init_file)
  return common.merge_params(tree, init_params, dont_load)
