"""FlexiViT on the H100 kernels -- host-side mirror of big_vision/models/proj/flexi/vit.py.

One set of parameters serves every sequence length.  The patch-embedding kernel [p0, p0, C, d] and the
position embedding [1, gh * gw, d] are stored at their base shapes; a call at `seqhw` uses patches of
p = H // seqhw pixels and a seqhw x seqhw token grid:
  - the kernel is resampled by the pseudo-inverse of the bilinear patch resize (tf.image.resize,
    half-pixel centres, no antialias): W'[:, :, c, j] = pinv(R^T) vec(W[:, :, c, j]);
  - the position embedding is resized like jax.image.resize(..., "linear"), which antialiases when it
    downsamples.
Both are linear maps fixed by the two shapes: their float64 matrices are built on the host, cached in fp32
per device, and applied to the CURRENT fp32 weights on every forward by bv_resample_fwd (bf16 GEMM operand
out), with bv_resample_bwd taking the gradient back to the stored shapes.  At p == p0 and a base-sized grid
nothing is resampled and the step is the plain ViT's.  The rest -- posemb added in the patch GEMM's
epilogue, [cls] prepended for "tok", the encoder, the pool, the head -- is vit.py's stages unchanged.

Unlike the reference, which runs this model in fp32, every matmul takes bf16 operands with fp32
accumulation (DESIGN.md, numerics), as the other towers here do.
"""
import copy
import math
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np
import torch

from big_vision_b200 import engine as E
from big_vision_b200 import ops
from big_vision_b200.models import common
from big_vision_b200.models import vit

_POOLS = {"gap": "mean", "tok": "first", "map": None}   # -> vit.NormPool's pool


# ------------------------------------------------------------------------------------------
# resize matrices (host, float64)
# ------------------------------------------------------------------------------------------
def resize_weights(n_in, n_out, antialias):
  """[n_out, n_in] weights of a 1-D linear resize with half-pixel centres (jax's compute_weight_mat for
  the "linear" kernel).  With `antialias` a downsampling resize widens the triangle kernel by
  n_in / n_out; tf.image.resize(..., "bilinear") is the form without."""
  inv = n_in / n_out
  ks = max(inv, 1.0) if antialias else 1.0
  s = (np.arange(n_out) + 0.5) * inv - 0.5
  w = np.maximum(0.0, 1.0 - np.abs(s[:, None] - np.arange(n_in)[None, :]) / ks)
  tot = w.sum(1, keepdims=True)
  w = np.where(np.abs(tot) > 1000 * np.finfo(np.float32).eps, w / np.where(tot != 0, tot, 1), 0.0)
  return np.where(((s >= -0.5) & (s <= n_in - 0.5))[:, None], w, 0.0)


def pi_resize_matrix(p0, p):
  """[p*p, p0*p0]: pinv(R^T) for R the bilinear resize of p0 x p0 patches to p x p (row-major pixels).
  For p >= p0, R^T pinv(R^T) = I: a resized patch under the resampled kernel gives the original
  embedding."""
  w = resize_weights(p0, p, antialias=False)
  return np.linalg.pinv(np.kron(w, w).T)


def posemb_resize_matrix(posemb_size, seqhw):
  """[seqhw^2, gh * gw]: the antialiased linear resize of a gh x gw position-embedding grid to
  seqhw x seqhw (row-major tokens)."""
  gh, gw = posemb_size
  return np.kron(resize_weights(gh, seqhw, True), resize_weights(gw, seqhw, True))


def resample_patchemb(old, new_hw):
  """The kernel [p0, p0, C, d] resampled to patch size new_hw (reference flexi/vit.py:30-71); returned
  unchanged when the shapes agree."""
  old = np.asarray(old)
  if tuple(old.shape[:2]) == tuple(new_hw):
    return old
  (p0, q0), (p, q) = old.shape[:2], new_hw
  if p0 != q0 or p != q:
    raise NotImplementedError(f"resample_patchemb {old.shape[:2]} -> {tuple(new_hw)}: square patches only")
  M = pi_resize_matrix(p0, p)
  return (M @ old.reshape(p0 * p0, -1).astype(np.float64)).reshape(p, p, *old.shape[2:]).astype(old.dtype)


_MATRICES = {}


def _device_matrix(kind, a, b, device):
  """The fp32 device copy of a resize matrix, built once per (kind, shapes, device)."""
  key = (kind, a, b, str(device))
  m = _MATRICES.get(key)
  if m is None:
    host = pi_resize_matrix(a, b) if kind == "patch" else posemb_resize_matrix(a, b)
    m = _MATRICES[key] = torch.from_numpy(host.astype(np.float32)).to(device)
  return m


# ------------------------------------------------------------------------------------------
# the flexible patch embedding
# ------------------------------------------------------------------------------------------
class FlexiPatchEmbedding(vit.PatchEmbedding):
  """vit.PatchEmbedding at any sequence length.  Each call runs vit.PatchEmbedding's own forward and
  backward (the GEMM, the posemb epilogue, [cls], the bias / cls / posemb sums) on a copy of the stage at
  this call's patch size and on a _CallParams: the bf16 kernel and position embedding it reads are resampled
  from the base shapes unless they already fit, and the kernel / posemb gradients it writes go to scratch
  buffers that bv_resample_bwd takes back to the stored shapes."""

  def __init__(self, prefix, patch_size, posemb_size, in_ch, d, posemb, cls):
    p0 = patch_size[0]
    super().__init__(prefix, "embedding", (p0 * posemb_size[0], p0 * posemb_size[1]), patch_size, in_ch, d,
                     posemb, cls)
    self.posemb_size = tuple(posemb_size)
    self._sincos32 = None

  def specs(self):
    """As vit's, with the flexi init: kernel normal(1/sqrt(width)) (flexi/vit.py:87-89)."""
    specs, aliases = super().specs()
    (ph, pw), d, in_ch = self.patch_size, self.d, self.in_ch
    K = ph * pw * in_ch
    Kp = (K + 7) // 8 * 8
    nrm = E.normal(1 / math.sqrt(d))
    specs[0] = E.ParamSpec(self.w + "kernel_flat", (Kp, d),
                           lambda rng, shape: np.concatenate([nrm(rng, (K, d)), np.zeros((Kp - K, d))], 0))
    return specs, aliases

  def geometry(self, image, geom):
    """(p, seqhw) of this forward: seqhw from the token count, p = H // seqhw."""
    seqhw = math.isqrt(geom.N - self.cls)
    return image.shape[1] // seqhw, seqhw

  def _pos32(self, P):
    """fp32 [gh * gw, d]: the learned table, or the fixed sincos table at posemb_size."""
    if self.posemb == "learn":
      return P.f(self.p + "pos_embedding").view(-1, self.d)
    if self._sincos32 is None or self._sincos32.device != P.device:
      self._sincos32 = torch.from_numpy(vit.posemb_sincos_2d(*self.posemb_size, self.d)).to(P.device)
    return self._sincos32

  def _posemb16(self, P):
    # reached from vit.PatchEmbedding.fwd only through a _CallParams, which carries this call's table
    return P.posemb16

  def _view(self, p):
    """A copy of this stage at patch size p, to run vit.PatchEmbedding's forward / backward on."""
    view = copy.copy(self)
    view.patch_size = (p, p)
    return view

  def fwd(self, P, image, geom, save=True):
    p, seqhw = self.geometry(image, geom)
    p0, d, C, w = self.patch_size[0], self.d, self.in_ch, self.w
    h16 = {}
    if p != p0:
      K = p * p * C
      kernel16 = torch.empty(((K + 7) // 8 * 8, d), dtype=torch.bfloat16, device=image.device)
      kernel16[K:].zero_()
      ops.resample_fwd(_device_matrix("patch", p0, p, P.device),
                       P.f(w + "kernel_flat")[:p0 * p0 * C].view(p0 * p0, C * d), out=kernel16)
      h16[w + "kernel_flat"] = kernel16
    posemb16 = None
    if self.posemb:
      if (seqhw, seqhw) == self.posemb_size:
        posemb16 = vit.PatchEmbedding._posemb16(self, P)
      else:
        posemb16 = ops.resample_fwd(_device_matrix("posemb", self.posemb_size, seqhw, P.device), self._pos32(P))
    x, patches = vit.PatchEmbedding.fwd(self._view(p), _CallParams(P, h16, {}, posemb16), image, geom, save)
    return x, ((patches, p) if save else None)

  def bwd(self, P, dx, saved, geom, sink=None, need_dx=False):
    patches, p = saved
    seqhw = math.isqrt(geom.N - self.cls)
    p0, d, C, w, pos = self.patch_size[0], self.d, self.in_ch, self.w, self.p + "pos_embedding"
    g = {}
    if p != p0:
      g[w + "kernel_flat"] = torch.zeros((patches.shape[1], d), dtype=torch.float32, device=dx.device)
    if self.posemb == "learn" and (seqhw, seqhw) != self.posemb_size:
      g[pos] = torch.zeros((1, seqhw * seqhw, d), dtype=torch.float32, device=dx.device)
    vit.PatchEmbedding.bwd(self._view(p), _CallParams(P, {}, g, None), dx, patches, geom)
    if p != p0:
      ops.resample_bwd(_device_matrix("patch", p0, p, P.device), g[w + "kernel_flat"][:p * p * C].view(p * p, C * d),
                       P.g(w + "kernel_flat")[:p0 * p0 * C].view(p0 * p0, C * d))
    if pos in g:
      ops.resample_bwd(_device_matrix("posemb", self.posemb_size, seqhw, P.device), g[pos].view(seqhw * seqhw, d),
                       P.g(pos).view(-1, d))


class _CallParams:
  """The parameters as one call of vit.PatchEmbedding's forward / backward sees them: `h(name)` of a name
  in `h16` is this call's bf16 operand (the resampled kernel), `g(name)` of a name in `grads` this call's
  scratch gradient (at the resampled shape), `posemb16` this call's position embedding; every other name
  is P's."""

  def __init__(self, P, h16, grads, posemb16):
    self.P, self.h16, self.grads, self.posemb16 = P, h16, grads, posemb16

  def f(self, name):
    return self.P.f(name)

  def h(self, name):
    return self.h16[name] if name in self.h16 else self.P.h(name)

  def g(self, name):
    return self.grads[name] if name in self.grads else self.P.g(name)


# ------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------
@dataclass
class _Model(E.Staged):
  """FlexiViT; fields as in flexi/vit.py:107-122.  `scan` / `remat_policy` are an extension (as in
  vit.Model): the encoder as one scanned, recomputed block, which long sequences need to fit in HBM."""
  num_classes: Optional[int] = None
  patch_size: Sequence[int] = (32, 32)
  posemb_size: Sequence[int] = (7, 7)
  width: int = 768
  depth: int = 12
  mlp_dim: Optional[int] = None
  num_heads: int = 12
  posemb: str = "learn"
  pool_type: str = "gap"
  head_zeroinit: bool = True
  seqhw: Optional[int] = None
  scan: bool = False
  remat_policy: str = "nothing_saveable"

  def __post_init__(self):
    if self.pool_type not in _POOLS:
      raise ValueError(f"Unknown pool type: '{self.pool_type}'")
    if self.posemb not in ("learn", "sincos2d"):
      raise ValueError(f"Unknown posemb type: {self.posemb}")
    if self.patch_size[0] != self.patch_size[1]:
      raise NotImplementedError(f"patch_size {tuple(self.patch_size)}: FlexiViT is built for square patches")
    vit.check_head_dim(self.width, self.num_heads)
    self.mlp = self.mlp_dim or 4 * self.width

  # ---- parameters ------------------------------------------------------------------------
  def specs(self, image_hw=None, in_ch=3):
    """Builds the backward stages -> (specs, aliases).  The parameters do not depend on the image size:
    `image_hw` is accepted for the signature of the other models and not used."""
    d, enc = self.width, "Transformer/"
    head_init = E.zeros if self.head_zeroinit else E.lecun_normal(d)
    self.head = common.Dense("head/", d, self.num_classes, head_init, pad=True) if self.num_classes else None
    embed = FlexiPatchEmbedding("", self.patch_size, self.posemb_size, in_ch, d, self.posemb, self.pool_type == "tok")
    stages = ([embed] + vit.encoder_stages(enc, self.depth, d, self.mlp, self.num_heads, self.scan, self.remat_policy)
              + [vit.NormPool(enc + "encoder_norm/", d, _POOLS[self.pool_type], torch.float32)])
    if self.pool_type == "map":
      stages.append(vit.MAPHead("MAPHead_0/", d, self.mlp, self.num_heads))
    if self.head is not None:
      stages.append(self.head)
    return self._build(stages)

  def init(self, seed, image_shape, device="cuda"):
    """Counterpart of model.init(rng, zeros_image)["params"]; only the channel count of image_shape
    matters."""
    specs, aliases = self.specs(image_shape[1:3], image_shape[3])
    return E.FlatParams(specs, aliases, device).init(seed)

  # ---- forward / backward ----------------------------------------------------------------
  def geom(self, image, seqhw=None):
    """E.Geom of a forward on `image` [n, H, W, C] at `seqhw` (else the field)."""
    seqhw = seqhw or self.seqhw
    if seqhw is None:
      raise ValueError("FlexiViT needs seqhw: pass it to the call or set the model's seqhw field")
    n, H, W = image.shape[:3]
    if H != W:
      raise NotImplementedError(f"FlexiViT on non-square images ({H}x{W})")
    if H % seqhw:
      raise NotImplementedError(f"FlexiViT at seqhw={seqhw}: the image side {H} is not a multiple of it")
    return E.Geom(n, seqhw * seqhw + (self.pool_type == "tok"))

  def fwd(self, P, image, seqhw=None, frozen=None):
    """image [n,H,W,C] fp32 -> (logits fp32 [n, num_classes] (the pooled representation without a head),
    saved).  `frozen` as in vit.Model.fwd."""
    return self._stages_fwd(P, image, self.geom(image, seqhw), frozen)

  def bwd(self, P, dout, saved):
    """dout fp32 [n, out] (the padded class count with a head).  Accumulates into P.grad."""
    self._stages_bwd(P, dout, saved)

  # ---- reference-style entry points --------------------------------------------------------
  def apply(self, variables, image, *, seqhw=None, train=False):
    """(x, out) like flax apply (flexi/vit.py:124-197); `out` holds what this path keeps."""
    x, _ = self.fwd(variables["params"], image, seqhw, frozen=True)
    return x, {"logits" if self.num_classes else "pre_logits": x}


def Model(num_classes=None, *, variant=None, **kw):  # pylint: disable=invalid-name
  """Factory, same signature as big_vision.models.proj.flexi.vit.Model."""
  return _Model(num_classes, **{**vit.decode_variant(variant), **kw})


def load(init_params, init_file, model_cfg, dont_load=()):
  """Parameters for `model_cfg` from checkpoint `init_file` (flexi/vit.py:200-221): older layouts are
  modernised, the encoder is (un)stacked to match `model_cfg["scan"]`, the position embedding is resized
  to the model's (vit.resample_posemb) and the patch-embedding kernel resampled to its patch size
  (resample_patchemb), then names matching `dont_load` keep their value from `init_params`."""
  from big_vision_b200 import utils
  tree = vit.fix_old_checkpoints(utils.load_params(init_file))
  stored_scanned = "encoderblock" in tree["Transformer"]
  if bool(model_cfg.get("scan")) != stored_scanned:
    tree = vit.scan_to_pyloop(tree) if stored_scanned else vit.pyloop_to_scan(tree)
  if init_params and "pos_embedding" in init_params and "pos_embedding" in tree:
    tree["pos_embedding"] = vit.resample_posemb(old=tree["pos_embedding"], new=init_params["pos_embedding"])
  cfg = {**vit.decode_variant(model_cfg.get("variant")), **dict(model_cfg)}
  tree["embedding"] = dict(tree["embedding"])
  tree["embedding"]["kernel"] = resample_patchemb(tree["embedding"]["kernel"], cfg.get("patch_size", (32, 32)))
  return common.merge_params(tree, init_params, dont_load)
