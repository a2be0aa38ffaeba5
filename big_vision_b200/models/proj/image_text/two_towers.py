"""Two-tower image/text model -- mirror of big_vision/models/proj/image_text/two_towers.py:28-90.

Builds the `img` and `txt` sub-models by import string exactly like the reference
(two_towers.py:51-53,64-66, but under the big_vision_b200.models namespace), L2-normalises
both embeddings (:60-61,:73-74) and owns the temperature `t` (stored as log t, :76-80) and
bias `b` (:83-85) parameters.  Returns (zimg, ztxt, out) with out["t"] = exp(t), out["b"].
"""
import importlib
import math
from dataclasses import dataclass
from typing import Any, Optional, Tuple, Union

import numpy as np
import torch

from big_vision_b200 import engine as E
from big_vision_b200 import ops

ConfigDict = Any


@dataclass
class Model:
  """Two towers transformer (fields as two_towers.py:30-36)."""
  image: Optional[ConfigDict] = None
  text: Optional[ConfigDict] = None
  text_model: str = "proj.image_text.text_transformer"
  image_model: str = "vit"
  out_dim: Union[int, Tuple[int, int]] = 128
  temperature_init: float = 1.0
  bias_init: Optional[float] = None

  def __post_init__(self):
    out_dims = self.out_dim
    if isinstance(out_dims, int):
      out_dims = (out_dims, out_dims)
    self.txt = importlib.import_module(f"big_vision_b200.models.{self.text_model}").Model(
        **{"num_classes": out_dims[1], **(dict(self.text or {}))}, name="txt")
    self.img = importlib.import_module(f"big_vision_b200.models.{self.image_model}").Model(
        **{"num_classes": out_dims[0], **(dict(self.image or {}))}, name="img")

  def specs(self, image_shape, text_shape):
    s_img, a_img = self.img.specs(image_shape[1:3], image_shape[3])
    s_txt, a_txt = self.txt.specs(text_shape[1])
    specs = s_img + s_txt + [E.ParamSpec("t", (1,), E.constant(math.log(self.temperature_init)))]
    if self.bias_init is not None:
      specs.append(E.ParamSpec("b", (1,), E.constant(self.bias_init)))
    return specs, a_img + a_txt

  def init(self, seed, image_shape, text_shape, device="cuda"):
    """Counterpart of model.init(rng, zeros_image, zeros_text)["params"] (siglip.py:193-203)."""
    specs, aliases = self.specs(image_shape, text_shape)
    return E.FlatParams(specs, aliases, device).init(seed)

  def tower_frozen(self, P, frozen):
    """(image tower wholly frozen, text tower wholly frozen) under `frozen` (optax.Chain.frozen()):
    such a tower runs forward-only, and neither the loss nor the backward computes its gradient."""
    return (self.img.cut(P, frozen) == len(self.img.stages()),
            self.txt.cut(P, frozen) == len(self.txt.stages()))

  def fwd(self, P, image, text, frozen=None, dropout=None):
    """-> (zimg fp32 [n,D], ztxt fp32 [n,D], saved).  `frozen` as in vit._Model.fwd; a wholly frozen
    tower keeps nothing for the backward (its saved entries are None).  `dropout`: the engine.DropoutKey of
    a training forward, or None; the image tower draws its masks as tower 0 and the text tower as tower 1,
    so no two sites share a stream."""
    saved = {}
    ztxt = zimg = None
    # only a tower with dropout takes a key
    kw = lambda m, tower: {"dropout": dropout._replace(tower=tower)} if dropout is not None and _drops(m) else {}
    if text is not None:
      e, s = self.txt.fwd(P, text, frozen=frozen, **kw(self.txt, 1))
      ztxt, nrm = ops.l2norm_fwd(e, eps=1e-8)
      live = self.txt.cut(P, frozen) < len(self.txt.stages())
      saved["txt"], saved["txt_norm"] = (s, (ztxt, nrm)) if live else (None, None)
    if image is not None:
      e, s = self.img.fwd(P, image, frozen=frozen, **kw(self.img, 0))
      zimg, nrm = ops.l2norm_fwd(e, eps=1e-8)
      live = self.img.cut(P, frozen) < len(self.img.stages())
      saved["img"], saved["img_norm"] = (s, (zimg, nrm)) if live else (None, None)
    return zimg, ztxt, saved

  def bwd(self, P, dzimg, dztxt, saved):
    """dzimg/dztxt: fp32 [n,D] gradients w.r.t. the normalised embeddings.  A tower is skipped, its
    L2-norm backward included, when its gradient is None or it was wholly frozen in the forward."""
    if dztxt is not None and saved.get("txt_norm") is not None:
      z, nrm = saved["txt_norm"]
      self.txt.bwd(P, ops.l2norm_bwd(dztxt, z, nrm, eps=1e-8), saved["txt"])
      saved["txt"] = None
    if dzimg is not None and saved.get("img_norm") is not None:
      z, nrm = saved["img_norm"]
      self.img.bwd(P, ops.l2norm_bwd(dzimg, z, nrm, eps=1e-8), saved["img"])
      saved["img"] = None

  def apply(self, variables, image, text=None, **kw):
    """(zimg, ztxt, out) like the flax apply (two_towers.py:39-90); forward-only (same bits as the
    training forward, nothing kept for a backward)."""
    if kw.get("train") and (_drops(self.img) or _drops(self.txt)):
      raise ValueError("apply(train=True) with dropout > 0 has no dropout key; call fwd(..., dropout=key)")
    P = variables["params"]
    zimg, ztxt, _ = self.fwd(P, image, text, frozen=True)
    out = {"t": P.f("t").exp(), "t/parameter": P.f("t")}
    if self.bias_init is not None:
      out["b"] = P.f("b")
    return zimg, ztxt, out


def _drops(tower):
  """Whether a tower trains with dropout: the ViT and text towers' `dropout`, BERT's two rates."""
  return any(getattr(tower, k, 0.0) for k in ("dropout", "dropout_rate", "attention_dropout_rate"))


# which entry of `init_files` feeds which part of the model: (part, accepted keys)
_LOAD_SOURCES = (("img", ("image", "img")), ("txt", ("text", "txt")), ("t", ("temperature", "t")),
                 ("b", ("bias", "b")))
_DEFAULT_TOWER = {"img": ("image_model", "vit", "image"),
                  "txt": ("text_model", "proj.image_text.text_transformer", "text")}


def load(init_params, init_files, model_cfg, img_load_kw=None, txt_load_kw=None):
  """Two-tower parameters from checkpoints (contract of two_towers.py:92-135).

  `init_files`: the path of ONE two-tower .npz -- its `img`, `txt`, `t` (and, for models with a
  bias, `b`) sub-trees are used -- or a dict naming a source per part ("image"/"img",
  "text"/"txt", "temperature"/"t", "bias"/"b", each "file.npz[:sub/tree]"); parts without a source
  keep their value from `init_params`.  Each tower is loaded by its own module's `load` with the
  tower's config and `img_load_kw` / `txt_load_kw` (e.g. dont_load).  Unknown keys are an error."""
  from big_vision_b200 import utils
  if isinstance(init_files, str):
    parts = [part for part, _ in _LOAD_SOURCES if part != "b" or "bias_init" in model_cfg.keys()]
    sources = {part: f"{init_files}:{part}" for part in parts}
  else:
    sources = dict(init_files)
  init_params = init_params or {"img": None, "txt": None}
  result = dict(init_params)
  tower_kw = {"img": img_load_kw or {}, "txt": txt_load_kw or {}}
  for part, keys in _LOAD_SOURCES:
    found = [sources.pop(k) for k in keys if k in sources]
    src = next((f for f in found if f), None)
    if not src:
      continue
    if part in _DEFAULT_TOWER:
      cfg_key, default_mod, tower_cfg = _DEFAULT_TOWER[part]
      mod = importlib.import_module(f"big_vision_b200.models.{model_cfg.get(cfg_key, default_mod)}")
      result[part] = mod.load(init_params[part], src, model_cfg.get(tower_cfg, {}), **tower_kw[part])
    else:
      result[part] = utils.load_params(src)
  if sources:
    raise AssertionError(f"Unused entries in `config.model_init` (typo?): {sources}")
  return result
