"""Text tower on the H100 kernels -- mirror of
big_vision/models/proj/image_text/text_transformer.py:29-99.

Embed(vocab, width) + learned posemb -> vit.Encoder (no attention mask: none is passed at
text_transformer.py:72-75) -> pool ("last" by default; "first", "mean"/"gap", "max"/"gmp", "map",
:82-93) -> Dense head (:97-98).
`out["vocab_logits"]` (:80) is dead in training and is never computed here.

The reference runs this tower in fp32 (it has no dtype_mm field); BASELINE.json's configs
ask for bf16 matmuls in both towers, which is what this does (fp32 accumulate).
"""
import math
from dataclasses import dataclass
from typing import Optional

import torch

from big_vision_b200 import engine as E
from big_vision_b200 import ops
from big_vision_b200.models import vit


@dataclass
class _Model:
  """Fields as text_transformer._Model (text_transformer.py:43-52)."""
  num_classes: Optional[int] = None
  width: int = 512
  depth: int = 12
  mlp_dim: int = 2048
  num_heads: int = 8
  dropout: float = 0.0
  vocab_size: int = 32_000
  pool_type: str = "last"
  scan: bool = False
  remat_policy: str = "nothing_saveable"
  name: str = ""

  def __post_init__(self):
    if self.dropout:
      raise NotImplementedError("dropout > 0 is not on the benchmarked path")
    if self.pool_type not in ("last", "first", "mean", "gap", "max", "gmp", "map"):
      raise NotImplementedError(f"Cannot do pooling '{self.pool_type}'")
    vit.check_head_dim(self.width, self.num_heads)
    self.prefix = (self.name + "/") if self.name else ""
    self.map_head = (vit.MAPHead(self.prefix + "MAPHead_0/", self.width, self.mlp_dim, self.num_heads)
                     if self.pool_type == "map" else None)
    self.encoder = vit.Encoder(self.prefix + "Encoder_0/", self.depth, self.width,
                               self.mlp_dim, self.num_heads, scan=self.scan, remat_policy=self.remat_policy)
    self._len = None

  def specs(self, text_len):
    self._len = text_len
    d, p = self.width, self.prefix
    specs = [
        # flax nn.Embed default init: variance_scaling(1.0, "fan_in", "normal", out_axis=0)
        E.ParamSpec(p + "Embed_0/embedding", (self.vocab_size, d), E.normal(1 / math.sqrt(d))),
        E.ParamSpec(p + "pos_embedding", (1, text_len, d), E.normal(1 / math.sqrt(d))),
    ]
    s, aliases = self.encoder.specs()
    specs += s
    if self.map_head is not None:
      s, a = self.map_head.specs()
      specs += s
      aliases += a
    if self.num_classes:
      specs += [E.ParamSpec(p + "head/kernel", (d, self.num_classes), E.lecun_normal(d)),
                E.ParamSpec(p + "head/bias", (self.num_classes,), E.zeros)]
    return specs, aliases

  def init(self, seed, text_shape, device="cuda"):
    specs, aliases = self.specs(text_shape[1])
    return E.FlatParams(specs, aliases, device).init(seed)

  def _tok(self, Ln):
    return {"last": Ln - 1, "first": 0}.get(self.pool_type)

  def stages(self):
    """Backward stages bottom-up (storage-name prefixes): Embed_0 with pos_embedding, every encoder
    block (the scan-stacked encoder is one), encoder_norm, the MAP head, head."""
    p = self.prefix
    out = [(p + "Embed_0/", p + "pos_embedding")] + self.encoder.stages()
    out.append((p + "Encoder_0/encoder_norm/",))
    if self.map_head is not None:
      out.append((self.map_head.p,))
    if self.num_classes:
      out.append((p + "head/",))
    return out

  def _stage_indices(self):
    """Indices into stages() of encoder_norm, the MAP head and head."""
    i_norm = 1 + (1 if self.scan else self.depth)
    i_map = i_norm + 1
    return i_norm, i_map, i_map + (self.map_head is not None)

  def cut(self, P, frozen):
    """Index into stages() of the lowest stage with a trained parameter (see vit._Model.cut)."""
    cache = self.__dict__.setdefault("_cuts", {})
    key = frozen if frozen is True or frozen is None else frozenset(frozen)
    if key not in cache:
      cache[key] = E.stage_cut(P.offsets, self.stages(), frozen)
    return cache[key]

  def fwd(self, P, text, frozen=None):
    """text int32 [n, L] -> (fp32 [n, out], saved).  `frozen` as in vit._Model.fwd: the stages below
    the cut run forward-only and save nothing."""
    n, Ln = text.shape
    d, p = self.width, self.prefix
    cut = self.cut(P, frozen)
    i_norm, i_map, i_head = self._stage_indices()
    x = ops.embed_fwd(text, P.f(p + "Embed_0/embedding"), P.f(p + "pos_embedding").view(Ln, d))
    train_from = 0 if cut <= 1 else (self.depth if self.scan else min(cut - 1, self.depth))
    x, enc_saved = self.encoder.fwd(P, x, n, Ln, train_from=train_from)
    en = p + "Encoder_0/encoder_norm/"
    saved = {"text": text, "enc": enc_saved, "n": n, "L": Ln, "cut": cut, "train_from": train_from}
    keep_norm = cut <= i_norm
    tok = self._tok(Ln)
    if tok is not None:
      # LayerNorm is per token: LN(x)[:, tok] == LN(x[:, tok]) -- normalise only the pooled row
      xt = ops.pool_fwd(x, n, Ln, 1, tok=tok)
      out, mean, rstd = ops.layernorm_fwd(xt, P.f(en + "scale"), P.f(en + "bias"))
      saved["norm"] = (xt, mean, rstd) if keep_norm else None
    else:
      encd, mean, rstd = ops.layernorm_fwd(x, P.f(en + "scale"), P.f(en + "bias"))
      saved["norm"] = (x, mean, rstd) if keep_norm else None
      if self.map_head is not None:
        out, saved["map"] = self.map_head.fwd(P, encd, n, Ln, save=cut <= i_map)
        out = vit._Model._to16(out)
      elif self.pool_type in ("max", "gmp"):
        out = ops.pool_fwd(encd, n, Ln, 2)
        saved["encd"] = encd if keep_norm else None
      else:
        out = ops.pool_fwd(encd, n, Ln, 0)
    if self.num_classes:
      saved["head_in"] = out if cut <= i_head else None
      out = ops.gemm(out, P.h(p + "head/kernel"), b_mn=True, bias=P.f(p + "head/bias"),
                     out_dtype=torch.float32)
    return out, saved

  def bwd(self, P, dout, saved):
    p, d = self.prefix, self.width
    n, Ln = saved["n"], saved["L"]
    cut, train_from = saved["cut"], saved["train_from"]
    if cut == len(self.stages()):        # wholly frozen: nothing to do
      return
    i_norm, i_map, i_head = self._stage_indices()
    en = p + "Encoder_0/encoder_norm/"
    if self.num_classes:
      d16 = vit._Model._to16(dout)
      ops.colsum(dout, P.g(p + "head/bias"))
      ops.gemm(saved["head_in"], d16, a_mn=True, b_mn=True, out=P.g(p + "head/kernel"), reduce_out=True)
      if cut == i_head:
        return
      dout = ops.gemm(d16, P.h(p + "head/kernel"))          # bf16 [n, d]
    else:
      dout = vit._Model._to16(dout)
    # below the cut the last block is frozen: its Dense_1 bias gradient stays zero
    last_b = self.encoder.last_bias_grad(P) if cut < i_norm else None
    tok = self._tok(Ln)
    if tok is not None:
      xs, mean, rstd = saved["norm"]
      dxt = ops.layernorm_bwd(dout, xs, P.f(en + "scale"), mean, rstd, dscale=P.g(en + "scale"),
                              dbias=P.g(en + "bias"), dx_colsum=last_b)
      dx = ops.pool_bwd(dxt, n, Ln, 1, tok=tok)
    else:
      if self.map_head is not None:
        denc = self.map_head.bwd(P, ops.cast(dout, torch.empty_like(dout, dtype=torch.float32)),
                                 saved["map"], n, Ln)
        if cut == i_map:
          return
      elif self.pool_type in ("max", "gmp"):
        denc = ops.pool_max_bwd(dout, saved["encd"], n, Ln)
      else:
        denc = ops.pool_bwd(dout, n, Ln, 0)
      xs, mean, rstd = saved["norm"]
      dx = ops.layernorm_bwd(denc, xs, P.f(en + "scale"), mean, rstd, dscale=P.g(en + "scale"),
                             dbias=P.g(en + "bias"), dx_colsum=last_b)
    if cut == i_norm:
      return
    dx = self.encoder.bwd(P, dx, saved["enc"], n, Ln, None, train_from=train_from)
    if cut > 0:          # Embed_0 and pos_embedding are frozen
      return
    ops.embed_bwd(saved["text"], dx, P.g(p + "Embed_0/embedding"), P.g(p + "pos_embedding").view(Ln, d))

  def apply(self, variables, text, *, train=False):
    x, _ = self.fwd(variables["params"], text, frozen=True)     # forward-only, same bits
    return x, {"logits" if self.num_classes else "pre_logits": x}


def Model(num_classes, *, variant=None, **kw):  # pylint: disable=invalid-name
  """Same factory as text_transformer.Model (text_transformer.py:102-105)."""
  return _Model(num_classes, **{**vit.decode_variant(variant), **kw})


def load(init_params, init_file, model_cfg, dont_load=()):
  """Text-tower parameters from a checkpoint (contract of text_transformer.py:107-119).  Early
  checkpoints carry a SECOND position embedding inside the encoder, applied right after the
  top-level one; the two tables are summed into the top-level parameter.  The encoder is (un)stacked
  to match `model_cfg["scan"]`."""
  from big_vision_b200 import utils
  from big_vision_b200.models import common
  tree = dict(utils.load_params(init_file))
  encoder = dict(tree["Encoder_0"])
  inner_table = encoder.pop("pos_embedding", None)
  if inner_table is not None:
    tree["pos_embedding"] = tree["pos_embedding"] + inner_table
  tree["Encoder_0"] = encoder
  stored_scanned = "encoderblock" in encoder
  if bool((model_cfg or {}).get("scan")) != stored_scanned:
    convert = vit.scan_to_pyloop if stored_scanned else vit.pyloop_to_scan
    tree = convert(tree, encoder="Encoder_0")
  return common.merge_params(tree, init_params, dont_load)
