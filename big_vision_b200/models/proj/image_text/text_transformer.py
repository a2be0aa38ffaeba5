"""Text tower on the H100 kernels -- mirror of
big_vision/models/proj/image_text/text_transformer.py:29-99.

Embed(vocab, width) + learned posemb -> the vit encoder blocks (no attention mask: none is passed at
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
from big_vision_b200.models import common, vit


class _Embed(E.Stage):
  """Embed_0 plus the learned position embedding (text_transformer.py:62-70) of `text_len` tokens."""

  def __init__(self, prefix, vocab_size, text_len, d):
    self.p, self.vocab_size, self.text_len, self.d = prefix, vocab_size, text_len, d
    self.prefixes = (prefix + "Embed_0/", prefix + "pos_embedding")

  def specs(self):
    # flax nn.Embed default init: variance_scaling(1.0, "fan_in", "normal", out_axis=0)
    d, init = self.d, E.normal(1 / math.sqrt(self.d))
    return [E.ParamSpec(self.p + "Embed_0/embedding", (self.vocab_size, d), init),
            E.ParamSpec(self.p + "pos_embedding", (1, self.text_len, d), init)], []

  def fwd(self, P, text, geom, save=True):
    Ln = geom.N
    x = ops.embed_fwd(text, P.f(self.p + "Embed_0/embedding"), P.f(self.p + "pos_embedding").view(Ln, self.d))
    return x, (text if save else None)

  def bwd(self, P, dx, text, geom, sink=None, need_dx=False):
    Ln = geom.N
    ops.embed_bwd(text, dx, P.g(self.p + "Embed_0/embedding"), P.g(self.p + "pos_embedding").view(Ln, self.d))


# pool_type -> vit.NormPool's pool ("map": encoder_norm alone, then the MAP head stage)
_POOLS = {"last": "last", "first": "first", "mean": "mean", "gap": "mean", "max": "max", "gmp": "max", "map": None}


@dataclass
class _Model(E.Staged):
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
    E.check_dropout_rate(self.dropout)
    if self.pool_type not in _POOLS:
      raise NotImplementedError(f"Cannot do pooling '{self.pool_type}'")
    vit.check_head_dim(self.width, self.num_heads)
    self.prefix = (self.name + "/") if self.name else ""

  def specs(self, text_len):
    """Builds the backward stages for [n, text_len] token ids -> (specs, aliases)."""
    p, d, enc = self.prefix, self.width, self.prefix + "Encoder_0/"
    # bottom-up; the pools and the MAP head output bf16
    stages = ([_Embed(p, self.vocab_size, text_len, d)]
              + vit.encoder_stages(enc, self.depth, d, self.mlp_dim, self.num_heads, self.scan, self.remat_policy)
              + [vit.NormPool(enc + "encoder_norm/", d, _POOLS[self.pool_type], torch.bfloat16)])
    if self.pool_type == "map":
      stages.append(vit.MAPHead(p + "MAPHead_0/", d, self.mlp_dim, self.num_heads, torch.bfloat16))
    if self.num_classes:    # text_transformer.py:97-98
      stages.append(common.Dense(p + "head/", d, self.num_classes, E.lecun_normal(d), dx_dtype=torch.bfloat16))
    return self._build(stages)

  def init(self, seed, text_shape, device="cuda"):
    specs, aliases = self.specs(text_shape[1])
    return E.FlatParams(specs, aliases, device).init(seed)

  def fwd(self, P, text, frozen=None, dropout=None):
    """text int32 [n, L] -> (fp32 [n, out], saved); bf16 [n, width] without a head.  `frozen` and `dropout`
    as in vit._Model.fwd: the stages below the cut run forward-only and save nothing.  Dropout applies in
    the encoder blocks only; the tower has no embedding dropout (text_transformer.py:68-74)."""
    n, Ln = text.shape
    return self._stages_fwd(P, text, E.Geom(n, Ln, dropout=E.dropout(self.dropout, dropout, Ln)), frozen)

  def bwd(self, P, dout, saved):
    if not self.num_classes:       # the tower's output is bf16
      dout = common.to16(dout)
    self._stages_bwd(P, dout, saved)

  def apply(self, variables, text, *, train=False):
    if train and self.dropout:
      raise ValueError("apply(train=True) with dropout > 0 has no dropout key; call fwd(..., dropout=key)")
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
