"""BERT text encoder on the H100 kernels -- mirror of big_vision/models/proj/flaxformer/bert.py.

Same factory (`Model(config, num_classes=None, head_zeroinit=True)`, config "base" or "large") and the
same `load`.  The reference builds flaxformer's `BertEncoder` (bert.py:45-56); flaxformer is not
available here, so the maths follows the original BERT that its checkpoint converter loads
(google-research/bert `modeling.py`), none of it checked against flaxformer itself:
  token + position + segment embeddings (segment ids all 0, bert.py:53) -> LayerNorm ->
  post-LN layers  x = LN(x + Attn(x));  x = LN(x + MLP(x))  (LayerNorm eps 1e-12, tanh GELU) ->
  x[:, 0] ([CLS], bert.py:58; no final norm) -> Dense head (bert.py:60-62).
The attention masks the padded keys, `input_mask = text != 0` (bert.py:54): token id 0 is the padding
of the reference's tokenizer.  Padded queries are not masked; their rows never reach [CLS] (every
later layer masks them as keys, every other op is per token), so the output and every parameter
gradient are those of a model that also masks them.

Dropout (bert.py:55 builds the encoder with enable_dropout=train), placed as the original BERT's
hidden_dropout_prob and attention_probs_dropout_prob (and transformers' BertModel): after the embedding
LayerNorm, on the attention probabilities, on the attention output and on the MLP output, each before its
residual add and LayerNorm; the GELU output is not dropped.  "base" and "large" train at 0.1 for both, as the
original BERT does.  The masks come from `fwd(..., dropout=engine.DropoutKey)` (include/bv_dropout.h): the
hidden sites (layer, kind) of engine.dropout_site with kinds EMBED, ATTN and MLP, and the attention
probabilities in the attention kernels under the layer's ATTN site.  The backward regenerates every mask.
They are not the reference's masks (jax's threefry is not reproduced).

Not built: the full-sequence `out["transformed"]`, and loading the original TF checkpoint (needs tensorflow).

Parameter names: the reference shows `BertEncoder_0/embedder/embedders_position_ids/embedding`
(bert.py:76-77) and `head/*`; every other name under `BertEncoder_0/` is this port's choice (DESIGN §4).
"""
import os
from dataclasses import dataclass
from typing import Optional, Union

import numpy as np
import torch

from big_vision_b200 import engine as E
from big_vision_b200 import lib as L
from big_vision_b200 import ops
from big_vision_b200.models import common, vit

# width, depth, num_heads, mlp_dim of BERT-Base / BERT-Large, and the original BERT's hidden_dropout_prob and
# attention_probs_dropout_prob; vocabulary, positions and segments of the original BERT's uncased vocabulary
# (both sizes)
CONFIGS = {
    "base": dict(width=768, depth=12, num_heads=12, mlp_dim=3072, dropout_rate=0.1, attention_dropout_rate=0.1),
    "large": dict(width=1024, depth=24, num_heads=16, mlp_dim=4096, dropout_rate=0.1, attention_dropout_rate=0.1),
}
VOCAB_SIZE, MAX_POSITIONS, SEGMENTS = 30_522, 512, 2
LN_EPS = 1e-12
PAD_ID = 0


def trunc_normal(std):
  """BERT's initializer: tf.truncated_normal_initializer(stddev=std), cut at two standard deviations."""
  def init(rng, shape):
    x = rng.standard_normal(size=shape)
    bad = np.abs(x) > 2
    while bad.any():
      x[bad] = rng.standard_normal(size=int(bad.sum()))
      bad = np.abs(x) > 2
    return x * std
  return init


class _Embed(E.Stage):
  """Token + position + segment-0 embeddings, then the embedding LayerNorm and its dropout.  The position
  table has MAX_POSITIONS rows; a forward of N tokens reads rows 0..N-1."""

  def __init__(self, prefix, d, vocab_size):
    self.p, self.d, self.vocab_size = prefix + "embedder/", d, vocab_size
    self.prefixes = (self.p,)

  def specs(self):
    init, d = trunc_normal(0.02), self.d
    return ([E.ParamSpec(self.p + "embedders_token_ids/embedding", (self.vocab_size, d), init),
             E.ParamSpec(self.p + "embedders_position_ids/embedding", (MAX_POSITIONS, d), init),
             E.ParamSpec(self.p + "embedders_segment_ids/embedding", (SEGMENTS, d), init)]
            + vit.ln_specs(self.p + "layer_norm/", d)), []

  def fwd(self, P, text, geom, save=True):
    N, p = geom.N, self.p
    # every token has segment 0: its row is folded into the N position rows (fp32)
    seg0 = ops.broadcast_row(P.f(p + "embedders_segment_ids/embedding")[0:1], N)
    pos = ops.axpby(P.f(p + "embedders_position_ids/embedding")[:N], seg0)
    x = ops.embed_fwd(text, P.f(p + "embedders_token_ids/embedding"), pos, out_dtype=torch.float32)
    y, mean, rstd = ops.layernorm_fwd(x, P.f(p + "layer_norm/scale"), P.f(p + "layer_norm/bias"), eps=LN_EPS)
    if geom.dropout is not None:
      ops.dropout(y, geom.dropout.mask(0, E.DROP_EMBED), out=y)
    return y, ((text, x, mean, rstd) if save else None)

  def bwd(self, P, dy, saved, geom, sink=None, need_dx=False):
    N, p = geom.N, self.p
    text, x, mean, rstd = saved
    if geom.dropout is not None:
      dy = ops.dropout(dy, geom.dropout.mask(0, E.DROP_EMBED))
    dx = ops.layernorm_bwd(dy, x, P.f(p + "layer_norm/scale"), mean, rstd, dx_dtype=torch.float32,
                           dscale=P.g(p + "layer_norm/scale"), dbias=P.g(p + "layer_norm/bias"))
    dpos = torch.zeros((N, self.d), dtype=torch.float32, device=dx.device)
    ops.embed_bwd(text, dx, P.g(p + "embedders_token_ids/embedding"), dpos)
    gpos = P.g(p + "embedders_position_ids/embedding")[:N]
    ops.axpby(gpos, dpos, out=gpos)
    ops.colsum(dpos, P.g(p + "embedders_segment_ids/embedding")[0])


class _Layer(E.Stage):
  """One post-LN encoder layer: x1 = LN(x + Attn(x)), x2 = LN(x1 + MLP(x1)), with the forward's key
  mask (geom.key_mask) in the attention.  Under dropout, x1 = LN(x + drop(Attn(x))) with the attention
  probabilities dropped too (geom.attn_dropout), and x2 = LN(x1 + drop(MLP(x1)))."""

  def __init__(self, prefix, d, m, heads, layer):
    self.p, self.d, self.m, self.heads, self.layer = prefix, d, m, heads, layer
    self.prefixes = (prefix,)
    self.ready = prefix + "self_attention/qkv/kernel"      # its first spec: see vit.EncoderBlock

  def specs(self):
    s, a = vit.mha_specs(self.p + "self_attention/", self.d, self.heads)
    mlp = vit.mlp_specs(self.p + "mlp/", self.d, self.m)
    for spec in s + mlp:
      spec.init = trunc_normal(0.02) if spec.name.endswith("kernel") else E.zeros
    return (s + vit.ln_specs(self.p + "attention_layer_norm/", self.d) + mlp
            + vit.ln_specs(self.p + "output_layer_norm/", self.d)), a

  def fwd(self, P, x, geom, save=True):
    n, N, d = geom.n, geom.N, self.d
    S = vit.Scope(P, self.p)
    A, M = S.sub("self_attention/"), S.sub("mlp/")
    dr, pdrop = geom.dropout, self.probs_key(geom)
    qkv = ops.gemm(x, A.h("qkv/kernel"), b_mn=True, bias=A.f("qkv/bias")).view(n, N, 3 * d)
    o, lse = ops.attention_fwd(qkv[:, :, 0:d], qkv[:, :, d:2 * d], qkv[:, :, 2 * d:], self.heads,
                               key_mask=geom.key_mask, dropout=pdrop)
    if dr is None:
      h1 = ops.gemm(o.view(n * N, d), A.h("out_proj/kernel"), b_mn=True, bias=A.f("out/bias"), aux=x,
                    epilogue=L.EPI_BIAS_RESID)
    else:    # transformers' BertSelfOutput: the attention output is dropped before the residual add
      h1 = ops.gemm(o.view(n * N, d), A.h("out_proj/kernel"), b_mn=True, bias=A.f("out/bias"))
      h1 = ops.dropout_add(x, h1, dr.mask(self.layer, E.DROP_ATTN), out=h1)
    x1, mean1, rstd1 = ops.layernorm_fwd(h1, S.f("attention_layer_norm/scale"), S.f("attention_layer_norm/bias"),
                                         eps=LN_EPS)
    # BertOutput: the MLP output is dropped before the residual add; the GELU output is not
    drop = None if dr is None else (None, dr.mask(self.layer, E.DROP_MLP))
    h2, mlp_saved = vit.mlp_fwd(M, x1, x1, save=save, drop=drop)
    x2, mean2, rstd2 = ops.layernorm_fwd(h2, S.f("output_layer_norm/scale"), S.f("output_layer_norm/bias"),
                                         eps=LN_EPS)
    if not save:
      return x2, None
    return x2, (x, qkv, o, lse, h1, mean1, rstd1, mlp_saved, h2, mean2, rstd2)

  def probs_key(self, geom):
    """The lib.DropoutKey of this layer's attention probabilities, or None."""
    return None if geom.attn_dropout is None else geom.attn_dropout.probs(self.layer, self.heads)

  def bwd(self, P, dx2, saved, geom, sink=None, need_dx=True):
    """Under dropout the forward's masks are regenerated: the gradients entering the MLP and the attention
    output projection are masked, and their output biases are summed from the masked gradients; the
    residual stream's gradient is not masked."""
    n, N, d = geom.n, geom.N, self.d
    S = vit.Scope(P, self.p)
    A, M = S.sub("self_attention/"), S.sub("mlp/")
    x, qkv, o, lse, h1, mean1, rstd1, (x1, act, pre), h2, mean2, rstd2 = saved
    dr = geom.dropout
    # output LayerNorm; without dropout the column sum of its input gradient is the MLP's output bias gradient
    dh2 = ops.layernorm_bwd(dx2, h2, S.f("output_layer_norm/scale"), mean2, rstd2,
                            dscale=S.g("output_layer_norm/scale"), dbias=S.g("output_layer_norm/bias"),
                            dx_colsum=M.g("Dense_1/bias") if dr is None else None)
    dm = dh2 if dr is None else ops.dropout(dh2, dr.mask(self.layer, E.DROP_MLP), colsum_into=M.g("Dense_1/bias"))
    # MLP (vit.mlp_bwd, with the residual dh2 added in the last GEMM's epilogue)
    ops.gemm(act, dm, a_mn=True, b_mn=True, out=M.g("Dense_1/kernel"), reduce_out=True)
    dpre = ops.gemm(dm, M.h("Dense_1/kernel"), aux=pre, epilogue=L.EPI_DGELU, colsum=M.g("Dense_0/bias"))
    del dm
    ops.gemm(x1, dpre, a_mn=True, b_mn=True, out=M.g("Dense_0/kernel"), reduce_out=True)
    dx1 = ops.gemm(dpre, M.h("Dense_0/kernel"), aux=dh2, epilogue=L.EPI_BIAS_RESID)
    del dpre, dh2
    # attention LayerNorm; without dropout the column sum of its input gradient is the output projection's
    # bias gradient
    dh1 = ops.layernorm_bwd(dx1, h1, S.f("attention_layer_norm/scale"), mean1, rstd1,
                            dscale=S.g("attention_layer_norm/scale"), dbias=S.g("attention_layer_norm/bias"),
                            dx_colsum=A.g("out/bias") if dr is None else None)
    del dx1
    da = dh1 if dr is None else ops.dropout(dh1, dr.mask(self.layer, E.DROP_ATTN), colsum_into=A.g("out/bias"))
    ops.gemm(o.view(n * N, d), da, a_mn=True, b_mn=True, out=A.g("out_proj/kernel"), reduce_out=True)
    do = ops.gemm(da, A.h("out_proj/kernel"))
    del da
    dqkv = torch.empty_like(qkv)
    gb = A.g("qkv/bias")
    ops.attention_bwd(do.view(n, N, d), qkv[:, :, 0:d], qkv[:, :, d:2 * d], qkv[:, :, 2 * d:], o, lse,
                      self.heads, dq=dqkv[:, :, 0:d], dk=dqkv[:, :, d:2 * d], dv=dqkv[:, :, 2 * d:],
                      dq_colsum=gb[0:d], dk_colsum=gb[d:2 * d], dv_colsum=gb[2 * d:], key_mask=geom.key_mask,
                      dropout=self.probs_key(geom))
    del do
    dqkv = dqkv.view(n * N, 3 * d)
    ops.gemm(x, dqkv, a_mn=True, b_mn=True, out=A.g("qkv/kernel"), reduce_out=True)
    if not need_dx:
      return None
    return ops.gemm(dqkv, A.h("qkv/kernel"), aux=dh1, epilogue=L.EPI_BIAS_RESID)    # + the residual


class _ClsPool(E.Stage):
  """x[:, 0]: the [CLS] token of the last layer (bert.py:58).  No parameters."""
  prefixes = ()

  def specs(self):
    return [], []

  def fwd(self, P, x, geom, save=True):
    return ops.pool_fwd(x, geom.n, geom.N, 1, tok=0), (True if save else None)

  def bwd(self, P, dy, saved, geom, sink=None, need_dx=True):
    return ops.pool_bwd(dy, geom.n, geom.N, 1, tok=0) if need_dx else None


@dataclass
class Model(E.Staged):
  """BERT encoder with a linear projection of the [CLS] token (bert.py:33-64).  `config`: "base",
  "large", or a dict with width, depth, num_heads and mlp_dim (and optionally `vocab_size`, and the dropout
  rates `dropout_rate` and `attention_dropout_rate`, 0.0 when missing) for other sizes."""
  config: Union[str, dict] = "base"
  num_classes: Optional[int] = None
  head_zeroinit: bool = True
  name: str = ""

  def __post_init__(self):
    cfg = dict(CONFIGS[self.config]) if isinstance(self.config, str) else dict(self.config)
    self.vocab_size = cfg.pop("vocab_size", VOCAB_SIZE)
    self.dropout_rate = float(cfg.pop("dropout_rate", 0.0))
    self.attention_dropout_rate = float(cfg.pop("attention_dropout_rate", 0.0))
    E.check_dropout_rate(self.dropout_rate)
    E.check_dropout_rate(self.attention_dropout_rate)
    self.width, self.depth, self.num_heads, self.mlp_dim = (cfg[k] for k in ("width", "depth", "num_heads",
                                                                              "mlp_dim"))
    vit.check_head_dim(self.width, self.num_heads)
    if self.width // self.num_heads != 64:
      raise NotImplementedError(f"BERT needs the key-masked attention, built at head dim 64 only (width "
                                f"{self.width} / {self.num_heads} heads)")
    self.prefix = (self.name + "/") if self.name else ""

  def specs(self, text_len):
    """Builds the backward stages for [n, text_len] token ids -> (specs, aliases)."""
    if text_len > MAX_POSITIONS:
      raise ValueError(f"BERT has {MAX_POSITIONS} positions, got {text_len} tokens")
    p, d = self.prefix, self.width
    enc = p + "BertEncoder_0/"
    stages = ([_Embed(enc, d, self.vocab_size)]
              + [_Layer(f"{enc}encoder_layer_{i}/", d, self.mlp_dim, self.num_heads, i) for i in range(self.depth)]
              + [_ClsPool()])
    if self.num_classes:     # bert.py:60-62
      init = E.zeros if self.head_zeroinit else E.lecun_normal(d)
      stages.append(common.Dense(p + "head/", d, self.num_classes, init, dx_dtype=torch.bfloat16))
    return self._build(stages)

  def init(self, seed, text_shape, device="cuda"):
    specs, aliases = self.specs(text_shape[1])
    return E.FlatParams(specs, aliases, device).init(seed)

  def fwd(self, P, text, frozen=None, dropout=None):
    """text int32 [n, L], zero-padded -> (fp32 [n, num_classes] or bf16 [n, width], saved).  `frozen` as
    in vit._Model.fwd.  `dropout`: the engine.DropoutKey of a training forward; without one (or at rates 0)
    no dropout is applied, as with train=False.  Frozen stages drop too."""
    key_mask = text != PAD_ID           # bert.py:54: input_mask = text != 0
    n, N = text.shape
    geom = E.Geom(n, N, key_mask=key_mask, dropout=E.dropout(self.dropout_rate, dropout, N),
                  attn_dropout=E.dropout(self.attention_dropout_rate, dropout, N))
    return self._stages_fwd(P, text, geom, frozen)

  def bwd(self, P, dout, saved):
    if not self.num_classes:       # the tower's output is bf16
      dout = common.to16(dout)
    self._stages_bwd(P, dout, saved)

  def apply(self, variables, text, *, train=False):
    """(x, out) like the flax apply, forward-only.  train=True is refused: it enables dropout, whose masks
    need a key, which apply() has no argument for; a training forward is fwd(..., dropout=key)."""
    if train:
      raise NotImplementedError("BERT dropout needs a dropout key, which apply() has no argument for; call "
                                "fwd(..., dropout=key) for a training forward")
    x, _ = self.fwd(variables["params"], text, frozen=True)
    return x, {"logits" if self.num_classes else "pre_logits": x}


def load(params, path, model_cfg=None, dont_load=()):
  """`params` with BERT weights from `path` (contract of bert.py:67-94): this repo's .npz tree
  ("file.npz[:sub/tree]"), the reference's fallback path.  A directory with the original TF checkpoint
  (`{path}/bert_model.ckpt`) is refused: converting it needs tensorflow and flaxformer's converter."""
  del model_cfg
  from big_vision_b200 import utils
  if os.path.exists(f"{path}/bert_model.ckpt.index"):
    raise NotImplementedError(
        f"{path}/bert_model.ckpt is an original TF BERT checkpoint; reading it needs tensorflow and "
        "flaxformer's bert_checkpoint_converter, which this port does not use. Convert it to an .npz tree "
        "under the parameter names of big_vision_b200.models.proj.flaxformer.bert and load that.")
  return common.merge_params(utils.load_params(path), params, dont_load)
