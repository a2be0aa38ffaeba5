"""float64 oracle of the BERT text tower (big_vision_b200/models/proj/flaxformer/bert.py) with an explicit
key mask, on torch-CPU with autograd gradients; the helpers are oracle/bv_oracle.py's.

`bert_forward` follows the original BERT (google-research/bert modeling.py): token + position +
segment-0 embeddings, embedding LayerNorm, post-LN layers x = LN(x + Attn(x)); x = LN(x + MLP(x)) with
LayerNorm eps 1e-12 and tanh GELU, then x[:, 0] and the optional head.  mm="bfloat16" rounds where the
kernels store bf16.  `mask_queries=True` also masks the padded queries the way flaxformer's
attention does (an additive finfo.min bias on every (query, key) pair with either side padded), which
must not change the [CLS] output or any parameter gradient."""
import math

import numpy as np
import torch

from oracle.bv_oracle import dense, gelu_tanh, layer_norm, rnd, sub

EPS = 1e-12


def masked_mha(x, p, heads, key_mask, mm, mask_queries=False):
  """Self-attention with a key mask [B, N] (True = attend).  A query with no attended key gets 0
  (the kernels' convention); with mask_queries the padded queries get flaxformer's finfo.min bias."""
  B, N, d = x.shape
  dh = d // heads

  def proj(name):
    y = rnd(dense(x, p[name + "/kernel"].reshape(d, d), p[name + "/bias"].reshape(d), mm), mm)
    return y.reshape(B, N, heads, dh).transpose(1, 2)

  q, k, v = proj("query"), proj("key"), proj("value")
  s = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
  keys = key_mask[:, None, None, :]
  if mask_queries:
    both = keys & key_mask[:, None, :, None]
    s = s + torch.where(both, torch.zeros((), dtype=s.dtype), torch.tensor(torch.finfo(s.dtype).min, dtype=s.dtype))
    live = torch.ones_like(both)
  else:
    live = keys
    s = s.masked_fill(~keys, -math.inf)
  any_live = live.any(-1, keepdim=True)
  m = torch.where(any_live, s.masked_fill(~live, -math.inf).amax(-1, keepdim=True), 0.0).detach()
  e = torch.where(live, torch.exp(s - m), 0.0)
  den = e.sum(-1, keepdim=True)
  o = (rnd(e, mm) @ v) / torch.where(any_live, den, 1.0)
  o = rnd(o, mm).transpose(1, 2).reshape(B, N, d)
  return dense(o, p["out/kernel"].reshape(d, d), p["out/bias"], mm)


def bert_forward(p, text, cfg, key_mask=None, mm="float32", mask_queries=False):
  """p: flat dict under the model's names (without the tower prefix); text int [B, N]; cfg: depth,
  num_heads, num_classes.  key_mask: bool [B, N] (default text != 0) -> fp64 [B, out]."""
  if key_mask is None:
    key_mask = text != 0
  e = sub(p, "BertEncoder_0/embedder/")
  N = text.shape[1]
  x = (e["embedders_token_ids/embedding"][text] + e["embedders_position_ids/embedding"][:N]
       + e["embedders_segment_ids/embedding"][0])
  x = rnd(layer_norm(x, e["layer_norm/scale"], e["layer_norm/bias"], eps=EPS), mm)
  for i in range(cfg["depth"]):
    lp = sub(p, f"BertEncoder_0/encoder_layer_{i}/")
    y = rnd(masked_mha(x, sub(lp, "self_attention/"), cfg["num_heads"], key_mask, mm, mask_queries), mm)
    x = rnd(x + y, mm)
    x = rnd(layer_norm(x, lp["attention_layer_norm/scale"], lp["attention_layer_norm/bias"], eps=EPS), mm)
    m = sub(lp, "mlp/")
    h = rnd(dense(x, m["Dense_0/kernel"], m["Dense_0/bias"], mm), mm)
    h = rnd(gelu_tanh(h), mm)
    y = rnd(dense(h, m["Dense_1/kernel"], m["Dense_1/bias"], mm), mm)
    x = rnd(x + y, mm)
    x = rnd(layer_norm(x, lp["output_layer_norm/scale"], lp["output_layer_norm/bias"], eps=EPS), mm)
  x = x[:, 0]
  if cfg.get("num_classes"):
    x = dense(x, p["head/kernel"], p["head/bias"], mm)
  return x


def padded_text(n, length, vocab, seed, min_len=1):
  """Token ids as the reference's BERT tokenizer writes them (pp/proj/flaxformer/bert_ops.py:77-83): a
  first token that is never 0, then tokens, zero-padded to `length`; caption 0 has no padding."""
  rng = np.random.default_rng(seed)
  text = np.zeros((n, length), dtype=np.int32)
  lens = rng.integers(min_len, length + 1, size=n)
  lens[0] = length
  for i in range(n):
    text[i, :lens[i]] = rng.integers(1, vocab, size=lens[i])
  return text
