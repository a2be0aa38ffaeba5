"""BERT dropout restated: the attention-probability mask stream of include/bv_dropout.h from numpy's Philox,
float64 masked attention with dropped probabilities, and the float64 BERT tower of tests/bert_oracle.py with
given masks at the original BERT's four sites (embedding LayerNorm output, attention probabilities, attention
output, MLP output), built on the operations of oracle/bv_oracle.py."""
import math

import numpy as np
import torch

import dropout_oracle as D
from oracle.bv_oracle import dense, gelu_tanh, layer_norm, rnd, sub

EPS = 1e-12
F64 = torch.float64


def attn_lanes(seed, step, site, row, Nk):
  """The 16-bit lanes of the Nk probabilities of global row `row`: key k uses lane k % 16 of block k // 16,
  np.random.Philox(key=seed, counter=[0, step, site, row + 1]).random_raw() words 4 b .. 4 b + 3."""
  raw = np.random.Philox(key=seed, counter=[0, step, site, row + 1]).random_raw(4 * ((Nk + 15) // 16))
  return raw.astype("<u8").view("<u2")[:Nk]


def attn_keep(seed, step, site, row0, B, H, Nq, Nk, rate):
  """bool [B, H, Nq, Nk]: True where probability (b, h, q, k) is kept; its row is row0 + (b H + h) Nq + q."""
  T = D.threshold(rate)
  rows = [attn_lanes(seed, step, site, row0 + r, Nk) >= T for r in range(B * H * Nq)]
  return np.stack(rows).reshape(B, H, Nq, Nk)


def attn_keep_of(key, B, H, Nq, Nk):
  """attn_keep of a lib.DropoutKey."""
  return attn_keep(key.seed, key.step, key.site, key.row0, B, H, Nq, Nk, key.rate)


def scaled(keep, rate):
  """float64 keep / (1 - rate), the divisor in float32 as the kernels compute it."""
  return torch.from_numpy(keep).to(F64) / float(D.keep_divisor(rate))


def attention(q, k, v, key_mask, probs_scale):
  """float64 attention of q, k, v [B, H, N, dh] with a key mask [B, Nk] (True = attend) and the scaled keep
  mask [B, H, Nq, Nk] of the probabilities (None: no dropout) -> (o [B, H, Nq, dh], lse [B, H, Nq]).  lse is
  that of the undropped softmax; a query with no attended key gets o = 0 and lse = 0."""
  s = (q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1])
  live = key_mask[:, None, None, :]
  any_live = live.any(-1, keepdim=True)
  m = torch.where(any_live, s.masked_fill(~live, -math.inf).amax(-1, keepdim=True), 0.0).detach()
  e = torch.where(live, torch.exp(s - m), 0.0)
  den = e.sum(-1, keepdim=True)
  p = e / torch.where(any_live, den, 1.0)
  lse = torch.where(any_live, m + torch.log(torch.where(any_live, den, 1.0)), 0.0)[..., 0]
  if probs_scale is not None:
    p = p * probs_scale
  return p @ v, lse


def masked_mha(x, p, heads, key_mask, probs_scale, mm):
  """tests/bert_oracle.masked_mha with the attention probabilities multiplied by `probs_scale` (None: none)."""
  B, N, d = x.shape
  dh = d // heads

  def proj(name):
    y = rnd(dense(x, p[name + "/kernel"].reshape(d, d), p[name + "/bias"].reshape(d), mm), mm)
    return y.reshape(B, N, heads, dh).transpose(1, 2)

  q, k, v = proj("query"), proj("key"), proj("value")
  s = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
  live = key_mask[:, None, None, :]
  s = s.masked_fill(~live, -math.inf)
  any_live = live.any(-1, keepdim=True)
  m = torch.where(any_live, s.amax(-1, keepdim=True), 0.0).detach()
  e = torch.where(live, torch.exp(s - m), 0.0)
  den = torch.where(any_live, e.sum(-1, keepdim=True), 1.0)
  e = rnd(e, mm)
  if probs_scale is not None:
    e = e * probs_scale
  o = rnd((e @ v) / den, mm).transpose(1, 2).reshape(B, N, d)
  return dense(o, p["out/kernel"].reshape(d, d), p["out/bias"], mm)


def bert_forward(p, text, cfg, masks, key_mask=None, mm="float32"):
  """tests/bert_oracle.bert_forward with dropout: masks.hidden(x, layer, kind) -> x times its scaled mask at
  the hidden sites (kinds engine.DROP_EMBED, DROP_ATTN, DROP_MLP) and masks.probs(layer, B, H, N) -> the
  scaled float64 mask of the attention probabilities of layer `layer`."""
  from big_vision_b200 import engine as E
  if key_mask is None:
    key_mask = text != 0
  e = sub(p, "BertEncoder_0/embedder/")
  B, N = text.shape
  heads = cfg["num_heads"]
  x = (e["embedders_token_ids/embedding"][text] + e["embedders_position_ids/embedding"][:N]
       + e["embedders_segment_ids/embedding"][0])
  x = rnd(masks.hidden(rnd(layer_norm(x, e["layer_norm/scale"], e["layer_norm/bias"], eps=EPS), mm), 0,
                       E.DROP_EMBED), mm)
  for i in range(cfg["depth"]):
    lp = sub(p, f"BertEncoder_0/encoder_layer_{i}/")
    y = rnd(masked_mha(x, sub(lp, "self_attention/"), heads, key_mask, masks.probs(i, B, heads, N), mm), mm)
    x = rnd(x + masks.hidden(y, i, E.DROP_ATTN), mm)
    x = rnd(layer_norm(x, lp["attention_layer_norm/scale"], lp["attention_layer_norm/bias"], eps=EPS), mm)
    m = sub(lp, "mlp/")
    h = rnd(dense(x, m["Dense_0/kernel"], m["Dense_0/bias"], mm), mm)
    h = rnd(gelu_tanh(h), mm)
    y = rnd(dense(h, m["Dense_1/kernel"], m["Dense_1/bias"], mm), mm)
    x = rnd(x + masks.hidden(y, i, E.DROP_MLP), mm)
    x = rnd(layer_norm(x, lp["output_layer_norm/scale"], lp["output_layer_norm/bias"], eps=EPS), mm)
  x = x[:, 0]
  if cfg.get("num_classes"):
    x = dense(x, p["head/kernel"], p["head/bias"], mm)
  return x


class PhiloxMasks:
  """The masks the BERT tower draws under engine.DropoutKey(seed, step, sample0, tower) at hidden rate `rate`
  and attention rate `attn_rate`, restated from numpy's Philox."""

  def __init__(self, rate, attn_rate, seed, step, sample0=0, tower=0):
    self.rate, self.attn_rate, self.seed, self.step, self.sample0, self.tower = (rate, attn_rate, seed, step,
                                                                                  sample0, tower)

  def hidden(self, x, layer, kind):
    if not self.rate:
      return x
    from big_vision_b200 import engine as E
    n, N, d = x.shape
    site = E.dropout_site(self.tower, layer, kind)
    keep = D.keep_mask(self.seed, self.step, site, self.sample0 * N, n * N, d, self.rate).reshape(n, N, d)
    return x * scaled(keep, self.rate).to(x.device)

  def probs(self, layer, B, H, N):
    if not self.attn_rate:
      return None
    from big_vision_b200 import engine as E
    site = E.dropout_site(self.tower, layer, E.DROP_ATTN)
    return scaled(attn_keep(self.seed, self.step, site, self.sample0 * H * N, B, H, N, N, self.attn_rate),
                  self.attn_rate)


class GivenMasks:
  """Masks given as arrays: hidden[(layer, kind)] float64 [n, N, d] and probs[layer] float64 [B, H, N, N], both
  already scaled by 1 / (1 - rate)."""

  def __init__(self, hidden, probs):
    self.h, self.p = hidden, probs

  def hidden(self, x, layer, kind):
    return x * self.h[(layer, kind)]

  def probs(self, layer, B, H, N):
    return self.p[layer]
