"""The dropout mask stream restated from numpy's Philox (include/bv_dropout.h), the bf16 kernels
emulated bit for bit, and float64 ViT / text towers that apply the restated masks at the reference's sites
(models/vit.py:76,100,109,228; text_transformer.py:68-75), built on the operations of oracle/bv_oracle.py."""
import numpy as np
import torch

from oracle import bv_oracle as O

F64 = torch.float64


def threshold(rate):
  """T of the drop rule: the 16-bit lanes below it are dropped (rate as the float32 the kernel sees)."""
  return int(np.rint(float(np.float32(rate)) * 65536.0))


def keep_divisor(rate):
  """1 - rate in float32: kept values are x / this."""
  return np.float32(1.0) - np.float32(rate)


def lanes(seed, step, site, start, end):
  """The 16-bit lanes of global elements [start, end): lane e % 16 of Philox block e // 16, block b being
  np.random.Philox(key=seed, counter=[0, step, site, 0]).random_raw() words 4 b .. 4 b + 3 (little-endian
  lanes: bits 16 (e % 4) of word (e % 16) // 4)."""
  b0, b1 = start // 16, (end - 1) // 16 + 1
  raw = np.random.Philox(key=seed, counter=[b0, step, site, 0]).random_raw((b1 - b0) * 4)
  return raw.astype("<u8").view("<u2")[start - 16 * b0:end - 16 * b0]


def keep_mask(seed, step, site, row0, rows, cols, rate):
  """bool [rows, cols]: True where the element of global row row0 + r, column c is kept."""
  start = row0 * cols
  return (lanes(seed, step, site, start, start + rows * cols) >= threshold(rate)).reshape(rows, cols)


def key_mask(key, rate, rows, cols):
  """keep_mask of a lib.DropoutKey."""
  return keep_mask(key.seed, key.step, key.site, key.row0, rows, cols, rate)


def dropout_bf16(x, keep, rate, resid=None):
  """The kernels' result for a float32 CPU tensor x of bf16 values: bf16(x / (1 - rate)) where kept, else 0;
  with resid, bf16(resid + that float32 quotient)."""
  q = x.float() / float(keep_divisor(rate))   # float32 / float32: IEEE, rounded to nearest
  q = torch.where(torch.from_numpy(keep), q, torch.zeros_like(q))
  if resid is not None:
    q = resid.float() + q
  return q.bfloat16()


class Masks:
  """Scaled float64 masks (keep / (1 - rate)) of one tower's sites for rows [row0, row0 + n * N)."""

  def __init__(self, rate, seed, step, sample0=0, tower=0):
    from big_vision_b200 import engine as E
    self.E, self.rate, self.seed, self.step, self.sample0, self.tower = E, rate, seed, step, sample0, tower

  def __call__(self, x, layer, kind):
    n, N, d = x.shape
    site = self.E.dropout_site(self.tower, layer, kind)
    keep = keep_mask(self.seed, self.step, site, self.sample0 * N, n * N, d, self.rate)
    return x * torch.from_numpy(keep.reshape(n, N, d)).to(F64) / float(keep_divisor(self.rate))


def encoder(x, p, depth, heads, masks):
  """vit.Encoder (models/vit.py:115-160) with dropout at the three block sites; returns the encoder_norm
  output."""
  E = masks.E
  for i in range(depth):
    b = O.sub(p, f"encoderblock_{i}/")
    y = O.layer_norm(x, b["LayerNorm_0/scale"], b["LayerNorm_0/bias"])
    y = O.mha(y, y, O.sub(b, "MultiHeadDotProductAttention_0/"), heads, "float32")
    x = x + masks(y, i, E.DROP_ATTN)
    y = O.layer_norm(x, b["LayerNorm_1/scale"], b["LayerNorm_1/bias"])
    m = O.sub(b, "MlpBlock_0/")
    h = masks(O.gelu_tanh(O.dense(y, m["Dense_0/kernel"], m["Dense_0/bias"], "float32")), i, E.DROP_GELU)
    x = x + masks(O.dense(h, m["Dense_1/kernel"], m["Dense_1/bias"], "float32"), i, E.DROP_MLP)
  return O.layer_norm(x, p["encoder_norm/scale"], p["encoder_norm/bias"])


def vit_forward(p, image, cfg, masks):
  """O.vit_forward in float64 with dropout after the embedding and in every encoder block."""
  image = image.to(F64)
  x = O.patch_embed(image, p["embedding/kernel"], p["embedding/bias"], "float32")
  n, _, d = x.shape
  if cfg.get("posemb", "learn") == "learn":
    x = x + p["pos_embedding"]
  else:
    ph, pw = p["embedding/kernel"].shape[:2]
    x = x + torch.from_numpy(O.posemb_sincos_2d(image.shape[1] // ph, image.shape[2] // pw, d)).to(F64)
  if cfg["pool_type"] == "tok":
    x = torch.cat([p["cls"].expand(n, -1, -1), x], dim=1)
  x = masks(x, 0, masks.E.DROP_EMBED)
  x = encoder(x, O.sub(p, "Transformer/"), cfg["depth"], cfg["num_heads"], masks)
  if cfg["pool_type"] == "map":
    x = O.map_head(x, O.sub(p, "MAPHead_0/"), cfg["num_heads"], "float32")
  elif cfg["pool_type"] == "gap":
    x = x.mean(1)
  elif cfg["pool_type"] in ("0", "tok"):
    x = x[:, 0]
  else:
    raise ValueError(cfg["pool_type"])
  if cfg.get("num_classes"):
    x = O.dense(x, p["head/kernel"], p["head/bias"], "float32")
  return x


def text_forward(p, text, cfg, masks):
  """O.text_forward in float64 with dropout in the encoder blocks only (no embedding dropout)."""
  x = p["Embed_0/embedding"][text.long()] + p["pos_embedding"]
  x = encoder(x, O.sub(p, "Encoder_0/"), cfg["depth"], cfg["num_heads"], masks)
  pool = cfg.get("pool_type", "last")
  if pool == "last":
    x = x[:, -1, :]
  elif pool == "map":
    x = O.map_head(x, O.sub(p, "MAPHead_0/"), cfg["num_heads"], "float32")
  else:
    raise NotImplementedError(pool)
  if cfg.get("num_classes"):
    x = O.dense(x, p["head/kernel"], p["head/bias"], "float32")
  return x


def two_towers_forward(p, image, text, cfg, rate_img, rate_txt, seed, step, sample0=0):
  """O.two_towers_forward with each tower's dropout: the image tower draws as tower 0, the text as tower 1."""
  ztxt = O.l2_normalize(text_forward(O.sub(p, "txt/"), text, cfg["text"], Masks(rate_txt, seed, step, sample0, 1)))
  zimg = O.l2_normalize(vit_forward(O.sub(p, "img/"), image, cfg["image"], Masks(rate_img, seed, step, sample0, 0)))
  return zimg, ztxt
