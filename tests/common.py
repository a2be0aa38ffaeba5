"""Shared tiny configurations for the tests (kept small so the CPU oracle runs in seconds), and the parse of
the C ABI headers."""
import glob
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# every header of the C ABI of libbv_b200.so
HEADERS = sorted(glob.glob(os.path.join(ROOT, "include", "bv_b200*.h")))

TINY = dict(
    image=dict(width=64, depth=2, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type="map"),
    text=dict(width=64, depth=2, mlp_dim=128, num_heads=1, vocab_size=64),
    out_dim=(None, 64), temperature_init=10.0, bias_init=-10.0,
)
TINY_IMAGE_SHAPE = (8, 64, 64, 3)
TINY_TEXT_SHAPE = (8, 16)


def oracle_cfg(model_kw):
  return {
      "image": dict(depth=model_kw["image"]["depth"], num_heads=model_kw["image"]["num_heads"],
                    pool_type=model_kw["image"].get("pool_type", "gap"),
                    posemb=model_kw["image"].get("posemb", "learn"),
                    rep_size=model_kw["image"].get("rep_size", False),
                    num_classes=model_kw["out_dim"][0]),
      "text": dict(depth=model_kw["text"]["depth"], num_heads=model_kw["text"]["num_heads"],
                   pool_type=model_kw["text"].get("pool_type", "last"),
                   num_classes=model_kw["out_dim"][1]),
  }


def synthetic_batch(image_shape, text_shape, vocab, seed=0):
  """SURVEY.md 8d synthetic inputs: images U(-1,1); text ids in [2,vocab) for a random length,
  then sticky EOS / pad id 1 to the end (so the last token is always 1)."""
  rng = np.random.default_rng(seed)
  image = rng.uniform(-1, 1, size=image_shape).astype(np.float32)
  n, L = text_shape
  text = np.ones((n, L), dtype=np.int32)
  lens = rng.integers(min(4, L - 1), L, size=n)
  for i in range(n):
    text[i, :lens[i]] = rng.integers(2, vocab, size=lens[i])
  return image, text


def header_functions(path):
  """Every `bv_name(` of a C header outside its comments: the functions it declares."""
  src = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
  return set(re.findall(r"\b(bv_[a-z0-9_]+)\s*\(", src))
