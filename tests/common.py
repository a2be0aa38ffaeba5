"""Shared tiny configurations for the tests (kept small so the CPU oracle runs in seconds), the parse of
the C ABI headers, and C programs built against them."""
import glob
import os
import re
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# every header of the C ABI of libbv_b200.so (the headers big_vision_b200.build hashes)
HEADERS = sorted(glob.glob(os.path.join(ROOT, "include", "bv_*.h")))

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


def run_c(tmp_path, source, cxx=False, link=False):
  """Writes `source` as a C99 (or, with cxx, C++17) program, compiles it with -Wall -Werror against include/
  (and, with link, libbv_b200.so), runs it and returns its stdout.  Skips the test without the compiler."""
  import pytest   # smoke() imports this module and must not need pytest
  cc = "g++" if cxx else "gcc"
  if shutil.which(cc) is None:
    pytest.skip(f"no {cc}")
  src, exe = tmp_path / ("main.cc" if cxx else "main.c"), tmp_path / "main"
  src.write_text(source)
  cmd = [cc, "-std=c++17" if cxx else "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
         str(src), "-o", str(exe)]
  if link:
    from big_vision_b200 import lib
    lib.load()
    libdir = os.path.dirname(os.path.abspath(lib.LIB_PATH))
    cmd += ["-L", libdir, "-lbv_b200", f"-Wl,-rpath,{libdir}"]
  subprocess.run(cmd, check=True)
  return subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
