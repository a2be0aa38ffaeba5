"""Builds big_vision_b200/libbv_b200.so in-tree with nvcc for sm_90a (H100).

nvcc cross-compiles without a GPU, so this also runs on a machine without one.
The .so and the object directory are build products (git-ignored).
"""
import glob
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libbv_b200.so")
SOURCES = ["host_utils.cu", "gemm.cu", "attention.cu", "layernorm.cu", "elementwise.cu",
           "loss.cu", "optim.cu", "eval.cu", "sam.cu", "distill.cu", "flexi.cu", "jet.cu", "dropout.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _digest(paths):
  h = hashlib.sha256()
  for p in sorted(paths):
    with open(p, "rb") as f:
      h.update(f.read())
  h.update(" ".join(FLAGS).encode())
  return h.hexdigest()


def _headers():
  out = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
  return out + glob.glob(os.path.join(os.path.dirname(HERE), "include", "bv_*.h"))


def _compile(src):
  obj = os.path.join(BUILD, src.replace(".cu", ".o"))
  stamp = obj + ".sha"
  dig = _digest([os.path.join(CSRC, src)] + _headers())
  if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
    return obj, False
  cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
  r = subprocess.run(cmd, capture_output=True, text=True)
  if r.returncode != 0:
    raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
  with open(stamp, "w") as f:
    f.write(dig)
  return obj, True


def build(force=False, verbose=True):
  os.makedirs(BUILD, exist_ok=True)
  if force:
    for f in os.listdir(BUILD):
      os.remove(os.path.join(BUILD, f))
  with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
    results = list(ex.map(_compile, SOURCES))
  objs = [o for o, _ in results]
  changed = any(c for _, c in results)
  if changed or not os.path.exists(LIB):
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
      raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    if verbose:
      print(f"[build] linked {LIB}")
  elif verbose:
    print(f"[build] up to date: {LIB}")
  return LIB


def build_variant(defines, suffix):
  """An experimental build of the same sources with extra -D flags into libbv_b200_<suffix>.so (own
  object directory); selected at run time with BV_LIB_PATH.  Not part of build()."""
  bdir = os.path.join(HERE, "build_" + suffix)
  os.makedirs(bdir, exist_ok=True)
  objs = []

  def one(src):
    obj = os.path.join(bdir, src.replace(".cu", ".o"))
    cmd = [NVCC] + FLAGS + [f"-D{d}" for d in defines] + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
      raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    return obj

  with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
    objs = list(ex.map(one, SOURCES))
  lib = os.path.join(HERE, f"libbv_b200_{suffix}.so")
  r = subprocess.run([NVCC, "-shared", "-o", lib] + objs + ["-lcudart"], capture_output=True, text=True)
  if r.returncode != 0:
    raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
  print(f"[build] linked {lib}")
  return lib


if __name__ == "__main__":
  if "--variant" in sys.argv:      # python -m big_vision_b200.build --variant BV_MBAR_SUSPEND_NS=20000 hint
    i = sys.argv.index("--variant")
    build_variant(sys.argv[i + 1].split(","), sys.argv[i + 2])
  else:
    build(force="--force" in sys.argv)
