"""Times every GEMM of one SigLIP B/16 training step (bench.py's headline workload, 768 pairs per GPU)
in isolation, with its real operand layouts and epilogue, and prints per shape the time, the achieved
TFLOP/s and the two lower bounds on the time: FLOPs at the H100 SXM's dense BF16 rate and the
algorithmic HBM bytes (operands read once, outputs written once) at its HBM3 bandwidth.

  python tools/gemm_shapes.py                    # table (CUDA events)
  python tools/gemm_shapes.py --dump DIR         # also write every output of one call per shape as .npy
  python tools/gemm_shapes.py --pairs 256        # a smaller batch
  python tools/gemm_shapes.py --block-n 128      # every GEMM at 128-column tiles

bf16 outputs are dumped as their uint16 bit patterns, fp32 outputs as float32, so two builds
(BV_LIB_PATH) can be compared bit for bit.  Inputs come from a seeded generator on the device.
"""
import argparse
import functools
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from big_vision_b200 import lib as L  # noqa: E402
from big_vision_b200 import ops  # noqa: E402

PEAK_TFLOPS = 989.0      # H100 SXM data sheet, dense BF16 (700 W)
PEAK_TBS = 3.35          # H100 SXM data sheet, HBM3

D, MLP, PATCH = 768, 3072, 16 * 16 * 3
IMG_TOKENS, TXT_TOKENS = 196, 64


def timeit(fn, reps):
  for _ in range(2):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / reps


class Bufs:
  """Seeded device tensors, created on first use and reused across cases of the same shape."""

  def __init__(self, seed):
    self.g = torch.Generator(device="cuda")
    self.g.manual_seed(seed)
    self.cache = {}

  def get(self, name, shape, scale=1.0, dtype=torch.bfloat16):
    key = (name, tuple(shape), dtype)
    if key not in self.cache:
      t = torch.randn(*shape, device="cuda", generator=self.g, dtype=torch.float32) * scale
      self.cache[key] = t.to(dtype)
    return self.cache[key]


def cases(pairs, bufs, block_n=0):
  """(name, M, N, K, out tensors, fn, algorithmic bytes) for every GEMM of the step.  Output tensors
  are allocated by the caller-visible closures so that a dump sees exactly what one call wrote."""
  out = []
  gemm = functools.partial(ops.gemm, block_n=block_n)

  def add(name, M, N, K, make, nbytes):
    out.append((name, M, N, K, make, nbytes))

  for tower, M in (("img", pairs * IMG_TOKENS), ("txt", pairs * TXT_TOKENS)):
    x = bufs.get(f"{tower}.x", (M, D))
    h = bufs.get(f"{tower}.h", (M, MLP))
    wq = bufs.get("wqkv", (D, 3 * D), 0.03)
    wo = bufs.get("wo", (D, D), 0.03)
    w0 = bufs.get("w0", (D, MLP), 0.03)
    w1 = bufs.get("w1", (MLP, D), 0.03)
    b3 = bufs.get("b2304", (3 * D,), 1.0, torch.float32)
    bd = bufs.get("b768", (D,), 1.0, torch.float32)
    bm = bufs.get("b3072", (MLP,), 1.0, torch.float32)
    dq = bufs.get(f"{tower}.dqkv", (M, 3 * D))
    bf = 2

    def fwd_qkv(x=x, wq=wq, b3=b3, M=M):
      o = torch.empty(M, 3 * D, device="cuda", dtype=torch.bfloat16)
      return [o], lambda: gemm(x, wq, b_mn=True, bias=b3, out=o)
    add(f"{tower} fwd qkv       bias", M, 3 * D, D, fwd_qkv, bf * (M * D + D * 3 * D + M * 3 * D))

    def fwd_out(x=x, wo=wo, bd=bd, M=M):
      o = torch.empty(M, D, device="cuda", dtype=torch.bfloat16)
      return [o], lambda: gemm(x, wo, b_mn=True, bias=bd, aux=x, out=o, epilogue=L.EPI_BIAS_RESID)
    add(f"{tower} fwd out_proj  +resid", M, D, D, fwd_out, bf * (M * D + D * D + M * D + M * D))

    def fwd_d0(x=x, w0=w0, bm=bm, M=M):
      o = torch.empty(M, MLP, device="cuda", dtype=torch.bfloat16)
      o2 = torch.empty(M, MLP, device="cuda", dtype=torch.bfloat16)
      return [o, o2], lambda: gemm(x, w0, b_mn=True, bias=bm, out=o, out2=o2, epilogue=L.EPI_BIAS_GELU)
    add(f"{tower} fwd Dense_0   gelu", M, MLP, D, fwd_d0, bf * (M * D + D * MLP + 2 * M * MLP))

    def fwd_d1(h=h, w1=w1, bd=bd, x=x, M=M):
      o = torch.empty(M, D, device="cuda", dtype=torch.bfloat16)
      return [o], lambda: gemm(h, w1, b_mn=True, bias=bd, aux=x, out=o, epilogue=L.EPI_BIAS_RESID)
    add(f"{tower} fwd Dense_1   +resid", M, D, MLP, fwd_d1, bf * (M * MLP + MLP * D + 2 * M * D))

    def wg_d1(h=h, x=x):
      o = torch.zeros(MLP, D, device="cuda", dtype=torch.float32)
      return [o], lambda: gemm(h, x, a_mn=True, b_mn=True, out=o, reduce_out=True)
    add(f"{tower} wgrad Dense_1 f32+=", MLP, D, M, wg_d1, bf * (M * MLP + M * D) + 4 * 2 * MLP * D)

    def dg_d1(x=x, w1=w1, h=h, M=M):
      o = torch.empty(M, MLP, device="cuda", dtype=torch.bfloat16)
      cs = torch.zeros(MLP, device="cuda", dtype=torch.float32)
      return [o, cs], lambda: gemm(x, w1, aux=h, out=o, epilogue=L.EPI_DGELU, colsum=cs)
    add(f"{tower} dgrad Dense_1 gelu'+colsum", M, MLP, D, dg_d1, bf * (M * D + MLP * D + 2 * M * MLP))

    def wg_d0(x=x, h=h):
      o = torch.zeros(D, MLP, device="cuda", dtype=torch.float32)
      return [o], lambda: gemm(x, h, a_mn=True, b_mn=True, out=o, reduce_out=True)
    add(f"{tower} wgrad Dense_0 f32+=", D, MLP, M, wg_d0, bf * (M * D + M * MLP) + 4 * 2 * MLP * D)

    def dg_d0(h=h, w0=w0, M=M):
      o = torch.empty(M, D, device="cuda", dtype=torch.bfloat16)
      return [o], lambda: gemm(h, w0, out=o)
    add(f"{tower} dgrad Dense_0", M, D, MLP, dg_d0, bf * (M * MLP + MLP * D + M * D))

    def wg_out(x=x):
      o = torch.zeros(D, D, device="cuda", dtype=torch.float32)
      return [o], lambda: gemm(x, x, a_mn=True, b_mn=True, out=o, reduce_out=True)
    add(f"{tower} wgrad out_proj f32+=", D, D, M, wg_out, bf * 2 * M * D + 4 * 2 * D * D)

    def dg_out(x=x, wo=wo, M=M):
      o = torch.empty(M, D, device="cuda", dtype=torch.bfloat16)
      return [o], lambda: gemm(x, wo, out=o)
    add(f"{tower} dgrad out_proj", M, D, D, dg_out, bf * (2 * M * D + D * D))

    def wg_qkv(x=x, dq=dq):
      o = torch.zeros(D, 3 * D, device="cuda", dtype=torch.float32)
      return [o], lambda: gemm(x, dq, a_mn=True, b_mn=True, out=o, reduce_out=True)
    add(f"{tower} wgrad qkv     f32+=", D, 3 * D, M, wg_qkv, bf * (M * D + M * 3 * D) + 4 * 2 * 3 * D * D)

    def dg_qkv(dq=dq, wq=wq, M=M):
      o = torch.empty(M, D, device="cuda", dtype=torch.bfloat16)
      return [o], lambda: gemm(dq, wq, out=o)
    add(f"{tower} dgrad qkv", M, D, 3 * D, dg_qkv, bf * (M * 3 * D + 3 * D * D + M * D))

  # image tower only: the patch embedding (position embedding added row-modulo) and the MAP head's
  # key/value projection over every token
  M = pairs * IMG_TOKENS
  pt = bufs.get("patches", (M, PATCH))
  we = bufs.get("wemb", (PATCH, D), 0.03)
  pos = bufs.get("posemb", (IMG_TOKENS, D))
  bd = bufs.get("b768", (D,), 1.0, torch.float32)
  x = bufs.get("img.x", (M, D))
  wkv = bufs.get("wkv", (D, 2 * D), 0.03)
  bkv = bufs.get("b1536", (2 * D,), 1.0, torch.float32)
  dkv = bufs.get("dkv", (M, 2 * D))

  def emb():
    o = torch.empty(M, D, device="cuda", dtype=torch.bfloat16)
    return [o], lambda: gemm(pt, we, b_mn=True, bias=bd, aux=pos, aux_row_mod=IMG_TOKENS, out=o,
                                 epilogue=L.EPI_BIAS_RESID)
  add("img fwd patch emb  +posemb", M, D, PATCH, emb, 2 * (M * PATCH + PATCH * D + M * D))

  def wg_emb():
    o = torch.zeros(PATCH, D, device="cuda", dtype=torch.float32)
    return [o], lambda: gemm(pt, x, a_mn=True, b_mn=True, out=o, reduce_out=True)
  add("img wgrad patch emb f32+=", PATCH, D, M, wg_emb, 2 * (M * PATCH + M * D) + 8 * PATCH * D)

  def kv():
    o = torch.empty(M, 2 * D, device="cuda", dtype=torch.bfloat16)
    return [o], lambda: gemm(x, wkv, b_mn=True, bias=bkv, out=o)
  add("img fwd MAP kv     bias", M, 2 * D, D, kv, 2 * (M * D + 2 * D * D + 2 * M * D))

  def wg_kv():
    o = torch.zeros(D, 2 * D, device="cuda", dtype=torch.float32)
    return [o], lambda: gemm(x, dkv, a_mn=True, b_mn=True, out=o, reduce_out=True)
  add("img wgrad MAP kv   f32+=", D, 2 * D, M, wg_kv, 2 * (M * D + 2 * M * D) + 8 * 2 * D * D)

  def dg_kv():
    o = torch.empty(M, D, device="cuda", dtype=torch.bfloat16)
    return [o], lambda: gemm(dkv, wkv, out=o)
  add("img dgrad MAP kv", M, D, 2 * D, dg_kv, 2 * (2 * M * D + 2 * D * D + M * D))

  # appended (earlier cases keep their --dump indices): gelu' without the bias-gradient colsum, so the
  # table separates the colsum's atomics from the rest of that GEMM
  x, w1, h = bufs.get("img.x", (M, D)), bufs.get("w1", (MLP, D), 0.03), bufs.get("img.h", (M, MLP))

  def dg_d1_nocs():
    o = torch.empty(M, MLP, device="cuda", dtype=torch.bfloat16)
    return [o], lambda: gemm(x, w1, aux=h, out=o, epilogue=L.EPI_DGELU)
  add("img dgrad Dense_1 gelu'", M, MLP, D, dg_d1_nocs, 2 * (M * D + MLP * D + 2 * M * MLP))

  # appended: the forward-only Dense_0 (a frozen tower, apply()) writes the activation only, no
  # pre-activation; compare with the "fwd Dense_0 gelu" rows of the same tower
  w0, bm = bufs.get("w0", (D, MLP), 0.03), bufs.get("b3072", (MLP,), 1.0, torch.float32)
  for tower, Mt in (("img", pairs * IMG_TOKENS), ("txt", pairs * TXT_TOKENS)):
    xt = bufs.get(f"{tower}.x", (Mt, D))

    def fwd_d0_act(xt=xt, Mt=Mt):
      o = torch.empty(Mt, MLP, device="cuda", dtype=torch.bfloat16)
      return [o], lambda: gemm(xt, w0, b_mn=True, bias=bm, out=o, epilogue=L.EPI_BIAS_GELU_ACT)
    add(f"{tower} fwd Dense_0   gelu act only", Mt, MLP, D, fwd_d0_act, 2 * (Mt * D + D * MLP + Mt * MLP))
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--pairs", type=int, default=768, help="image-text pairs per step (bench.py: 768)")
  ap.add_argument("--reps", type=int, default=10)
  ap.add_argument("--dump", metavar="DIR", default=None)
  ap.add_argument("--block-n", type=int, default=0, choices=[0, 128, 256],
                  help="tile width of every GEMM (0: the library's choice)")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("gemm_shapes.py needs a GPU")
  L.load()
  bufs = Bufs(0)
  total_ms = total_flop = 0.0
  print(f"{'case':34s} {'M':>7s} {'N':>5s} {'K':>7s} {'us':>9s} {'TFLOP/s':>8s} {'flop-lb us':>10s} "
        f"{'byte-lb us':>10s}")
  for i, (name, M, N, K, make, nbytes) in enumerate(cases(args.pairs, bufs, args.block_n)):
    outs, fn = make()
    if args.dump:
      fn()
      torch.cuda.synchronize()
      os.makedirs(args.dump, exist_ok=True)
      for j, o in enumerate(outs):
        a = o.view(torch.int16).cpu().numpy().view(np.uint16) if o.dtype == torch.bfloat16 else o.cpu().numpy()
        np.save(os.path.join(args.dump, f"{i:02d}_{j}.npy"), a)
    ms = timeit(fn, args.reps)
    flop = 2.0 * M * N * K
    total_ms += ms
    total_flop += flop
    print(f"{name:34s} {M:7d} {N:5d} {K:7d} {ms * 1e3:9.1f} {flop / ms * 1e-9:8.1f} "
          f"{flop / (PEAK_TFLOPS * 1e12) * 1e6:10.1f} {nbytes / (PEAK_TBS * 1e12) * 1e6:10.1f}", flush=True)
    del outs, fn
  print(f"{'all (each shape once)':34s} {'':7s} {'':5s} {'':7s} {total_ms * 1e3:9.1f} "
        f"{total_flop / total_ms * 1e-9:8.1f}")
  print(f"device: {torch.cuda.get_device_name()}")


if __name__ == "__main__":
  main()
