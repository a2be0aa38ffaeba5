"""LABELLED STAND-IN: the Jet training step of configs/proj/jet/imagenet64.py (big_vision/models/proj/jet/jet.py,
trainers/proj/jet/train.py) in plain PyTorch, the library-kernel implementation a practitioner would write on
this box: bf16 autocast, cuBLAS GEMMs, `scaled_dot_product_attention`, torch.utils.checkpoint per coupling
(the reference's nn.remat(nothing_saveable)), gradient clipping and fused AdamW.  It is NOT the reference, and
none of this repository's kernels or models are on its path; tools/bench_jet.py times it beside the product
step on the same shapes.  The couplings' permutations are index gathers and scatters (the masks are
permutation matrices); the flow state stays fp32 as in the product.

  python -m baseline.torch_jet --batch 128 --steps 4 --warmup 2      # prints one JSON line
"""
import argparse
import json
import math
import time

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.utils.checkpoint import checkpoint

from baseline.torch_gpu import Block


class Coupling(nn.Module):
  """One affine coupling: x1 -> DNN -> (bias, raw scale); x2 -> (x2 + bias) * sigmoid(raw) * 2."""

  def __init__(self, T, c, d, depth, heads):
    super().__init__()
    self.T, self.c = T, c
    self.init_proj = nn.Linear(c, d)
    self.posemb = nn.Parameter(torch.randn(1, T, d) / math.sqrt(d))
    self.blocks = nn.ModuleList([Block(d, 4 * d, heads) for _ in range(depth)])
    self.norm = nn.LayerNorm(d, eps=1e-6)
    self.final_proj = nn.Linear(d, 2 * c)
    nn.init.zeros_(self.final_proj.weight)
    nn.init.zeros_(self.final_proj.bias)

  def forward(self, x, idx):
    n = x.shape[0]
    half = idx.shape[0] // 2
    x1 = x[:, idx[:half]].view(n, self.T, self.c)
    x2 = x[:, idx[half:]]
    with torch.autocast("cuda", dtype=torch.bfloat16):
      h = self.init_proj(x1) + self.posemb
      for b in self.blocks:
        h = b(h)
      out = self.final_proj(self.norm(h))
    bias, raw = out.float().view(n, self.T, 2 * self.c).chunk(2, dim=-1)
    y2 = (x2 + bias.reshape(n, -1)) * (torch.sigmoid(raw) * 2).reshape(n, -1)
    logdet = (F.logsigmoid(raw) + math.log(2)).sum(dim=(1, 2))
    return x.scatter(1, idx[half:].expand(n, -1), y2), logdet


class Jet(nn.Module):
  def __init__(self, tables, T, c, d, block_depth, heads, ps):
    super().__init__()
    self.ps = ps
    self.register_buffer("idx", torch.as_tensor(tables, dtype=torch.int64))
    self.couplings = nn.ModuleList([Coupling(T, c, d, block_depth, heads) for _ in range(len(tables))])

  def forward(self, image):
    n, H, W, C = image.shape
    p = self.ps
    x = image.view(n, H // p, p, W // p, p, C).permute(0, 1, 3, 2, 4, 5).reshape(n, -1)
    logdet = torch.zeros(n, device=image.device)
    for i, cp in enumerate(self.couplings):
      x, ld = checkpoint(cp, x, self.idx[i], use_reentrant=False)
      logdet = logdet + ld
    return x, logdet


def bits_loss(z, logdet):
  D = z.shape[1]
  nll = (0.5 * z * z).sum(1) + D * (0.5 * math.log(2 * math.pi) + math.log(127.5))
  return ((nll - logdet) / (D * math.log(2))).mean()


def make_step(model, lr=3e-4, wd=1e-5, clip=1.0):
  opt = torch.optim.AdamW(model.parameters(), lr=lr, betas=(0.9, 0.95), weight_decay=wd / lr, fused=True)

  def step(image):
    noisy = image + torch.rand_like(image) / 127.5
    z, logdet = model(noisy)
    loss = bits_loss(z, logdet)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    torch.nn.utils.clip_grad_norm_(model.parameters(), clip)
    opt.step()
    return loss

  return step


def random_tables(depth, T, dt, seed=0):
  """Gather tables of `depth` couplings: channel permutations of the dt values of each token, except every
  fifth coupling, which permutes the tokens (the imagenet64 interleave)."""
  rng = np.random.default_rng(seed)
  out = []
  for i in range(depth):
    if i % 5 == 4:
      q = rng.permutation(T)
      out.append((q[:, None] * dt + np.arange(dt)[None]).reshape(-1))
    else:
      p = rng.permutation(dt)
      t = np.arange(T)[:, None] * dt
      out.append(np.concatenate([(t + p[None, :dt // 2]).reshape(-1), (t + p[None, dt // 2:]).reshape(-1)]))
  return np.stack(out)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, default=128)
  ap.add_argument("--steps", type=int, default=4)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--depth", type=int, default=32)
  ap.add_argument("--block-depth", type=int, default=2)
  args = ap.parse_args()
  torch.manual_seed(0)
  res, ps, C, d, heads = 64, 4, 3, 512, 8
  T, dt = (res // ps) ** 2, ps * ps * C
  model = Jet(random_tables(args.depth, T, dt), T, dt // 2, d, args.block_depth, heads, ps).cuda()
  step = make_step(model)
  image = torch.rand(args.batch, res, res, C, device="cuda") * 2 - 1
  for _ in range(args.warmup):
    step(image)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    loss = step(image)
  torch.cuda.synchronize()
  ms = (time.perf_counter() - t0) * 1e3 / args.steps
  print(json.dumps({"impl": "torch_jet", "label": "STAND-IN, not the reference: PyTorch eager, bf16 autocast, "
                    "cuBLAS + SDPA, checkpoint per coupling, fused AdamW", "per_gpu_batch": args.batch,
                    "ms_per_step": round(ms, 2), "img_per_s": round(args.batch / ms * 1e3, 1),
                    "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2),
                    "loss": float(loss)}), flush=True)


if __name__ == "__main__":
  main()
