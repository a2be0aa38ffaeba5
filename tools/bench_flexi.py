"""FlexiViT-B pre-training step of configs/proj/flexivit/i21k_sup.py: 240x240, base patch 8 and a 7x7
position-embedding grid, tok pool, 21,843 classes, sigmoid_xent, init_head_bias -10, Adam with bf16 mu,
grad_clip_norm 1, mixup p 0.2, at 512 images per GPU (the config's 4096 over 8 GPUs) with scan=True (each
encoder block recomputed in the backward; without it seqhw 30 does not fit in 80 GB).

Measures, in one run:
  - per seqhw of the config: img/s, ms per step and peak memory of trainers/proj/flexi's step, every shape
    warmed up first; and the config's expected step time, the p-weighted mean over seqhw;
  - the flexi overhead: plain vit.Model B/16 at 240 px (225 tokens, same head, optimizer and scan) against
    flexi at seqhw 15, which is also patch 16 and 225 tokens;
  - bv_resample_fwd / bv_resample_bwd alone at each shape the step uses, CUDA events around 50 launches,
    against their bytes at the H100 SXM data sheet's 3.35 TB/s.

  python tools/bench_flexi.py [--steps 4] [--warmup 2] [--per-gpu-batch 512]

Prints one JSON line, with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RES, CLASSES = 240, 21843
SEQHW = (5, 6, 8, 10, 12, 15, 16, 20, 24, 30)
P_SEQHW = (1,) * len(SEQHW)
HBM_BYTES_PER_S = 3.35e12
CONFIG = dict(optax_name="scale_by_adam", optax=dict(mu_dtype="bfloat16"), grad_clip_norm=1.0, lr=0.001, wd=0.0001,
              schedule=dict(warmup_steps=10_000, decay_type="cosine"), loss="sigmoid_xent", mixup=dict(p=0.2),
              flexi=dict(seqhw=dict(v=SEQHW, p=P_SEQHW)))
MODEL = dict(variant="B", pool_type="tok", posemb="learn", patch_size=(8, 8), posemb_size=(7, 7), scan=True)


def gpu_info():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return {"name": name, "power_limit": power}
  except Exception as e:   # pylint: disable=broad-except
    return {"unavailable": f"{type(e).__name__}: {e}"[:200]}


def make_step(model, n, update_fn_factory):
  import torch
  from big_vision_b200 import optax as bv_optax
  P = model.init(0, (n, RES, RES, 3), device="cuda")
  P.tree("f")["head/bias"].fill_(-10.0)                    # config.init_head_bias
  tx, _ = bv_optax.make(CONFIG, P, sched_kw=dict(total_steps=100_000, batch_size=n, data_size=10_000_000))
  state = {"params": P, "opt": tx.init(P)}
  rng = np.random.default_rng(0)
  image = torch.from_numpy(rng.random((n, RES, RES, 3), dtype=np.float32) * 2 - 1).cuda()
  labels = torch.zeros((n, CLASSES), device="cuda")
  labels[torch.arange(n), torch.from_numpy(rng.integers(0, CLASSES, n)).cuda()] = 1.0
  return state, update_fn_factory(model, tx, CONFIG), {"image": image, "labels": labels}, rng


def time_steps(state, fn, batch, rng, steps, warmup, **kw):
  """(ms per step, peak GiB) of `steps` steps after `warmup`, host clock around a synchronised window."""
  import torch
  for _ in range(warmup):
    state, _ = fn(state, rng, batch, **kw)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.perf_counter()
  for _ in range(steps):
    state, m = fn(state, rng, batch, **kw)
  torch.cuda.synchronize()
  ms = (time.perf_counter() - t0) * 1e3 / steps
  assert np.isfinite(float(m["training_loss"]))
  return ms, torch.cuda.max_memory_allocated() / 2**30


def time_kernels(d=768, C=3, iters=50):
  """bv_resample_fwd / _bwd at every shape of the step: {label: {...}}."""
  import torch
  from big_vision_b200 import ops
  from big_vision_b200.models.proj.flexi import vit as fv
  shapes = [(f"kernel p={RES // s}", fv.pi_resize_matrix(8, RES // s), C * d) for s in SEQHW if RES // s != 8]
  shapes += [(f"posemb seqhw={s}", fv.posemb_resize_matrix((7, 7), s), d) for s in SEQHW]
  out = {}
  g = torch.Generator(device="cuda").manual_seed(0)
  for label, M, J in shapes:
    M = torch.from_numpy(M.astype(np.float32)).cuda()
    R, K = M.shape
    x = torch.randn(K, J, device="cuda", generator=g)
    dy = torch.randn(R, J, device="cuda", generator=g)
    y = torch.empty(R, J, dtype=torch.bfloat16, device="cuda")
    dx = torch.zeros(K, J, device="cuda")
    row = {"R": R, "K": K, "J": J}
    for name, call, nbytes in (("fwd", lambda: ops.resample_fwd(M, x, out=y), 4 * R * K + 4 * K * J + 2 * R * J),
                               ("bwd", lambda: ops.resample_bwd(M, dy, dx), 4 * R * K + 4 * R * J + 8 * K * J)):
      for _ in range(5):
        call()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(iters):
        call()
      e1.record()
      torch.cuda.synchronize()
      us = e0.elapsed_time(e1) / iters * 1e3
      floor = nbytes / HBM_BYTES_PER_S * 1e6
      row[name] = {"us": round(us, 2), "bytes": nbytes, "hbm_floor_us": round(floor, 2),
                   "share_of_3.35TBps": round(floor / us, 3)}
    out[label] = row
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=4)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--per-gpu-batch", type=int, default=512)
  args = ap.parse_args()
  import torch
  from big_vision_b200 import train
  from big_vision_b200 import lib as L
  from big_vision_b200.models import vit
  from big_vision_b200.models.proj.flexi import vit as fv
  from big_vision_b200.trainers.proj.flexi import train as ft
  if L.load().bv_device_supported() != 1:
    raise RuntimeError("bench_flexi needs a compute-capability 9.x GPU")
  info = gpu_info()
  n = args.per_gpu_batch
  line = {"metric": "flexivit_b_i21k_sup", "unit": "img/s", "per_gpu_batch": n, "res": RES, "classes": CLASSES,
          "model": MODEL, "gpu": info}

  state, fn, batch, rng = make_step(fv.Model(CLASSES, **MODEL), n, ft.make_update_fn)
  for s in SEQHW:                                # every shape once before any timing
    state, _ = fn(state, rng, batch, seqhw=s)
  per = {}
  for s in SEQHW:
    ms, mem = time_steps(state, fn, batch, rng, args.steps, args.warmup, seqhw=s)
    per[str(s)] = {"patch": RES // s, "tokens": s * s + 1, "ms_per_step": round(ms, 2), "img_per_s": round(n / ms * 1e3, 1),
                   "peak_mem_gib": round(mem, 2)}
  w = np.array(P_SEQHW, dtype=np.float64) / sum(P_SEQHW)
  expected = float(sum(wi * per[str(s)]["ms_per_step"] for wi, s in zip(w, SEQHW)))
  line["per_seqhw"] = per
  line["expected_ms_per_step"] = round(expected, 2)
  line["value"] = round(n / expected * 1e3, 1)
  flexi15 = per["15"]["ms_per_step"]
  del state, fn, batch
  torch.cuda.empty_cache()

  plain_kw = dict(variant="B/16", pool_type="tok", posemb="learn", rep_size=False, scan=True)
  state, fn, batch, rng = make_step(vit.Model(CLASSES, **plain_kw), n, train.make_update_fn)
  ms, mem = time_steps(state, fn, batch, rng, args.steps, args.warmup)
  line["overhead"] = {"vit_b16_ms_per_step": round(ms, 2), "vit_b16_peak_mem_gib": round(mem, 2),
                      "flexi_seqhw15_ms_per_step": flexi15, "flexi_minus_vit_ms": round(flexi15 - ms, 2),
                      "ratio": round(flexi15 / ms, 4)}
  del state, fn, batch
  torch.cuda.empty_cache()
  line["kernels"] = time_kernels()
  print(json.dumps(line), flush=True)


if __name__ == "__main__":
  main()
