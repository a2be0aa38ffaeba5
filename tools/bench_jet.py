"""Jet training step of configs/proj/jet/imagenet64.py: 64x64x3 images, patch 4 (256 tokens of 48 values),
32 couplings of 2 ViT blocks at width 512 with 8 heads, Adam with bf16 mu and b2 0.95, grad_clip_norm 1, masks
frozen.  The config's batch of 1024 is 128 images per GPU on 8 GPUs.

Measures, in one run:
  - img/s, ms per step and peak memory of trainers/proj/jet's step at 128 images per GPU and at --big-batch;
  - the forward GFLOP per image, from the shapes;
  - each kernel of include/bv_b200_jet.h alone at the step's shapes (128 images), CUDA events around 50
    launches, against its bytes at the H100 SXM data sheet's 3.35 TB/s, and the Jet kernels' share of the
    step (their times times their launches per step, over the step time);
  - in a process of its own, baseline/torch_jet.py, a labelled PyTorch stand-in of the same step.

  python tools/bench_jet.py [--steps 4] [--warmup 2] [--big-batch 512]

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

RES, C = 64, 3
HBM_BYTES_PER_S = 3.35e12
MODEL = dict(depth=32, block_depth=2, emb_dim=512, num_heads=8,
             kinds=("channels", "channels", "channels", "channels", "spatial"), channels_coupling_projs=("random",),
             spatial_coupling_projs=("checkerboard", "checkerboard-inv", "vstripes", "vstripes-inv", "hstripes",
                                     "hstripes-inv"))
CONFIG = dict(seed=0, optax_name="scale_by_adam", optax=dict(mu_dtype="bfloat16", b2=0.95), grad_clip_norm=1.0,
              lr=3e-4, wd=1e-5, wd_mults=((".*", 1.0),),
              schedule=[(".*FREEZE_ME.*", None), (".*", dict(decay_type="cosine", warmup_percent=0.1))])


def gpu_info():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return {"name": name, "power_limit": power}
  except Exception as e:   # pylint: disable=broad-except
    return {"unavailable": f"{type(e).__name__}: {e}"[:200]}


def forward_flop_per_image(m=MODEL, res=RES, ps=4, in_ch=C):
  """Multiply-adds x 2 of one forward: per coupling and token, init_proj, the blocks (q/k/v/out, the MLP, and
  QK^T and PV over T keys) and final_proj."""
  d, T, c = m["emb_dim"], (res // ps) ** 2, ps * ps * in_ch // 2
  block = 2 * (4 * d * d + 2 * d * 4 * d + 2 * T * d)
  return m["depth"] * T * (2 * c * d + m["block_depth"] * block + 2 * d * 2 * c)


def make_step(model, n):
  import torch
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.trainers.proj.jet import train as jt
  P = model.init(0, (n, RES, RES, C), device="cuda")
  tx, _ = bv_optax.make(CONFIG, P, sched_kw=dict(total_steps=100_000, batch_size=n, data_size=1_281_167))
  state = {"params": P, "opt": tx.init(P)}
  rng = np.random.default_rng(0)
  image = torch.from_numpy(rng.random((n, RES, RES, C), dtype=np.float32) * 2 - 1).cuda()
  return state, jt.make_update_fn(model, tx, CONFIG), {"image": image}


def time_steps(state, fn, batch, steps, warmup):
  """(ms per step, peak GiB, last loss) of `steps` steps after `warmup`, host clock around a synchronised window."""
  import torch
  for _ in range(warmup):
    state, _ = fn(state, None, batch)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.perf_counter()
  for _ in range(steps):
    state, m = fn(state, None, batch)
  torch.cuda.synchronize()
  ms = (time.perf_counter() - t0) * 1e3 / steps
  assert np.isfinite(float(m["training_loss"]))
  return ms, torch.cuda.max_memory_allocated() / 2**30, float(m["training_loss"])


def time_kernels(model, P, n, iters=50):
  """Each Jet kernel at the step's shapes: {name: {us, bytes, hbm_floor_us, share_of_3.35TBps, per_step}}."""
  import torch
  from big_vision_b200 import ops
  T, c, depth = model.T, model.c, model.depth
  D = 2 * T * c
  g = torch.Generator(device="cuda").manual_seed(0)
  image = torch.rand(n, RES, RES, C, device="cuda", generator=g) * 2 - 1
  x = torch.randn(n, T, 2 * c, device="cuda", generator=g)
  y = torch.empty_like(x)
  br = torch.randn(n * T, 2 * c, device="cuda", generator=g)
  dy = torch.randn(n, T, 2 * c, device="cuda", generator=g)
  dx1 = torch.randn(n * T, c, device="cuda", generator=g)
  dbr = torch.empty(n * T, 2 * c, dtype=torch.bfloat16, device="cuda")
  x1 = torch.empty(n * T, c, dtype=torch.bfloat16, device="cuda")
  logdet = torch.zeros(n, device="cuda")
  idx = P.jet_tables[0]
  N, half = n * D, n * D // 2
  cases = [
      ("dequantize_patchify", lambda: ops.jet_dequantize_patchify(image, model.ps, 0, 1, 0, out=y), 8 * N, 1),
      ("unpatchify", lambda: ops.jet_unpatchify(x, image.shape, model.ps, out=image), 8 * N, 0),
      ("split", lambda: ops.jet_split(x, idx, T, c, out=x1), 6 * half + 4 * D // 2, 2 * depth),
      ("coupling_fwd", lambda: ops.jet_coupling_fwd(x, idx, br, logdet, T, c, out=y), 16 * half + 4 * N + 4 * D,
       depth),
      ("coupling_bwd", lambda: ops.jet_coupling_bwd(dy, x, idx, br, -1e-6, T, c, dx=y, dbr=dbr),
       12 * half + 6 * N + 2 * D, depth),
      ("merge_grad", lambda: ops.jet_merge_grad(dy, dx1, idx, T, c, dx=y), 12 * half + 2 * D, depth),
      ("bits", lambda: ops.jet_bits(x, logdet, 1e-6, dz=y), 8 * N, 1),
  ]
  out = {}
  for name, call, nbytes, per_step in cases:
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
    out[name] = {"us": round(us, 2), "bytes": nbytes, "hbm_floor_us": round(floor, 2),
                 "share_of_3.35TBps": round(floor / us, 3), "launches_per_step": per_step}
  return out


def stand_in(n, steps, warmup):
  """baseline/torch_jet.py in a process of its own -> its JSON line (or the failure)."""
  r = subprocess.run([sys.executable, "-m", "baseline.torch_jet", "--batch", str(n), "--steps", str(steps),
                      "--warmup", str(warmup)], cwd=ROOT, capture_output=True, text=True, timeout=3600)
  lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
  if r.returncode != 0 or not lines:
    return {"impl": "torch_jet", "unavailable": (r.stderr or r.stdout)[-400:]}
  return json.loads(lines[-1])


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=4)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--big-batch", type=int, default=512)
  args = ap.parse_args()
  import torch
  from big_vision_b200 import lib as L
  from big_vision_b200.models.proj.jet import jet
  if L.load().bv_device_supported() != 1:
    raise RuntimeError("bench_jet needs a compute-capability 9.x GPU")
  info = gpu_info()
  flop = forward_flop_per_image()
  line = {"metric": "jet_imagenet64", "unit": "img/s", "res": RES, "model": MODEL, "gpu": info,
          "forward_gflop_per_image": round(flop / 1e9, 2), "train_gflop_per_image": round(3 * flop / 1e9, 2),
          "executed_gflop_per_image": round(4 * flop / 1e9, 2)}
  model = jet.Model(**MODEL)
  per = {}
  for n in (128, args.big_batch):
    state, fn, batch = make_step(model, n)
    ms, mem, loss = time_steps(state, fn, batch, args.steps, args.warmup)
    per[str(n)] = {"ms_per_step": round(ms, 2), "img_per_s": round(n / ms * 1e3, 1), "peak_mem_gib": round(mem, 2),
                   "loss": round(loss, 4),
                   "executed_tflop_per_s": round(4 * flop * n / ms / 1e9, 1)}
    if n == 128:
      kernels = time_kernels(model, state["params"], n)
      jet_us = sum(k["us"] * k["launches_per_step"] for k in kernels.values())
      per[str(n)]["jet_kernels_ms"] = round(jet_us / 1e3, 3)
      per[str(n)]["jet_kernels_share_of_step"] = round(jet_us / 1e3 / ms, 4)
    del state, fn, batch
    torch.cuda.empty_cache()
  line["per_gpu_batch"] = per
  line["value"] = per["128"]["img_per_s"]
  line["kernels_at_128"] = kernels
  line["stand_in"] = {str(n): stand_in(n, args.steps, args.warmup) for n in (128, args.big_batch)}
  print(json.dumps(line), flush=True)


if __name__ == "__main__":
  main()
