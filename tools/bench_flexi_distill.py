"""FlexiViT distillation step of configs/proj/flexivit/i21k_distill.py (trainers/proj/flexi/distill): a
FlexiViT-B student (240 px, base patch 8, 7x7 position-embedding grid, tok pool, scan=True) under a frozen
ViT-B/8 teacher at 224 px (785 tokens with [cls], tok pool), 21,843 classes, `kl` at t = 1, mixup p 1,
init_head_bias -10, Adam with bf16 mu and grad_clip_norm 1, at 512 images per GPU (the config's 4096 over 8
GPUs).

Measures, in one run, after every shape has run once, with a device synchronise around every timed window:
  - per seqhw of the config: img/s, ms per step and peak memory of the distillation step; and the config's
    expected step time, the p-weighted mean over seqhw;
  - the teacher's apply() alone, and the plain trainers/proj/flexi step of the same student (sigmoid_xent,
    same optimizer and mixup) at each seqhw, so that the distillation overhead (step - plain - teacher)
    shows;
  - with --profile-seqhw S: one torch.profiler window of two distillation steps at seqhw S, in a pass of its
    own after the timings, listing every device kernel that is not one of this library's (`bv::`) and
    every copy or memset; with --trace-dir the chrome trace is written there.

  python tools/bench_flexi_distill.py [--steps 4] [--warmup 2] [--per-gpu-batch 512] [--profile-seqhw 15]

Prints one JSON line, with the card's name and power limit read in the same run.  There is no CPU path.
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RES, TEACHER_RES, CLASSES = 240, 224, 21843
SEQHW = (5, 6, 8, 10, 12, 15, 16, 20, 24, 30)
P_SEQHW = (1,) * len(SEQHW)
STUDENT = dict(variant="B", pool_type="tok", posemb="learn", patch_size=(8, 8), posemb_size=(7, 7), scan=True)
TEACHER = dict(variant="B/8", pool_type="tok", rep_size=False)
OPT = dict(optax_name="scale_by_adam", optax=dict(mu_dtype="bfloat16"), grad_clip_norm=1.0, lr=1e-4, wd=1e-5,
           schedule=dict(warmup_steps=5000, decay_type="cosine"), mixup=dict(p=1.0),
           flexi=dict(seqhw=dict(v=SEQHW, p=P_SEQHW)))
DISTILL = dict(OPT, teachers=["prof"], distance="kl", distance_kw=dict(t=1.0), init_head_bias=-10.0)
PLAIN = dict(OPT, loss="sigmoid_xent")


def gpu_info():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return {"name": name, "power_limit": power}
  except Exception as e:   # pylint: disable=broad-except
    return {"unavailable": f"{type(e).__name__}: {e}"[:200]}


def time_ms(fn, steps, warmup):
  """(ms per call, peak GiB) of `steps` calls after `warmup`, host clock around a synchronised window."""
  import torch
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.perf_counter()
  for _ in range(steps):
    fn()
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) * 1e3 / steps, torch.cuda.max_memory_allocated() / 2**30


def profile_step(fn, trace_dir):
  """Device activity of two calls of `fn` under torch.profiler: {"bv_kernels": launches, "other_kernels":
  {name: launches}, "copies_and_memsets": {name: launches}}."""
  import torch
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    for _ in range(2):
      fn()
    torch.cuda.synchronize()
  ours, other, copies = 0, collections.Counter(), collections.Counter()
  for e in prof.events():
    if e.device_type != torch.autograd.DeviceType.CUDA:
      continue
    if "bv::" in e.name:
      ours += 1
    elif e.name.startswith(("Memcpy", "Memset")):
      copies[e.name] += 1
    else:
      other[e.name[:160]] += 1
  if trace_dir:
    os.makedirs(trace_dir, exist_ok=True)
    prof.export_chrome_trace(os.path.join(trace_dir, "flexi_distill_step.pt.trace.json"))
  return {"steps": 2, "bv_kernels": ours, "other_kernels": dict(other), "copies_and_memsets": dict(copies)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=4)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--per-gpu-batch", type=int, default=512)
  ap.add_argument("--profile-seqhw", type=int, default=None)
  ap.add_argument("--trace-dir", default=None)
  args = ap.parse_args()
  import torch
  from big_vision_b200 import lib as L
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.models import vit
  from big_vision_b200.models.proj.flexi import vit as fv
  from big_vision_b200.trainers.proj.flexi import distill as fd
  from big_vision_b200.trainers.proj.flexi import train as ft
  if L.load().bv_device_supported() != 1:
    raise RuntimeError("bench_flexi_distill needs a compute-capability 9.x GPU")
  info = gpu_info()
  n = args.per_gpu_batch
  g = torch.Generator(device="cuda").manual_seed(0)
  batch = {"image": torch.rand((n, RES, RES, 3), device="cuda", generator=g) * 2 - 1,
           "prof": torch.rand((n, TEACHER_RES, TEACHER_RES, 3), device="cuda", generator=g) * 2 - 1,
           "labels": torch.nn.functional.one_hot(torch.randint(0, CLASSES, (n,), device="cuda", generator=g),
                                                 CLASSES).float()}
  sched_kw = dict(total_steps=100_000, batch_size=n, data_size=10_000_000)
  rng = np.random.default_rng(0)
  line = {"metric": "flexivit_b_i21k_distill", "unit": "img/s", "per_gpu_batch": n, "res": RES,
          "teacher_res": TEACHER_RES, "classes": CLASSES, "student": STUDENT, "teacher": TEACHER, "gpu": info,
          "config": {"distance": "kl, t=1", "mixup_p": 1.0, "optimizer": "scale_by_adam, mu bf16, grad_clip_norm 1",
                     "init_head_bias": -10.0, "steps": args.steps, "warmup": args.warmup}}

  student, teacher = fv.Model(CLASSES, **STUDENT), vit.Model(CLASSES, **TEACHER)
  Pt = teacher.init(1, (n, TEACHER_RES, TEACHER_RES, 3)).drop_grad()
  Pt.tree("f")["head/kernel"].normal_(0.0, 0.02, generator=g)    # a zero head would make every logit 0
  Pt.sync_half()

  def fresh_student():
    P = student.init(0, (n, RES, RES, 3))
    P.tree("f")["head/bias"].fill_(DISTILL["init_head_bias"])
    P.sync_half()
    return P

  # ---- the distillation step
  P = fresh_student()
  tx, _ = bv_optax.make(DISTILL, P, sched_kw=sched_kw)
  state = {"params": {"student": P, "prof": Pt}, "opt": tx.init(P)}
  fn = fd.make_update_fn({"student": student, "prof": teacher}, tx, DISTILL)
  for s in SEQHW:                                # every shape once before any timing
    fn(state, rng, batch, seqhw=s)
  per = {}
  for s in SEQHW:
    ms, mem = time_ms(lambda s=s: fn(state, rng, batch, seqhw=s), args.steps, args.warmup)
    per[str(s)] = {"patch": RES // s, "tokens": s * s + 1, "ms_per_step": round(ms, 2),
                   "img_per_s": round(n / ms * 1e3, 1), "peak_mem_gib": round(mem, 2)}
  _, m = fn(state, rng, batch, seqhw=SEQHW[-1])
  line["last_step"] = {k: float(v) for k, v in m.items()}
  w = np.array(P_SEQHW, dtype=np.float64) / sum(P_SEQHW)
  expected = float(sum(wi * per[str(s)]["ms_per_step"] for wi, s in zip(w, SEQHW)))
  line["per_seqhw"] = per
  line["expected_ms_per_step"] = round(expected, 2)
  line["value"] = round(n / expected * 1e3, 1)
  if args.profile_seqhw:
    line["profile"] = dict(seqhw=args.profile_seqhw, **profile_step(
        lambda: fn(state, rng, batch, seqhw=args.profile_seqhw), args.trace_dir))
  del state, fn, tx, P
  torch.cuda.empty_cache()

  # ---- the teacher's forward alone, and the plain flexi step of the same student
  ms_t, mem_t = time_ms(lambda: teacher.apply({"params": Pt}, batch["prof"]), args.steps, args.warmup)
  line["teacher_apply"] = {"ms": round(ms_t, 2), "img_per_s": round(n / ms_t * 1e3, 1), "peak_mem_gib": round(mem_t, 2)}
  P = fresh_student()
  tx, _ = bv_optax.make(PLAIN, P, sched_kw=sched_kw)
  state = {"params": P, "opt": tx.init(P)}
  fn = ft.make_update_fn(student, tx, PLAIN)
  for s in SEQHW:
    fn(state, rng, batch, seqhw=s)
  plain = {}
  for s in SEQHW:
    ms, mem = time_ms(lambda s=s: fn(state, rng, batch, seqhw=s), args.steps, args.warmup)
    plain[str(s)] = {"ms_per_step": round(ms, 2), "peak_mem_gib": round(mem, 2),
                     "distill_minus_plain_minus_teacher_ms": round(per[str(s)]["ms_per_step"] - ms - ms_t, 2)}
  line["plain_flexi_step"] = plain
  line["plain_expected_ms_per_step"] = round(float(sum(wi * plain[str(s)]["ms_per_step"] for wi, s in zip(w, SEQHW))), 2)
  del state, fn, tx, P
  torch.cuda.empty_cache()
  print(json.dumps(line), flush=True)


if __name__ == "__main__":
  main()
