"""Distillation step (trainers/proj/distill): a ViT-S/16 student at 224 px under a frozen ViT-B/16 teacher at
384 px (577 tokens, pool_type "tok"), 1000 classes, 256 images per GPU, `kl` at t = 1, mixup p = 1, Adam with
bf16 mu and grad_clip_norm 1 (the optimizer of configs/proj/flexivit/i1k_deit3_distill.py).

In one run, after warm-up and with a device synchronise around every timed window:
  * the distill step: img/s, ms per step, peak device memory;
  * the plain train.py step of the student (softmax_xent, same optimizer and mixup) and the teacher's apply()
    alone, so that step ~ student step + teacher forward shows, and what the rest costs;
  * bv_distill_loss alone, CUDA events over `--kernel-iters` launches, at (256, 1000) and (1024, 21843), against
    its bytes over the H100 SXM data sheet's 3.35 TB/s (a data-sheet bound, not a measured one), with
    ops.softmax_xent at the same shapes for scale.

  python tools/bench_distill.py [--steps 8] [--warmup 3] [--per-gpu-batch 256] [--kernel-iters 50]

Prints one JSON line, with the card's name and power limit read in the same run.  There is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CLASSES = 1000
STUDENT = dict(variant="S/16", pool_type="tok", rep_size=False)
TEACHER = dict(variant="B/16", pool_type="tok", rep_size=False)
STUDENT_RES, TEACHER_RES = 224, 384
OPT_CONFIG = dict(optax_name="scale_by_adam", optax=dict(mu_dtype="bfloat16"), grad_clip_norm=1.0, lr=1e-3, wd=1e-4,
                  schedule=dict(warmup_steps=1_000, decay_type="cosine"), mixup=dict(p=1.0))
HBM_BYTES_PER_S = 3.35e12
KERNEL_SHAPES = ((256, 1000), (1024, 21843))


def gpu_info():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return {"name": name, "power_limit": power}
  except Exception as e:   # pylint: disable=broad-except
    return {"unavailable": f"{type(e).__name__}: {e}"[:200]}


def timed_ms(fn, steps, warmup):
  """Host clock around `steps` calls that end in a device synchronise -> ms per call."""
  import torch
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(steps):
    fn()
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) / steps * 1e3


def time_kernels(iters):
  """bv_distill_loss (kl, t = 1, with labels and gradient) and ops.softmax_xent at KERNEL_SHAPES."""
  import torch
  from big_vision_b200 import ops
  res = {}
  for n, C in KERNEL_SHAPES:
    g = torch.Generator(device="cuda").manual_seed(0)
    Cp = (C + 7) // 8 * 8                                        # the padded head's storage
    s, u = (torch.randn(n, Cp, device="cuda", generator=g)[:, :C] * 3 for _ in range(2))
    labels = torch.nn.functional.one_hot(torch.randint(0, C, (n,), device="cuda", generator=g), C).float()
    loss = torch.zeros(1, device="cuda")
    calls = {
        # reads s, u, labels and writes ds: 4 matrices; softmax_xent reads logits, labels and writes ds: 3
        "bv_distill_loss": (4, lambda: ops.distill_loss(s, u, labels, "kl", dlogits_cols=Cp)),
        "bv_softmax_xent_ld": (3, lambda: ops.softmax_xent(s, labels, loss, dlogits_cols=Cp)),
    }
    for name, (mats, fn) in calls.items():
      for _ in range(5):
        fn()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(iters):
        fn()
      e1.record()
      torch.cuda.synchronize()
      ms = e0.elapsed_time(e1) / iters
      floor_ms = mats * n * C * 4 / HBM_BYTES_PER_S * 1e3
      res[f"{name} ({n}, {C})"] = {"ms": ms, "bytes": mats * n * C * 4, "hbm_floor_ms": floor_ms,
                                   "share_of_3.35TBps": floor_ms / ms, "launches_timed": iters}
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=8)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--per-gpu-batch", type=int, default=256)
  ap.add_argument("--kernel-iters", type=int, default=50)
  args = ap.parse_args()
  import numpy as np
  import torch
  if not torch.cuda.is_available() or torch.cuda.get_device_capability(0)[0] != 9:
    raise SystemExit("bench_distill.py measures on a compute-capability 9.x GPU; there is no CPU path")
  from big_vision_b200 import optax as bv_optax, train
  from big_vision_b200.models import vit
  from big_vision_b200.trainers.proj.distill import distill as D
  info = gpu_info()
  n = args.per_gpu_batch
  student, teacher = vit.Model(CLASSES, **STUDENT), vit.Model(CLASSES, **TEACHER)
  s_shape, t_shape = (n, STUDENT_RES, STUDENT_RES, 3), (n, TEACHER_RES, TEACHER_RES, 3)
  g = torch.Generator(device="cuda").manual_seed(0)
  batch = {"image": torch.rand(s_shape, device="cuda", generator=g) * 2 - 1,
           "prof": torch.rand(t_shape, device="cuda", generator=g) * 2 - 1,
           "labels": torch.nn.functional.one_hot(torch.randint(0, CLASSES, (n,), device="cuda", generator=g),
                                                 CLASSES).float()}

  def small_head(P):                 # zero-initialised heads would make every logit 0 and the KL trivially 0
    P.tree("f")["head/kernel"].normal_(0.0, 0.02, generator=g)
    P.sync_half()
    return P

  Pt = small_head(teacher.init(1, t_shape)).drop_grad()
  sched_kw = dict(total_steps=10_000, batch_size=n, data_size=1_281_167)
  out = {"metric": "distill_vit_s16_from_b16_384_img_per_sec", "unit": "img/s", "gpu": info,
         "config": {"student": "ViT-S/16 @224 tok", "teacher": "ViT-B/16 @384 tok, frozen, no gradient buffer",
                    "classes": CLASSES, "per_gpu_batch": n, "distance": "kl, t=1", "mixup_p": 1.0,
                    "optimizer": "scale_by_adam, mu bf16, grad_clip_norm 1", "steps": args.steps,
                    "warmup": args.warmup}}

  # ---- the distill step
  P = small_head(student.init(0, s_shape))
  models, config = {"student": student, "prof": teacher}, dict(OPT_CONFIG, teachers=["prof"], distance="kl")
  tx, _ = bv_optax.make(config, P, sched_kw=sched_kw)
  state = {"params": {"student": P, "prof": Pt}, "opt": tx.init(P)}
  fn = D.make_update_fn(models, tx, config)
  rng = np.random.default_rng(0)
  torch.cuda.reset_peak_memory_stats()
  ms = timed_ms(lambda: fn(state, rng, batch), args.steps, args.warmup)
  _, m = fn(state, rng, batch)
  out.update(value=n / ms * 1e3, ms_per_step=ms, peak_mem_gib=torch.cuda.max_memory_allocated() / 2 ** 30,
             last_step={k: float(v) for k, v in m.items()})
  del state, fn, tx, P

  # ---- the plain train.py step of the student, and the teacher's forward alone
  P = small_head(student.init(0, s_shape))
  config = dict(OPT_CONFIG, loss="softmax_xent")
  tx, _ = bv_optax.make(config, P, sched_kw=sched_kw)
  state = {"params": P, "opt": tx.init(P)}
  fn = train.make_update_fn(student, tx, config)
  torch.cuda.reset_peak_memory_stats()
  ms_plain = timed_ms(lambda: fn(state, rng, batch), args.steps, args.warmup)
  out["plain_student_step"] = {"ms_per_step": ms_plain, "img_per_sec": n / ms_plain * 1e3,
                               "peak_mem_gib": torch.cuda.max_memory_allocated() / 2 ** 30}
  ms_teacher = timed_ms(lambda: teacher.apply({"params": Pt}, batch["prof"]), args.steps, args.warmup)
  out["teacher_apply"] = {"ms": ms_teacher, "img_per_sec": n / ms_teacher * 1e3}
  out["rest_ms"] = out["ms_per_step"] - ms_plain - ms_teacher      # the second mixup, the loss kernel, noise
  del state, fn, tx, P

  out["kernels"] = time_kernels(args.kernel_iters)
  print(json.dumps(out), flush=True)


if __name__ == "__main__":
  main()
