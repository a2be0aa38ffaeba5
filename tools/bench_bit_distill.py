"""Times the BiT distillation of configs/proj/distill/bit_i1k.py on one GPU, and the convolution kernels it runs.

  python tools/bench_bit_distill.py --batch 256 --steps 10 --warmup 3 [--out DIR]

Prints one JSON line with the card's name and power limit, then:
  - "distill": the step of trainers/proj/distill (R50x1 student under a frozen R152x2 teacher, 224 px, KL):
    images/s, ms per step and peak memory;
  - "student_train": the student's plain classifier step (forward, softmax xent, backward) alone;
  - "teacher_apply": the teacher's forward-only apply() alone;
  - "kernels": achieved TFLOP/s of the main convolution shapes (forward, data and kernel gradient), with
    FLOPs computed from the shapes (2 * pixels * k^2 * cin * cout) over CUDA-event time.
The optimizer update is not included in any step time."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from big_vision_b200 import ops  # noqa: E402
from big_vision_b200 import train  # noqa: E402
from big_vision_b200.models import bit_paper  # noqa: E402
from big_vision_b200.trainers.proj.distill import distill  # noqa: E402


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().split("\n")[0]
  return q


def timed(fn, steps, warmup):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(steps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated() / 2**30


# (k, stride, cin, cout, h): R50x1's 3 x 3 convolutions at 224 px and its strided projections
KERNEL_SHAPES = [(3, 1, 64, 64, 56), (3, 2, 128, 128, 56), (3, 1, 128, 128, 28), (3, 2, 256, 256, 28),
                 (3, 1, 256, 256, 14), (3, 2, 512, 512, 14), (3, 1, 512, 512, 7), (1, 2, 256, 512, 56),
                 (1, 2, 1024, 2048, 14)]


def kernel_rates(batch, steps, warmup):
  out = []
  for k, s, cin, cout, h in KERNEL_SHAPES:
    ho = (h + 2 * (k // 2) - k) // s + 1
    x = torch.randn(batch, h, h, cin, device="cuda").to(torch.bfloat16)
    w = (torch.randn(k, k, cin, cout, device="cuda") * (k * k * cin) ** -0.5).to(torch.bfloat16)
    dy = torch.randn(batch, ho, ho, cout, device="cuda").to(torch.bfloat16)
    flops = 2.0 * batch * ho * ho * k * k * cin * cout
    row = {"k": k, "stride": s, "cin": cin, "cout": cout, "h": h, "batch": batch}
    for name, fn in (("fwd", lambda: ops.conv_fwd(x, w, s)), ("dgrad", lambda: ops.conv_dgrad(dy, w, h, h, s)),
                     ("wgrad", lambda: ops.conv_wgrad(x, dy, k, s))):
      ms, _ = timed(fn, steps, warmup)
      row[name] = {"ms": round(ms, 4), "tflops": round(flops / ms / 1e9, 1)}
    out.append(row)
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, default=256)
  ap.add_argument("--steps", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  B = a.batch
  student = bit_paper.Model(num_classes=1000, depth=50, width=1)
  teacher = bit_paper.Model(num_classes=1000, depth=152, width=2)
  Ps = student.init(0, (1, 224, 224, 3))
  Pt = teacher.init(1, (1, 224, 224, 3)).drop_grad()
  image = torch.randn(B, 224, 224, 3, device="cuda")
  labels = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), device="cuda"), 1000).float()
  models, params = {"student": student, "prof_m": teacher}, {"student": Ps, "prof_m": Pt}
  res = {"card": card(), "batch": B, "image": 224}

  ms, mem = timed(lambda: distill.loss_and_grads(models, params, {"image": image}, ("prof_m",), "kl"), a.steps,
                  a.warmup)
  res["distill"] = {"ms_per_step": round(ms, 2), "img_per_s": round(B / ms * 1e3, 1), "peak_gib": round(mem, 2)}
  ms, mem = timed(lambda: train.loss_and_grads(student, Ps, image, labels, "softmax_xent"), a.steps, a.warmup)
  res["student_train"] = {"ms_per_step": round(ms, 2), "img_per_s": round(B / ms * 1e3, 1), "peak_gib": round(mem, 2)}
  ms, mem = timed(lambda: teacher.apply({"params": Pt}, image), a.steps, a.warmup)
  res["teacher_apply"] = {"ms_per_step": round(ms, 2), "img_per_s": round(B / ms * 1e3, 1), "peak_gib": round(mem, 2)}
  del image
  res["kernels"] = kernel_rates(min(B, 64), a.steps, a.warmup)
  line = json.dumps(res)
  print(line)
  if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_bit_distill.json"), "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
