"""What dropout costs: the `configs/vit_i1k.py` ViT-B/16 step (bench.py's vit_b16_cls) at dropout 0.1 against
0.0, and the siglip_b16 step with dropout 0.1 in both towers against 0.0, then each dropout kernel against its
bytes over the H100 SXM data sheet's 3.35 TB/s.

Registers the dropout copies of the two workloads into bench.WORKLOADS in this process only and reuses
bench.py's measurement and JSON line for each arm, alternating rate 0 and 0.1 `--rounds` times.  The kernels
are timed with CUDA events at the shapes of one ViT-B/16 block at 256 images (M = 256 * 197 rows): the GELU
site (in place, 3072 columns) and a residual site (768 columns).

  python tools/bench_dropout.py [--steps 8] [--warmup 3] [--rounds 1]

Prints one JSON line: per workload and rate the step's ms, img/s or pairs/s, peak memory and launches, the
kernels, and the card's name and power limit read in the same run.
"""
import argparse
import contextlib
import io
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  pylint: disable=wrong-import-position
from bench_gsam import gpu_info  # noqa: E402  pylint: disable=wrong-import-position

HBM_BYTES_PER_S = 3.35e12
RATE = 0.1


def with_dropout(name, rate):
  """bench.WORKLOADS[name] with `rate` in every tower, registered as `<name>_drop<rate>`."""
  wl = dict(bench.WORKLOADS[name])
  kw = dict(wl["model_kw"])
  if wl["kind"] == "siglip":
    kw["image"] = dict(kw["image"], dropout=rate)
    kw["text"] = dict(kw["text"], dropout=rate)
  else:
    kw["dropout"] = rate
  wl["model_kw"] = kw
  wl["desc"] = f"{wl['desc']}; dropout {rate}"
  key = f"{name}_drop{rate}"
  bench.WORKLOADS[key] = wl
  return key


def run_arm(args, workload):
  import torch
  sys.argv = ["bench.py", "--workload", workload, "--steps", str(args.steps), "--warmup", str(args.warmup),
              "--no-cpu-baseline", "--no-gpu-baseline"]
  torch.cuda.reset_peak_memory_stats()
  buf = io.StringIO()
  with contextlib.redirect_stdout(buf):
    bench.main()
  line = json.loads(buf.getvalue().strip().splitlines()[-1])
  return {"value": line["value"], "unit": line.get("unit"), "ms_per_step": line.get("ms_per_step"),
          "peak_mem_gib": line["config"]["peak_mem_gib"], "gpu_launches": line.get("gpu_launches")}


def time_kernels(rows=256 * 197, iters=50):
  """bv_dropout in place at the GELU site and bv_dropout_add at a residual site, CUDA events around `iters`
  launches -> {name: {...}}."""
  import torch
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  key = L.DropoutKey(seed=0, step=1, site=7, row0=0, rate=RATE)
  act = torch.randn((rows, 3072), device="cuda").bfloat16()
  resid, y = (torch.randn((rows, 768), device="cuda").bfloat16() for _ in range(2))
  out = torch.empty_like(y)
  calls = {"bv_dropout [M, 3072] in place": (lambda: ops.dropout(act, key, out=act), 4 * rows * 3072),
           "bv_dropout_add [M, 768]": (lambda: ops.dropout_add(resid, y, key, out=out), 6 * rows * 768)}
  res = {}
  for name, (fn, nbytes) in calls.items():
    for _ in range(5):
      fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
      fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    floor_ms = nbytes / HBM_BYTES_PER_S * 1e3
    res[name] = {"ms": ms, "bytes": nbytes, "hbm_floor_ms": floor_ms, "share_of_3.35TBps": floor_ms / ms,
                 "TBps": nbytes / ms / 1e9}
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=8)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--rounds", type=int, default=1)
  args = ap.parse_args()
  info = gpu_info()
  out = {"gpu": info}
  for name in ("vit_b16_cls", "siglip_b16"):
    arms = {rate: with_dropout(name, rate) for rate in (0.0, RATE)}
    res = {str(rate): [] for rate in arms}
    for _ in range(args.rounds):
      for rate, wl in arms.items():
        res[str(rate)].append(run_arm(args, wl))
    out[name] = res
    out[name]["step_time_ratio"] = (min(r["ms_per_step"] for r in res[str(RATE)])
                                    / min(r["ms_per_step"] for r in res["0.0"]))
  out["kernels"] = time_kernels()
  print(json.dumps(out), flush=True)


if __name__ == "__main__":
  main()
