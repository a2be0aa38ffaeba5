"""SigLiT (locked-image tuning) training step: the siglip_b16 workload with the image tower frozen by
the optimizer schedule, `[("img/.*", None), (".*", cosine)]` (big_vision's
configs/proj/image_text/siglip_lit_coco.py).  The image tower runs forward-only, the loss computes no
image-embedding gradient and the all-reduce covers the text tower, `t` and `b` only.  Registers
`siglip_b16_lit` into bench.WORKLOADS and overrides bench.OPT_CONFIG's schedule in its own processes
only; bench.py's workloads and optimizer stay as they are.

  python tools/bench_siglit.py [--steps 8] [--warmup 3] [--repeats 3] [--per-gpu-batch 768,max]

Prints one JSON line: for every per-GPU batch ("max" = the largest multiple of 128 whose predicted peak
fits the card, extrapolated from the peaks at 768 and 1536 and then measured) the median pairs/s over
`repeats` runs, their spread and the peak memory; the PyTorch stand-in (baseline/torch_gpu.py) with
its image tower frozen (requires_grad_(False), forward under torch.no_grad()) at 768; and plain
`bench.py --gpus 1` (the full siglip_b16 step) over the same repeats.  Every arm runs in its own
process, so each starts with an empty device.
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  pylint: disable=wrong-import-position
from bench_so400m import tower_fwd_flops  # noqa: E402  pylint: disable=wrong-import-position

NAME = "siglip_b16_lit"
RES, PATCH, WIDTH, DEPTH, MLP = 224, 16, 768, 12, 3072
LIT_SCHEDULE = [("img/.*", None), (".*", dict(bench.OPT_CONFIG["schedule"]))]


def pair_flops(global_batch):
  """Algorithmic FLOPs per pair of a SigLiT step: the image tower's forward once, the text tower's
  three times (forward + backward), and the loss's two [n, B] x D products per pair (dots and the
  text-embedding gradient; the image-embedding gradient is not computed)."""
  n_img = (RES // PATCH) ** 2
  img = (2 * n_img * PATCH * PATCH * 3 * WIDTH + tower_fwd_flops(n_img, WIDTH, MLP, DEPTH)
         + 4 * n_img * WIDTH * WIDTH + 4 * WIDTH * WIDTH + 4 * n_img * WIDTH + 4 * WIDTH * MLP)   # + MAP head
  txt = tower_fwd_flops(bench.TXT_LEN, WIDTH, MLP, DEPTH) + 2 * WIDTH * WIDTH
  return img + 3 * txt + 2 * 2 * global_batch * WIDTH


WORKLOAD = dict(bench.WORKLOADS["siglip_b16"], metric="siglip_b16_lit_pairs_per_sec", flops=pair_flops(768),
                freeze_img=True,
                desc="SigLiT: SigLIP two_towers ViT-B/16 (map pool) FROZEN by schedule [('img/.*', None), "
                     "('.*', cosine)] + text-B trained (64 tok, vocab 32000), 224x224, full update_fn")


def register(per_gpu_batch=768):
  bench.WORKLOADS[NAME] = dict(WORKLOAD, flops=pair_flops(per_gpu_batch))
  bench.OPT_CONFIG["schedule"] = LIT_SCHEDULE
  return bench.WORKLOADS[NAME]


def run_one(args):
  """One arm in this process: bench.main's JSON line, plus the card's memory."""
  import torch
  n = args.per_gpu_batch or WORKLOAD["per_gpu_batch"]
  register(n)
  argv = ["bench.py", "--workload", NAME, "--steps", str(args.steps), "--warmup", str(args.warmup),
          "--per-gpu-batch", str(n)]
  if args.impl == "torch_gpu":
    sys.argv = argv + ["--impl", "torch_gpu"]
  else:
    sys.argv = argv + ["--no-cpu-baseline", "--no-gpu-baseline"]
  buf = io.StringIO()
  with contextlib.redirect_stdout(buf):
    bench.main()
  line = json.loads(buf.getvalue().strip().splitlines()[-1])
  line["total_mem_gib"] = torch.cuda.get_device_properties(0).total_memory / 2**30
  print(json.dumps(line), flush=True)


def _child(cmd, timeout=1200):
  out = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, cwd=ROOT)
  lines = out.stdout.strip().splitlines()
  if out.returncode != 0 or not lines:
    return {"unavailable": f"exit {out.returncode}: {out.stderr.strip()[-400:]}"}
  return json.loads(lines[-1])


def _ours(args, n):
  return _child([sys.executable, os.path.abspath(__file__), "--impl", "ours", "--per-gpu-batch", str(n),
                 "--steps", str(args.steps), "--warmup", str(args.warmup)])


def _summary(lines):
  ok = [l for l in lines if "value" in l]
  if not ok:
    return {"unavailable": lines[-1].get("unavailable") if lines else "no run"}
  vals = sorted(l["value"] for l in ok)
  return {"median": statistics.median(vals), "min": vals[0], "max": vals[-1], "runs": vals,
          "spread_pct": 100.0 * (vals[-1] - vals[0]) / statistics.median(vals),
          "ms_per_step": statistics.median(l["ms_per_step"] for l in ok),
          "peak_mem_gib": max(l["config"]["peak_mem_gib"] for l in ok),
          "per_gpu_batch": ok[0]["config"]["per_gpu_batch"],
          "step_mfu": statistics.median(l["roofline"]["step_mfu"] for l in ok),
          "final_loss": ok[-1]["config"]["final_loss"]}


def suite(args):
  result = {"metric": WORKLOAD["metric"], "unit": "pairs/s", "workload": f"{NAME}: {WORKLOAD['desc']}",
            "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "lit": {}}
  batches = [b for b in args.per_gpu_batch.split(",") if b]
  probe = {}
  if "max" in batches:
    # peak = fixed + per_pair * n: two points give the line, the card's memory the largest n
    for n in (768, 1536):
      probe[n] = _ours(args, n)
    a, b = probe[768], probe[1536]
    if "config" in a and "config" in b:
      per_pair = (b["config"]["peak_mem_gib"] - a["config"]["peak_mem_gib"]) / 768
      fixed = a["config"]["peak_mem_gib"] - 768 * per_pair
      budget = 0.97 * a["total_mem_gib"]
      n_max = int((budget - fixed) / per_pair) // 128 * 128
      result["max_batch_fit"] = {"gib_per_pair": per_pair, "fixed_gib": fixed, "budget_gib": budget,
                                 "per_gpu_batch": n_max}
    else:
      n_max = None
      result["max_batch_fit"] = {"unavailable": [a.get("unavailable"), b.get("unavailable")]}
  for tag in batches:
    n = n_max if tag == "max" else int(tag)
    if n is None:
      continue
    runs = [probe[n]] if n in probe else []          # a probe run is the first repeat
    runs += [_ours(args, n) for _ in range(args.repeats - len(runs))]
    result["lit"][tag] = _summary(runs)
  if not args.no_gpu_baseline:
    result["gpu_baseline_lit_768"] = _child([sys.executable, os.path.abspath(__file__), "--impl", "torch_gpu",
                                             "--per-gpu-batch", "768", "--steps", str(min(args.steps, 6)),
                                             "--warmup", "3"])
  if not args.no_full:
    full = [_child([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps),
                    "--warmup", str(args.warmup), "--no-cpu-baseline", "--no-gpu-baseline"])
            for _ in range(args.repeats)]
    result["full_siglip_b16"] = _summary(full)
  print(json.dumps(result), flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=8)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--repeats", type=int, default=3)
  ap.add_argument("--per-gpu-batch", default="768,max",
                  help="comma list of per-GPU batches (suite) or one batch (--impl ours / torch_gpu)")
  ap.add_argument("--impl", default="suite", choices=["suite", "ours", "torch_gpu"])
  ap.add_argument("--no-gpu-baseline", action="store_true")
  ap.add_argument("--no-full", action="store_true", help="skip the full-step bench.py runs")
  args = ap.parse_args()
  if args.impl == "suite":
    suite(args)
  else:
    args.per_gpu_batch = int(args.per_gpu_batch)
    run_one(args)


if __name__ == "__main__":
  main()
