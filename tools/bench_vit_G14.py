"""ViT-G/14 classification pre-training step (configs/proj/scaling_laws/train_vit_g.py with its one-line
switch to `G/14`): 224x224, MAP pool, the 29,593-class JFT head, sigmoid_xent, BV-Adafactor, per-block
recompute.  Head dim 104 (1664 / 16) and a class count that is not a multiple of 8, so the head is
stored padded (models/common.py Dense, pad=True).  1,930.4 M parameters: the flat fp32 parameter and
gradient buffers are 7.2 GiB each.

Registers `scaling_laws_vit_G14` into bench.WORKLOADS and sets bench.OPT_CONFIG to the config's
optimizer, in this process only, then reuses bench.py's measurement and JSON line; bench.py's own
workload list and optimizer stay the BASELINE.json ones.  Mixup is not on the timed path (bench.py
steps with rng=None).

  python tools/bench_vit_G14.py [--steps 8] [--warmup 3] [--per-gpu-batch N] [--profile-calls]

Prints one JSON line: our arm as bench.py prints it plus parameter counts, with the labelled PyTorch
stand-in (baseline/torch_gpu.py: fused AdamW, not Adafactor) measured in its own process in
`gpu_baseline`.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  pylint: disable=wrong-import-position

NAME = "scaling_laws_vit_G14"
# per-GPU batch 512: 57.0 GiB peak on an 80 GB H100 (DESIGN.md section 5); larger batches not measured
RES, PATCH, WIDTH, DEPTH, MLP, HEADS, CLASSES = 224, 14, 1664, 48, 8192, 16, 29_593

# configs/proj/scaling_laws/train_vit_g.py, optimizer section.  The schedule keeps the config's shape (rsqrt
# with warmup and cooldown) with its durations cut to fit bench.py's 10,000-step horizon (the config's
# warmup alone is 10,000 steps); the step time does not depend on them.
OPT_CONFIG = dict(optax_name="big_vision.scale_by_adafactor", grad_clip_norm=1.0, lr=8e-4, wd=0.03 * 8e-4,
                  wd_mults=[(".*head/kernel", 100.0), (".*/kernel", 1.0)],
                  schedule=dict(decay_type="rsqrt", timescale=1_000, warmup_steps=1_000, cooldown_steps=5_000))


def image_train_flops(res=RES, patch=PATCH, d=WIDTH, m=MLP, depth=DEPTH, classes=CLASSES):
  """Algorithmic training FLOPs per image (SURVEY.md 8d): 3 x forward, recompute not counted."""
  n = (res // patch) ** 2
  block = 8 * n * d * d + 4 * n * d * m + 4 * n * n * d          # q, k, v, out; MLP; S and P V
  fwd = (2 * n * patch * patch * 3 * d                             # patch embedding
         + depth * block
         + 4 * n * d * d + 4 * d * d + 4 * n * d + 4 * d * m       # MAP head: k, v; q, out; attention; MLP
         + 2 * d * classes)                                        # class head
  return 3 * fwd


WORKLOAD = dict(
    kind="cls", model="vit", metric="vit_G14_cls_img_per_sec", unit="img/s", res=RES, per_gpu_batch=512,
    flops=image_train_flops(), num_classes=CLASSES, loss="sigmoid_xent", remat=True,
    model_kw=dict(variant=f"G/{PATCH}", pool_type="map", scan=True),
    oracle=dict(depth=DEPTH, num_heads=HEADS, pool_type="map", posemb="learn", rep_size=False, num_classes=CLASSES),
    desc="ViT-G/14 (configs/proj/scaling_laws/train_vit_g.py: 256 tokens, map pool, head dim 104, 29593 "
         "classes, sigmoid_xent, BV-Adafactor, grad_clip_norm 1, wd_mults), 224x224, full update_fn with "
         "per-block recompute (models/vit.py:129-148 nn.remat, nothing_saveable)")


def register():
  bench.WORKLOADS[NAME] = WORKLOAD
  bench.OPT_CONFIG = OPT_CONFIG
  return WORKLOAD


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=8)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--per-gpu-batch", type=int, default=0, help=f"0 = {WORKLOAD['per_gpu_batch']}")
  ap.add_argument("--impl", default="ours", choices=["ours", "torch_gpu"])
  ap.add_argument("--profile-calls", action="store_true")
  ap.add_argument("--no-gpu-baseline", action="store_true")
  args = ap.parse_args()
  register()
  argv = ["bench.py", "--workload", NAME, "--steps", str(args.steps), "--warmup", str(args.warmup),
          "--per-gpu-batch", str(args.per_gpu_batch)]
  if args.impl == "torch_gpu":
    sys.argv = argv + ["--impl", "torch_gpu"]
    bench.main()
    return
  sys.argv = argv + ["--no-cpu-baseline", "--no-gpu-baseline"] + (["--profile-calls"] if args.profile_calls else [])
  buf = io.StringIO()
  with contextlib.redirect_stdout(buf):
    bench.main()
  line = json.loads(buf.getvalue().strip().splitlines()[-1])
  line["config"]["params"] = param_counts()
  line["config"]["optimizer"] = "big_vision.scale_by_adafactor (train_vit_g.py)"
  if not args.no_gpu_baseline:
    # the stand-in in its own process (this one's device memory is released when it exits)
    cmd = [sys.executable, os.path.abspath(__file__), "--impl", "torch_gpu", "--steps", str(min(args.steps, 6)),
           "--warmup", "3", "--per-gpu-batch", str(args.per_gpu_batch)]
    try:
      out = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
      line["gpu_baseline"] = json.loads(out.stdout.strip().splitlines()[-1])
    except Exception as e:   # pylint: disable=broad-except
      line["gpu_baseline"] = {"impl": "torch_gpu", "unavailable": f"{type(e).__name__}: {e}"[:300]}
    line["gpu_baseline"]["optimizer"] = "fused AdamW (torch.optim), not Adafactor"
  print(json.dumps(line), flush=True)


def param_counts():
  """Parameter counts under the reference names and shapes (nothing allocated)."""
  from big_vision_b200 import engine as E
  model = bench.build_model(WORKLOAD)
  specs, aliases = model.specs((RES, RES), 3)
  tree = E.FlatParams(specs, aliases, "meta").tree("f")
  head = sum(v.numel() for k, v in tree.items() if k.startswith("head/"))
  return {"total": sum(v.numel() for v in tree.values()), "head": head}


if __name__ == "__main__":
  main()
