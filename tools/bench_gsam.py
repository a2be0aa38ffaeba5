"""GSAM ViT-B/32 classification step (configs/proj/gsam/vit_i1k_gsam_no_aug.py): 224x224, gap pool, no
rep_size, 1000 classes, sigmoid_xent, init_head_bias -10, Adam with fp32 mu, grad_clip_norm 1, and the
config's gsam dict; 512 images per GPU (the config's 4096 over 8 GPUs).

Registers `gsam_vit_b32` into bench.WORKLOADS and sets bench.OPT_CONFIG to the config's optimizer, in this
process only, then reuses bench.py's measurement and JSON line twice in the same run: once with the GSAM
step (trainers/proj/gsam/train.py) and once with the plain train.py step on the same workload.  Then it
times each GSAM kernel (bv_sam_perturb, bv_sam_dots, bv_gsam_combine) with CUDA events on buffers of the
model's parameter count, against its bytes over the H100 SXM data sheet's 3.35 TB/s.

  python tools/bench_gsam.py [--steps 8] [--warmup 3] [--per-gpu-batch N]

Prints one JSON line: the GSAM arm as bench.py prints it, plus `plain` (the train.py arm), `ratio`
(GSAM img/s over plain img/s), `kernels` and the card's name and power limit read in the same run.
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

NAME = "gsam_vit_b32"
RES, PATCH, WIDTH, DEPTH, MLP, CLASSES = 224, 32, 768, 12, 3072, 1000
LR = 0.003

# configs/proj/gsam/vit_i1k_gsam_no_aug.py, optimizer and GSAM sections.  The warmup is cut from 10,000 to
# 1,000 steps to fit bench.py's 10,000-step horizon; the step time does not depend on it.
OPT_CONFIG = dict(optax_name="scale_by_adam", optax=dict(mu_dtype="float32"), grad_clip_norm=1.0, lr=LR, wd=0.001,
                  schedule=dict(warmup_steps=1_000, decay_type="linear", linear_end=0.01),
                  gsam=dict(rho_max=0.6, rho_min=0.1, alpha=0.6, lr_max=LR, lr_min=0.01 * LR))
HBM_BYTES_PER_S = 3.35e12
# bytes per parameter each kernel must move (fp32 4 B, bf16 2 B)
KERNEL_BYTES = {"bv_sam_dots (||g_c||^2, one buffer)": 4, "bv_sam_perturb": 14, "bv_sam_dots (g_c.g_r, ||g_r||^2)": 8,
                "bv_gsam_combine": 12}


def image_fwd_flops(res=RES, patch=PATCH, d=WIDTH, m=MLP, depth=DEPTH, classes=CLASSES):
  """Forward FLOPs per image (SURVEY.md 8d), gap pool, no pre-logits."""
  n = (res // patch) ** 2
  block = 8 * n * d * d + 4 * n * d * m + 4 * n * n * d          # q, k, v, out; MLP; S and P V
  return 2 * n * patch * patch * 3 * d + depth * block + 2 * d * classes


WORKLOAD = dict(
    kind="cls", model="vit", metric="gsam_vit_b32_img_per_sec", unit="img/s", res=RES, per_gpu_batch=512,
    flops=2 * 3 * image_fwd_flops(), num_classes=CLASSES, loss="sigmoid_xent",
    model_kw=dict(variant=f"B/{PATCH}", pool_type="gap", rep_size=False),
    oracle=dict(depth=DEPTH, num_heads=12, pool_type="gap", posemb="learn", rep_size=False, num_classes=CLASSES),
    desc="ViT-B/32 GSAM (configs/proj/gsam/vit_i1k_gsam_no_aug.py: gap pool, no rep_size, sigmoid_xent, "
         "init_head_bias -10, Adam fp32 mu, grad_clip_norm 1, rho 0.6..0.1, alpha 0.6), 224x224, two "
         "forward+backward passes per step")


def register():
  bench.WORKLOADS[NAME] = WORKLOAD
  bench.OPT_CONFIG = OPT_CONFIG
  init = bench.init_params

  def init_with_head_bias(wl, model, n, device):      # train.py: config.init_head_bias
    P = init(wl, model, n, device)
    if wl is WORKLOAD:
      P.tree("f")["head/bias"].fill_(-10.0)
    return P

  bench.init_params = init_with_head_bias
  return WORKLOAD


def run_arm(args, gsam):
  """One bench.py measurement of WORKLOAD; `gsam` selects trainers/proj/gsam's update_fn."""
  import torch
  from big_vision_b200 import train
  from big_vision_b200.trainers.proj.gsam import train as gtrain
  plain = train.make_update_fn
  if gsam:
    train.make_update_fn = gtrain.make_update_fn
  sys.argv = ["bench.py", "--workload", NAME, "--steps", str(args.steps), "--warmup", str(args.warmup),
              "--per-gpu-batch", str(args.per_gpu_batch), "--no-cpu-baseline", "--no-gpu-baseline"]
  torch.cuda.reset_peak_memory_stats()
  buf = io.StringIO()
  try:
    with contextlib.redirect_stdout(buf):
      bench.main()
  finally:
    train.make_update_fn = plain
  return json.loads(buf.getvalue().strip().splitlines()[-1])


def time_kernels(n, iters=50):
  """Each GSAM kernel on n-element buffers, CUDA events around `iters` launches -> {name: {...}}."""
  import torch
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  g = torch.Generator(device="cuda").manual_seed(0)
  w, gc, gr = (torch.randn(n, device="cuda", generator=g) for _ in range(3))
  out, out16 = torch.empty_like(w), torch.empty(n, dtype=torch.bfloat16, device="cuda")
  sc, ws = torch.zeros(4, device="cuda"), torch.empty(L.SAM_WS_FLOATS, device="cuda")
  ops.sam_dots(gc, gc, out=sc[0:2], ws=ws)
  ops.sam_dots(gc, gr, out=sc[2:4], ws=ws)
  calls = {
      "bv_sam_dots (||g_c||^2, one buffer)": lambda: ops.sam_dots(gc, gc, out=sc[0:2], ws=ws),
      "bv_sam_perturb": lambda: ops.sam_perturb(w, gc, sc[0:1], 0.5, 1e-12, False, out=out, out_bf16=out16),
      "bv_sam_dots (g_c.g_r, ||g_r||^2)": lambda: ops.sam_dots(gc, gr, out=sc[2:4], ws=ws),
      # alpha 0 keeps the buffer's values from growing over the repeated in-place launches
      "bv_gsam_combine": lambda: ops.gsam_combine(out, gr, sc[2:3], sc[3:4], 0.0, True),
  }
  res = {}
  for name, fn in calls.items():
    for _ in range(5):
      fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
      fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    floor_ms = KERNEL_BYTES[name] * n / HBM_BYTES_PER_S * 1e3
    res[name] = {"ms": ms, "bytes_per_param": KERNEL_BYTES[name], "hbm_floor_ms": floor_ms,
                 "share_of_3.35TBps": floor_ms / ms}
  res["total"] = {"ms": sum(v["ms"] for v in res.values()), "bytes_per_param": sum(KERNEL_BYTES.values())}
  return res


def gpu_info():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return {"name": name, "power_limit": power}
  except Exception as e:   # pylint: disable=broad-except
    return {"unavailable": f"{type(e).__name__}: {e}"[:200]}


def param_count():
  from big_vision_b200 import engine as E
  model = bench.build_model(WORKLOAD)
  specs, aliases = model.specs((RES, RES), 3)
  P = E.FlatParams(specs, aliases, "meta")
  return P.total, sum(v.numel() for v in P.tree("f").values())


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=8)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--per-gpu-batch", type=int, default=0, help=f"0 = {WORKLOAD['per_gpu_batch']}")
  args = ap.parse_args()
  register()
  info = gpu_info()
  plain = run_arm(args, gsam=False)
  line = run_arm(args, gsam=True)
  flat, params = param_count()
  line["config"]["params"] = params
  line["config"]["seq_len"] = (RES // PATCH) ** 2          # bench.py's line assumes 16-pixel patches
  line["config"]["optimizer"] = "scale_by_adam, mu fp32 (vit_i1k_gsam_no_aug.py)"
  line["plain"] = {"metric": "plain train.py step, same workload", "value": plain["value"],
                   "ms_per_step": plain["ms_per_step"], "peak_mem_gib": plain["config"]["peak_mem_gib"],
                   "gpu_launches": plain["gpu_launches"]}
  line["ratio"] = line["value"] / plain["value"]
  line["step_time_ratio"] = line["ms_per_step"] / plain["ms_per_step"]
  line["kernels"] = time_kernels(flat)
  line["gpu"] = info
  print(json.dumps(line), flush=True)


if __name__ == "__main__":
  main()
