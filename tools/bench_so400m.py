"""SigLIP So400m/14 training step (image So400m/14 @224, map pool + text So400m): the first workload
with a head dim other than 64 (width 1152 / 16 heads = 72).  Registers `siglip_so400m14_224` into
bench.WORKLOADS in this process only and reuses bench.py's measurement and JSON line; bench.py's own
workload list stays the BASELINE.json configs.

  python tools/bench_so400m.py [--steps 8] [--warmup 3] [--per-gpu-batch N] [--profile-calls]

Prints one JSON line: our arm as bench.py prints it, with the labelled PyTorch stand-in
(baseline/torch_gpu.py) measured in its own process in `gpu_baseline`.
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

NAME = "siglip_so400m14_224"
# per-GPU batch 1024: 51.0 GiB peak on an 80 GB H100 (512: 32.0 GiB; DESIGN.md section 5)
RES, PATCH, WIDTH, DEPTH, MLP, HEADS = 224, 14, 1152, 27, 4304, 16


def tower_fwd_flops(n_tok, d, m, depth):
  """SURVEY.md 8d: per pre-LN block 8*N*d^2 (q, k, v, out) + 4*N*d*m (MLP) + 4*N^2*d (S and P V)."""
  return depth * (8 * n_tok * d * d + 4 * n_tok * d * m + 4 * n_tok * n_tok * d)


def pair_train_flops(res=RES, patch=PATCH, txt_len=bench.TXT_LEN, d=WIDTH, m=MLP, depth=DEPTH, out=WIDTH):
  """Algorithmic training FLOPs per image-text pair: 3 x forward (recompute not counted)."""
  n_img = (res // patch) ** 2
  img = (2 * n_img * patch * patch * 3 * d                       # patch embedding
         + tower_fwd_flops(n_img, d, m, depth)
         + 4 * n_img * d * d + 4 * d * d + 4 * n_img * d + 4 * d * m)   # MAP head: k, v; q, out; attention; MLP
  txt = tower_fwd_flops(txt_len, d, m, depth) + 2 * d * out          # text encoder + projection head
  return 3 * (img + txt)


WORKLOAD = dict(
    kind="siglip", metric="siglip_so400m14_224_pairs_per_sec", unit="pairs/s", res=RES, per_gpu_batch=1024,
    flops=pair_train_flops(), remat=True,
    model_kw=dict(image=dict(variant=f"So400m/{PATCH}", pool_type="map"),
                  text=dict(variant="So400m", vocab_size=32_000),
                  out_dim=(None, WIDTH), temperature_init=10.0, bias_init=-10.0),
    oracle=dict(image=dict(depth=DEPTH, num_heads=HEADS, pool_type="map", posemb="learn", rep_size=False,
                           num_classes=None),
                text=dict(depth=DEPTH, num_heads=HEADS, pool_type="last", num_classes=WIDTH)),
    desc="SigLIP two_towers So400m/14 (256 tokens, map pool, head dim 72) + text So400m (64 tok, vocab 32000; "
         "the released checkpoints use 16 text tokens), 224x224, full update_fn with per-block recompute "
         "(models/vit.py:129-148 nn.remat, nothing_saveable)")


def register():
  bench.WORKLOADS[NAME] = WORKLOAD
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
  if not args.no_gpu_baseline:
    # the stand-in in its own process (this one's device memory is released when it exits)
    cmd = [sys.executable, os.path.abspath(__file__), "--impl", "torch_gpu", "--steps", str(min(args.steps, 6)),
           "--warmup", "3", "--per-gpu-batch", str(args.per_gpu_batch)]
    try:
      out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
      line["gpu_baseline"] = json.loads(out.stdout.strip().splitlines()[-1])
    except Exception as e:   # pylint: disable=broad-except
      line["gpu_baseline"] = {"impl": "torch_gpu", "unavailable": f"{type(e).__name__}: {e}"[:300]}
  print(json.dumps(line), flush=True)


def param_counts():
  """Parameter counts of the two towers (shapes only, nothing allocated)."""
  from big_vision_b200 import engine as E
  model = bench.build_model(WORKLOAD)
  specs, aliases = model.specs((1, RES, RES, 3), (1, bench.TXT_LEN))
  tree = E.FlatParams(specs, aliases, "meta").tree("f")
  count = lambda prefix: sum(v.numel() for k, v in tree.items() if k.startswith(prefix))  # noqa: E731
  return {"img": count("img/"), "txt": count("txt/"), "total": sum(v.numel() for v in tree.values())}


if __name__ == "__main__":
  main()
