"""What BERT's dropout costs: the SigLiT step of `configs/proj/image_text/siglip_lit_coco.py` with
txt=bert_base (tools/bench_siglit.py's workload: frozen ViT-B/16, BERT-Base on 16 zero-padded tokens, 512 pairs
per GPU) at the config's rates (0.1 hidden and attention dropout, bert.CONFIGS["base"]) against rates 0, and
the key-masked attention forward + backward with and without BV_ATTN_DROPOUT.

The step arms reuse bench.py's measurement and JSON line through bench_siglit.register, alternating the two
rate settings `--rounds` times in this process.  The attention is timed with CUDA events over `--iters`
calls at BERT-Base's shape (512 captions x 12 heads, N = 16, caption-length masks) and at N = 128 and
N = 512 (random masks, 60 % of the keys attended), 12 heads of 64, at 8192 query rows per head.

  python tools/bench_bert_dropout.py [--steps 8] [--warmup 3] [--rounds 2] [--iters 50]

Prints one JSON line: per rate setting the step's ms, pairs/s, peak memory and launches, the attention times,
and the card's name and power limit read in the same run.
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
import bench_siglit  # noqa: E402  pylint: disable=wrong-import-position
from bench_gsam import gpu_info  # noqa: E402  pylint: disable=wrong-import-position

RATE = 0.1
# BERT-Base as a dict config: the same tower with both dropout rates left at 0
BASE_NO_DROPOUT = dict(width=768, depth=12, num_heads=12, mlp_dim=3072)


def run_arm(args, text_config):
  import torch
  wl = bench.WORKLOADS[bench_siglit.NAME]
  wl["model_kw"] = dict(wl["model_kw"], text=dict(wl["model_kw"]["text"], config=text_config))
  sys.argv = ["bench.py", "--workload", bench_siglit.NAME, "--steps", str(args.steps), "--warmup", str(args.warmup),
              "--per-gpu-batch", str(bench_siglit.BERT_BATCH), "--no-cpu-baseline", "--no-gpu-baseline"]
  torch.cuda.empty_cache()
  torch.cuda.reset_peak_memory_stats()
  buf = io.StringIO()
  with contextlib.redirect_stdout(buf):
    bench.main()
  line = json.loads(buf.getvalue().strip().splitlines()[-1])
  return {"value": line["value"], "unit": line.get("unit"), "ms_per_step": line.get("ms_per_step"),
          "peak_mem_gib": line["config"]["peak_mem_gib"], "gpu_launches": line.get("gpu_launches")}


def time_attention(iters):
  """Masked attention forward + backward without and with BV_ATTN_DROPOUT (rate 0.1) -> {shape: {...}}."""
  import numpy as np
  import torch
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  heads, d = 12, 12 * 64
  key = L.DropoutKey(seed=0, step=1, site=2, row0=0, rate=RATE)
  out = {}
  for B, N, kind in ((512, 16, "captions"), (64, 128, "random"), (16, 512, "random")):
    rng = np.random.default_rng(N)
    qkv = torch.from_numpy(rng.standard_normal((B, N, 3 * d), dtype=np.float32)).cuda().bfloat16()
    do = torch.from_numpy(rng.standard_normal((B, N, d), dtype=np.float32)).cuda().bfloat16()
    if kind == "captions":
      mask = np.arange(N)[None, :] < rng.integers(4, N + 1, size=B)[:, None]
    else:
      mask = rng.random((B, N)) < 0.6
      mask[:, 0] = True
    mask = torch.from_numpy(mask.astype(np.uint8)).cuda()
    q, k, v = qkv[:, :, :d], qkv[:, :, d:2 * d], qkv[:, :, 2 * d:]
    row = {}
    for label, drop in (("masked", None), ("masked+dropout", key)):
      def call(drop=drop):
        o, lse = ops.attention_fwd(q, k, v, heads, key_mask=mask, dropout=drop)
        ops.attention_bwd(do, q, k, v, o, lse, heads, key_mask=mask, dropout=drop)
      for _ in range(5):
        call()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(iters):
        call()
      e1.record()
      torch.cuda.synchronize()
      row[label + "_ms"] = e0.elapsed_time(e1) / iters
    row["ratio"] = row["masked+dropout_ms"] / row["masked_ms"]
    out[f"{B}x{heads}x{N} {kind}"] = row
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=8)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--rounds", type=int, default=2)
  ap.add_argument("--iters", type=int, default=50)
  args = ap.parse_args()
  out = {"gpu": gpu_info()}
  bench_siglit.register(txt="bert_base")
  arms = {"rates 0.1 (config)": "base", "rates 0": BASE_NO_DROPOUT}
  res = {name: [] for name in arms}
  for _ in range(args.rounds):
    for name, cfg in arms.items():
      res[name].append(run_arm(args, cfg))
  out["siglit_bert_base"] = res
  out["siglit_bert_base"]["step_time_ratio"] = (min(r["ms_per_step"] for r in res["rates 0.1 (config)"])
                                                / min(r["ms_per_step"] for r in res["rates 0"]))
  out["attention_fwd_bwd"] = time_attention(args.iters)
  print(json.dumps(out), flush=True)


if __name__ == "__main__":
  main()
