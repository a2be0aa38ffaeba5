"""SigLiT (locked-image tuning) training step: the siglip_b16 workload with the image tower frozen by
the optimizer schedule, `[("img/.*", None), (".*", cosine)]` (big_vision's
configs/proj/image_text/siglip_lit_coco.py).  The image tower runs forward-only, the loss computes no
image-embedding gradient and the all-reduce covers the text tower, `t` and `b` only.  Registers
`siglip_b16_lit` into bench.WORKLOADS and overrides bench.OPT_CONFIG's schedule in its own processes
only; bench.py's workloads and optimizer stay as they are.

  python tools/bench_siglit.py [--steps 8] [--warmup 3] [--repeats 3] [--per-gpu-batch 768,max]

With --txt bert_base | bert_large it runs the step of that config as written instead: the frozen B/16 image
tower at 224 with pool_type='tok' and no image head, the BERT text tower (models/proj/flaxformer/bert.py)
on 16 zero-padded tokens, bias_init -2.71, Adam (Adafactor for bert_large), lr 1e-3, wd 0.01, cosine
schedule, gradient clip 1, at the config's 512 pairs per GPU and the largest batch that fits.  The stand-in
is `transformers.BertModel` (random weights from a BertConfig, nothing downloaded) under bf16 autocast
with the same frozen image tower (baseline/torch_gpu.py's ViT); and the masked attention is timed against
the unmasked one at the BERT shapes (B x 12 heads, N = 16) and at N = 128 with random masks.

  python tools/bench_siglit.py --txt bert_base [--per-gpu-batch 512,max]

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

# configs/proj/image_text/siglip_lit_coco.py with txt=bert_base / bert_large
BERT_TOKENS, BERT_BATCH, BERT_MAX_BATCH = 16, 512, 4096
BERT = {"bert_base": dict(config="base", width=768, depth=12, mlp=3072, heads=12, optax_name="scale_by_adam"),
        "bert_large": dict(config="large", width=1024, depth=24, mlp=4096, heads=16,
                           optax_name="big_vision.scale_by_adafactor")}


def bert_pair_flops(txt):
  """As pair_flops, with the BERT tower of 16 tokens (its embedding LayerNorm and gathers not counted) and
  the image tower's [cls] token instead of the MAP head."""
  b = BERT[txt]
  n_img = (RES // PATCH) ** 2 + 1
  img = 2 * (n_img - 1) * PATCH * PATCH * 3 * WIDTH + tower_fwd_flops(n_img, WIDTH, MLP, DEPTH)
  txt_f = tower_fwd_flops(BERT_TOKENS, b["width"], b["mlp"], b["depth"]) + 2 * b["width"] * b["width"]
  return img + 3 * txt_f


def bert_workload(txt):
  b = BERT[txt]
  return dict(bench.WORKLOADS["siglip_b16"], metric=f"siglit_{txt}_pairs_per_sec", per_gpu_batch=BERT_BATCH,
              flops=bert_pair_flops(txt), freeze_img=True,
              model_kw=dict(image=dict(variant="B/16", pool_type="tok", head_zeroinit=False),
                            text_model="proj.flaxformer.bert", text=dict(config=b["config"], head_zeroinit=False),
                            out_dim=(None, WIDTH), temperature_init=10.0, bias_init=-2.71),
              desc=f"SigLiT of siglip_lit_coco.py txt={txt}: ViT-B/16 (tok pool, no head) FROZEN + BERT-"
                   f"{b['config']} trained ({BERT_TOKENS} zero-padded tokens), 224x224, {b['optax_name']}, "
                   "full update_fn")


def _bert_batch(orig):
  """bench.synthetic_batch with BERT's token ids: a first token, then ids in [1, 30522) for a random length,
  zero-padded to 16 (pp/proj/flaxformer/bert_ops.py:77-83)."""
  import numpy as np

  def batch(wl, n, seed, uint8=False):
    out = orig(wl, n, seed, uint8)
    rng = np.random.default_rng(seed + 1)
    text = np.zeros((n, BERT_TOKENS), dtype=np.int32)
    lens = rng.integers(4, BERT_TOKENS + 1, size=n)
    for i in range(n):
      text[i, :lens[i]] = rng.integers(1, 30_522, size=lens[i])
    out["labels"] = text
    return out
  return batch


def register(per_gpu_batch=768, txt=None):
  if txt is None:
    bench.WORKLOADS[NAME] = dict(WORKLOAD, flops=pair_flops(per_gpu_batch))
    bench.OPT_CONFIG["schedule"] = LIT_SCHEDULE
    return bench.WORKLOADS[NAME]
  # the config's optimizer as written (optax defaults, no bf16 moments), in this process only
  bench.TXT_LEN = BERT_TOKENS
  bench.synthetic_batch = _bert_batch(bench.synthetic_batch)
  bench.OPT_CONFIG.clear()
  bench.OPT_CONFIG.update(optax_name=BERT[txt]["optax_name"], optax={}, lr=1e-3, wd=0.01, grad_clip_norm=1.0,
                          schedule=[("img/.*", None), (".*", dict(decay_type="cosine", warmup_steps=150))])
  bench.WORKLOADS[NAME] = bert_workload(txt)
  return bench.WORKLOADS[NAME]


def run_one(args):
  """One arm in this process: bench.main's JSON line, plus the card's memory."""
  import torch
  n = args.per_gpu_batch or WORKLOAD["per_gpu_batch"]
  register(n, args.txt)
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
                 "--steps", str(args.steps), "--warmup", str(args.warmup)] + (["--txt", args.txt] if args.txt else []))


def run_torch_bert(args):
  """The stand-in: baseline/torch_gpu.py's ViT-B/16 ([cls] pool, no head) frozen under no_grad, and
  transformers.BertModel (random weights from a BertConfig: gelu_new, LayerNorm eps 1e-12, no dropout) with a
  Linear head, bf16 autocast, sigmoid loss, AdamW lr 1e-3 / wd 0.01, clip 1."""
  import math
  import torch
  from transformers import BertConfig, BertModel
  from baseline import torch_gpu as TG
  b, n = BERT[args.txt], args.per_gpu_batch
  torch.manual_seed(0)
  img = TG.ViT("B/16", RES, None, pool="tok").cuda().to(memory_format=torch.channels_last).requires_grad_(False)
  conf = BertConfig(vocab_size=30_522, hidden_size=b["width"], num_hidden_layers=b["depth"],
                    num_attention_heads=b["heads"], intermediate_size=b["mlp"], hidden_act="gelu_new",
                    layer_norm_eps=1e-12, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
  txt = BertModel(conf, add_pooling_layer=False).cuda()
  head = torch.nn.Linear(b["width"], WIDTH).cuda()
  t = torch.nn.Parameter(torch.tensor([math.log(10.0)], device="cuda"))
  bias = torch.nn.Parameter(torch.tensor([-2.71], device="cuda"))
  params = list(txt.parameters()) + list(head.parameters()) + [t, bias]
  opt = torch.optim.AdamW(params, lr=1e-3, weight_decay=0.01, fused=True)
  host = _bert_batch(bench.synthetic_batch)(dict(bench.WORKLOADS["siglip_b16"]), n, 0)
  image, text = torch.from_numpy(host["image"]).cuda(), torch.from_numpy(host["labels"]).cuda()

  def step():
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
      with torch.no_grad():
        zi = img(image).float()
      h = txt(input_ids=text, attention_mask=(text != 0).long()).last_hidden_state[:, 0]
      zt = head(h).float()
    zi = zi / (zi.norm(dim=-1, keepdim=True) + 1e-8)
    zt = zt / (zt.norm(dim=-1, keepdim=True) + 1e-8)
    loss = TG.siglip_loss(zi, zt, t, bias, 0, n)
    loss.backward()
    torch.nn.utils.clip_grad_norm_(params, 1.0, foreach=True)
    opt.step()
    return loss.detach()

  for _ in range(args.warmup):
    step()
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(args.steps):
    loss = step()
  e1.record()
  torch.cuda.synchronize()
  ms = e0.elapsed_time(e1) / args.steps
  print(json.dumps({"impl": "transformers.BertModel + baseline ViT (bf16 autocast)", "per_gpu_batch": n,
                    "value": n / ms * 1e3, "ms_per_step": ms, "final_loss": float(loss),
                    "peak_mem_gib": torch.cuda.max_memory_allocated() / 2**30}), flush=True)


def run_attention(args):
  """Masked against unmasked attention, forward + backward, at the BERT shapes (B x heads, N = 16; the
  caption-length mask of the batch) and at N = 128 with random masks (60 % of the keys attended)."""
  import numpy as np
  import torch
  from big_vision_b200 import ops
  b, n = BERT[args.txt], args.per_gpu_batch
  out = {}
  for N, kind in ((BERT_TOKENS, "captions"), (128, "random")):
    rng = np.random.default_rng(N)
    d = b["heads"] * 64
    qkv = torch.from_numpy(rng.standard_normal((n, N, 3 * d), dtype=np.float32)).cuda().bfloat16()
    do = torch.from_numpy(rng.standard_normal((n, N, d), dtype=np.float32)).cuda().bfloat16()
    if kind == "captions":
      lens = rng.integers(4, N + 1, size=n)
      mask = np.arange(N)[None, :] < lens[:, None]
    else:
      mask = rng.random((n, N)) < 0.6
      mask[:, 0] = True
    mask = torch.from_numpy(mask.astype(np.uint8)).cuda()
    q, k, v = qkv[:, :, :d], qkv[:, :, d:2 * d], qkv[:, :, 2 * d:]
    row = {}
    for label, m in (("unmasked", None), ("masked", mask)):
      kw = {} if m is None else {"key_mask": m}

      def call():
        o, lse = ops.attention_fwd(q, k, v, b["heads"], **kw)
        ops.attention_bwd(do, q, k, v, o, lse, b["heads"], **kw)
      times = []
      for rep in range(args.repeats + 1):
        for _ in range(3):
          call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
          call()
        e1.record()
        torch.cuda.synchronize()
        if rep:
          times.append(e0.elapsed_time(e1) / 50 * 1e3)
      row[label + "_us"] = statistics.median(times)
      row[label + "_runs_us"] = times
    row["masked_over_unmasked"] = row["masked_us"] / row["unmasked_us"]
    out[f"B{n}xH{b['heads']}_N{N}_{kind}"] = row
  print(json.dumps(out), flush=True)


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


def _card():
  """The card's name and power limit, read in the same run as the numbers they qualify."""
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
  return out.stdout.strip() or f"unavailable: {out.stderr.strip()[-200:]}"


def suite(args):
  wl = bert_workload(args.txt) if args.txt else WORKLOAD
  result = {"metric": wl["metric"], "unit": "pairs/s", "workload": f"{NAME}: {wl['desc']}",
            "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "card": _card(), "lit": {}}
  batches = [b for b in (args.per_gpu_batch or ("512,max" if args.txt else "768,max")).split(",") if b]
  probe = {}
  lo = BERT_BATCH if args.txt else 768
  if "max" in batches:
    # peak = fixed + per_pair * n: two points give the line, the card's memory the largest n
    for n in (lo, 2 * lo):
      probe[n] = _ours(args, n)
    a, b = probe[lo], probe[2 * lo]
    if "config" in a and "config" in b:
      per_pair = (b["config"]["peak_mem_gib"] - a["config"]["peak_mem_gib"]) / lo
      fixed = a["config"]["peak_mem_gib"] - lo * per_pair
      budget = 0.97 * a["total_mem_gib"]
      n_max = int((budget - fixed) / per_pair) // 128 * 128
      if args.txt and n_max > BERT_MAX_BATCH:
        # the frozen image tower and 16 text tokens leave most of the card free; the host-side synthetic
        # batch (600 KB of fp32 pixels per pair) bounds the search instead
        result["max_batch_fit"] = {"capped_from": n_max}
        n_max = BERT_MAX_BATCH
      result["max_batch_fit"] = dict(result.get("max_batch_fit", {}), gib_per_pair=per_pair, fixed_gib=fixed,
                                     budget_gib=budget, per_gpu_batch=n_max)
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
  if args.txt:
    if not args.no_gpu_baseline:
      result[f"gpu_baseline_transformers_bert_{BERT_BATCH}"] = _child(
          [sys.executable, os.path.abspath(__file__), "--impl", "torch_bert", "--txt", args.txt, "--per-gpu-batch",
           str(BERT_BATCH), "--steps", str(args.steps), "--warmup", str(args.warmup)])
    result["attention_masked_vs_unmasked"] = _child(
        [sys.executable, os.path.abspath(__file__), "--impl", "attn", "--txt", args.txt, "--per-gpu-batch",
         str(BERT_BATCH), "--repeats", str(args.repeats)])
    print(json.dumps(result), flush=True)
    return
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
  ap.add_argument("--per-gpu-batch", default=None,
                  help="comma list of per-GPU batches (suite; default 768,max, or 512,max with --txt) or one batch "
                       "(the single-arm impls)")
  ap.add_argument("--impl", default="suite", choices=["suite", "ours", "torch_gpu", "torch_bert", "attn"])
  ap.add_argument("--txt", default=None, choices=sorted(BERT),
                  help="the text tower of siglip_lit_coco.py (default: the siglip_b16 text-B tower)")
  ap.add_argument("--no-gpu-baseline", action="store_true")
  ap.add_argument("--no-full", action="store_true", help="skip the full-step bench.py runs")
  args = ap.parse_args()
  if args.impl == "suite":
    suite(args)
    return
  args.per_gpu_batch = int(args.per_gpu_batch or (BERT_BATCH if args.txt else WORKLOAD["per_gpu_batch"]))
  if args.impl in ("torch_bert", "attn") and not args.txt:
    ap.error(f"--impl {args.impl} needs --txt")
  {"torch_bert": run_torch_bert, "attn": run_attention}.get(args.impl, run_one)(args)


if __name__ == "__main__":
  main()
