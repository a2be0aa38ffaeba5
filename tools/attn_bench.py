"""Times bv_attention_fwd / bwd at the bench shapes with CUDA events (after warm-up):
  python tools/attn_bench.py [fwd|bwd|both] [--head-dim DH]      env BV_BENCH_SHAPES="B,H,N;..." overrides the shapes.
FLOPs are counted with the real head dim DH (default 64), not the k16-padded one the kernels compute."""
import os
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from big_vision_b200 import ops

def run(B, H, N, what, iters=10, dh=64):
  d = H * dh
  qkv = (torch.randn(B, N, 3 * d, device="cuda") * 1.0).to(torch.bfloat16)
  do = torch.randn(B, N, d, device="cuda").to(torch.bfloat16)
  q, k, v = qkv[:, :, 0:d], qkv[:, :, d:2 * d], qkv[:, :, 2 * d:]
  o, lse = ops.attention_fwd(q, k, v, H)
  dqkv = torch.empty_like(qkv)
  fb = lambda: ops.attention_bwd(do, q, k, v, o, lse, H, dq=dqkv[:, :, 0:d], dk=dqkv[:, :, d:2 * d], dv=dqkv[:, :, 2 * d:])
  ff = lambda: ops.attention_fwd(q, k, v, H)
  out = {}
  for name, fn, fl in (("fwd", ff, 4), ("bwd", fb, 10)):
    if what not in (name, "both"):
      continue
    for _ in range(3):
      fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
      fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    out[name] = (ms, fl * B * H * N * N * dh / ms * 1e-9)
  return out

args = sys.argv[1:]
dh = 64
if "--head-dim" in args:
  i = args.index("--head-dim")
  dh = int(args[i + 1])
  del args[i:i + 2]
what = args[0] if args else "both"
shapes = ((1024, 12, 196), (1024, 12, 64), (256, 12, 197), (512, 16, 576))
if os.environ.get("BV_BENCH_SHAPES"):
  shapes = tuple(tuple(int(x) for x in sh.split(",")) for sh in os.environ["BV_BENCH_SHAPES"].split(";"))
for B, H, N in shapes:
  r = run(B, H, N, what, dh=dh)
  print(f"B={B} H={H} N={N} dh={dh} " + "  ".join(f"{k}: {v[0]:.3f} ms {v[1]:.0f} TFLOP/s" for k, v in r.items()),
        flush=True)
