"""Times bv_attention_fwd_hd / bwd_hd at the bench shapes with CUDA events (after warm-up):
  python tools/attn_bench.py [fwd|bwd|both] [--head-dim DH] [--dump DIR]
env BV_BENCH_SHAPES="B,H,N;..." overrides the shapes.
FLOPs are counted with the real head dim DH (default 64), not the k16-padded one the kernels compute.
The byte bound is the least HBM traffic of the call (q, k, v, o, dO read once and dq, dk, dv written once
in the backward; q, k, v read and o written in the forward; lse either way) at the H100 SXM data
sheet's 3.35 TB/s.
--dump DIR writes each shape's backward outputs (dq, dk, dv and their fused column sums, from seeded
inputs) to DIR/attn_bwd_B{B}_H{H}_N{N}_dh{DH}.pt, so that two builds of the library (BV_LIB_PATH) can be
compared bit for bit."""
import os
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from big_vision_b200 import ops

HBM_BYTES_PER_S = 3.35e12


def run(B, H, N, what, iters=10, dh=64, dump=None):
  d = H * dh
  g = torch.Generator(device="cuda").manual_seed(B * 1000 + N + dh)
  qkv = torch.randn(B, N, 3 * d, device="cuda", generator=g).to(torch.bfloat16)
  do = torch.randn(B, N, d, device="cuda", generator=g).to(torch.bfloat16)
  q, k, v = qkv[:, :, 0:d], qkv[:, :, d:2 * d], qkv[:, :, 2 * d:]
  o, lse = ops.attention_fwd(q, k, v, H)
  dqkv = torch.empty_like(qkv)
  fb = lambda: ops.attention_bwd(do, q, k, v, o, lse, H, dq=dqkv[:, :, 0:d], dk=dqkv[:, :, d:2 * d], dv=dqkv[:, :, 2 * d:])
  ff = lambda: ops.attention_fwd(q, k, v, H)
  if dump:
    cs = torch.zeros(3, d, device="cuda")
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, H, dq_colsum=cs[0], dk_colsum=cs[1], dv_colsum=cs[2])
    torch.save({"dq": dq.cpu(), "dk": dk.cpu(), "dv": dv.cpu(), "colsum": cs.cpu()},
               os.path.join(dump, f"attn_bwd_B{B}_H{H}_N{N}_dh{dh}.pt"))
  tensor_bytes, lse_bytes = B * N * d * 2, B * H * N * 4
  out = {}
  for name, fn, fl, nbytes in (("fwd", ff, 4, 4 * tensor_bytes + lse_bytes),
                               ("bwd", fb, 10, 8 * tensor_bytes + lse_bytes)):
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
    out[name] = (ms, fl * B * H * N * N * dh / ms * 1e-9, nbytes / HBM_BYTES_PER_S * 1e3)
  return out


args = sys.argv[1:]
dh = 64
if "--head-dim" in args:
  i = args.index("--head-dim")
  dh = int(args[i + 1])
  del args[i:i + 2]
dump = None
if "--dump" in args:
  i = args.index("--dump")
  dump = args[i + 1]
  del args[i:i + 2]
  os.makedirs(dump, exist_ok=True)
what = args[0] if args else "both"
shapes = ((1024, 12, 196), (1024, 12, 64), (256, 12, 197), (512, 16, 576))
if os.environ.get("BV_BENCH_SHAPES"):
  shapes = tuple(tuple(int(x) for x in sh.split(",")) for sh in os.environ["BV_BENCH_SHAPES"].split(";"))
for B, H, N in shapes:
  r = run(B, H, N, what, dh=dh, dump=dump)
  print(f"B={B} H={H} N={N} dh={dh} " +
        "  ".join(f"{k}: {v[0]:.3f} ms {v[1]:.0f} TFLOP/s (byte bound {v[2]:.3f} ms, {v[2] / v[0]:.0%})"
                  for k, v in r.items()), flush=True)
