"""Launches every kernel of the hot path once or twice at bench-like shapes, so that one profiler pass
(for example `ncu --set full python tools/kernel_zoo.py`) captures all of them.  Not a benchmark: no
timing here."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from big_vision_b200 import lib as L, ops

dev = "cuda"
bf = torch.bfloat16
g = torch.Generator(device=dev).manual_seed(0)
rn = lambda *s, dt=bf, sc=1.0: (torch.randn(*s, device=dev, generator=g) * sc).to(dt)
n, N, d, m, H = 256, 196, 768, 3072, 12
M = n * N
x, w_dm, w_md = rn(M, d), rn(d, m, sc=0.03), rn(m, d, sc=0.03)
b_m, b_d = rn(m, dt=torch.float32), rn(d, dt=torch.float32)
for _ in range(2):
  act, pre = ops.gemm(x, w_dm, b_mn=True, bias=b_m, epilogue=L.EPI_BIAS_GELU)                  # gelu pair
  y = ops.gemm(act, w_md, b_mn=True, bias=b_d, aux=x, epilogue=L.EPI_BIAS_RESID)             # bias + residual
  dact = ops.gemm(y, w_md, aux=pre, epilogue=L.EPI_DGELU, colsum=torch.zeros(m, device=dev))   # gelu'
  dx = ops.gemm(dact, w_dm)                                                                    # plain dgrad
  ops.gemm(x, dact, a_mn=True, b_mn=True, out=torch.zeros(d, m, device=dev), reduce_out=True)  # wgrad, split-K
  qkv = ops.gemm(x, rn(d, 3 * d, sc=0.03), b_mn=True, bias=rn(3 * d, dt=torch.float32))        # bias
  q3 = qkv.view(n, N, 3 * d)
  o, lse = ops.attention_fwd(q3[:, :, 0:d], q3[:, :, d:2 * d], q3[:, :, 2 * d:], H)
  dq3 = torch.empty_like(q3)
  ops.attention_bwd(rn(n, N, d), q3[:, :, 0:d], q3[:, :, d:2 * d], q3[:, :, 2 * d:], o, lse, H,
                    dq=dq3[:, :, 0:d], dk=dq3[:, :, d:2 * d], dv=dq3[:, :, 2 * d:])
  # config-5 shape through the streaming kernels
  ql = rn(32, 576, 3 * 1024)
  ol, lsel = ops.attention_fwd(ql[:, :, 0:1024], ql[:, :, 1024:2048], ql[:, :, 2048:], 16)
  dql = torch.empty_like(ql)
  ops.attention_bwd(rn(32, 576, 1024), ql[:, :, 0:1024], ql[:, :, 1024:2048], ql[:, :, 2048:], ol, lsel, 16,
                    dq=dql[:, :, 0:1024], dk=dql[:, :, 1024:2048], dv=dql[:, :, 2048:])
  sc, bi = torch.ones(d, device=dev), torch.zeros(d, device=dev)
  ln, mean, rstd = ops.layernorm_fwd(x, sc, bi)
  ops.layernorm_bwd(y, x, sc, mean, rstd, dres=y, dscale=torch.zeros(d, device=dev), dbias=torch.zeros(d, device=dev),
                    dx_colsum=torch.zeros(d, device=dev))
  x1k = rn(n * 576 // 4, 1024)
  l1k, m1k, r1k = ops.layernorm_fwd(x1k, torch.ones(1024, device=dev), torch.zeros(1024, device=dev))
  ops.layernorm_bwd(x1k, x1k, torch.ones(1024, device=dev), m1k, r1k, dres=x1k)
  dots = rn(1024, 8192, dt=torch.float32, sc=0.3)
  t, b, scal = torch.tensor([2.3], device=dev), torch.tensor([-10.0], device=dev), torch.zeros(4, device=dev)
  ops.siglip_loss(dots, 0, t, b, 8192, scal[0:1], scal[1:2], scal[2:3])
  ops.softmax_contrastive_loss(dots, 0, t, 8192, 0.5, scal[0:1], scal[1:2], scal[2:3])
  lg = rn(n, 1000, dt=torch.float32)
  lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (n,), device=dev), 1000).float()
  ops.sigmoid_xent(lg, lab, scal[0:1]); ops.softmax_xent(lg, lab, scal[0:1])
  P = 50_000_000
  p32, g32 = rn(P, dt=torch.float32), rn(P, dt=torch.float32, sc=0.01)
  ops.sumsq(g32, scal[0:1])
  ops.adam_step(p32, g32, torch.zeros(P, dtype=bf, device=dev), torch.zeros(P, device=dev), torch.empty(P, dtype=bf, device=dev),
                lr_eff=1e-3, b1=0.9, b2=0.95, eps=1e-8, wd_eff=1e-4, step=1, clip_norm=1.0, gnorm_sq=scal[0:1],
                upd_sq=scal[1:2], param_sq=scal[2:3])
  img = rn(n, 224, 224, 3, dt=torch.float32).clamp(-1, 1)
  ops.patchify(img, 16)
  ops.patchify(torch.randint(0, 256, (n, 224, 224, 3), dtype=torch.uint8, device=dev), 16)
  ids = torch.randint(0, 32000, (1024, 64), dtype=torch.int32, device=dev)
  tab, pos = rn(32000, d, dt=torch.float32), rn(64, d, dt=torch.float32)
  e = ops.embed_fwd(ids, tab, pos)
  ops.embed_bwd(ids, e, torch.zeros_like(tab), torch.zeros_like(pos))
  ops.colsum(x, torch.zeros(d, device=dev))
  ops.cast(p32[:10_000_000], torch.empty(10_000_000, dtype=bf, device=dev))
  z, nrm = ops.l2norm_fwd(rn(1024, d, dt=torch.float32))
  ops.l2norm_bwd(z, z, nrm)
  pl = ops.pool_fwd(x, n, N, 0, out_dtype=torch.float32)
  ops.pool_bwd(pl, n, N, 0)
  pm = ops.pool_fwd(x, n, N, 2)
  ops.pool_max_bwd(pm, x, n, N)
  ops.mixup(img, 0.7)
  ops.row_select(x, y, (torch.rand(n, device=dev) > 0.1).float(), n, N)
  yt = ops.transpose_tokens(x, n, N, d)
  ops.untranspose_add(yt, x, n, N, d)
  ops.top1(lg, lab)
  ops.retrieval_ranks(rn(1000, 5000, dt=torch.float32), torch.randint(0, 1000, (5000,), device=dev))
torch.cuda.synchronize()
print("zoo done, launches:", L.LAUNCHES[0])
