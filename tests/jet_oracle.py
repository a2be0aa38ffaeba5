"""TEST INFRASTRUCTURE: the Jet flow (big_vision/models/proj/jet/jet.py, trainers/proj/jet/train.py) in float64
on torch-CPU autograd, on top of oracle/bv_oracle.py's ViT encoder.  The masks are applied as MATRICES with
einsum, as the reference does, so the library's gather tables are checked independently of how they were
derived.  Parameters are a flat dict of reference names ("couplings/dnn/init_proj/kernel", ...), every
`couplings/` leaf with its leading depth axis."""
import itertools
import math

import numpy as np
import torch

from oracle import bv_oracle as O

F64 = torch.float64
CH, SP = "channel_coupling_masks-FREEZE_ME", "spatial_coupling_masks-FREEZE_ME"


def kinds_of(depth, kinds, channels_coupling_projs, spatial_coupling_projs):
  """1 (channels) or 0 (spatial) per coupling: the kinds cycle through `kinds`."""
  return [1 if k == "channels" else 0 for k in itertools.islice(itertools.cycle(kinds), depth)]


def patchify(image, ps):
  """b (h hp) (w wp) c -> b (h w) (hp wp c)."""
  n, H, W, C = image.shape
  x = image.reshape(n, H // ps, ps, W // ps, ps, C).permute(0, 1, 3, 2, 4, 5)
  return x.reshape(n, (H // ps) * (W // ps), ps * ps * C)


def unpatchify(x, image_shape, ps):
  n, H, W, C = image_shape
  x = x.reshape(n, H // ps, W // ps, ps, ps, C).permute(0, 1, 3, 2, 4, 5)
  return x.reshape(n, H, W, C)


def split(x, kind, cm, sm):
  """x [n, T, 2c] -> (x1, x2) of [n, T, c] each."""
  if kind == 1:
    y = torch.einsum("ntk,km->ntm", x, cm)
    return y.chunk(2, dim=-1)
  y = torch.einsum("ntk,tm->nmk", x, sm)
  n, T, dt = y.shape
  return tuple(h.reshape(n, T, dt // 2) for h in y.chunk(2, dim=1))      # n (s c) -> (n s) c, s = 2


def merge(x1, x2, kind, cm, sm):
  if kind == 1:
    return torch.einsum("ntk,km->ntm", torch.cat([x1, x2], -1), cm.T)
  n, T, c = x1.shape
  y = torch.cat([x1.reshape(n, T // 2, 2 * c), x2.reshape(n, T // 2, 2 * c)], dim=1)
  return torch.einsum("ntk,tm->nmk", y, sm.T)


def coupling_params(p, i):
  """Slice i of every `couplings/dnn/` leaf, named relative to `couplings/dnn/`."""
  pre = "couplings/dnn/"
  return {k[len(pre):]: v[i] for k, v in p.items() if k.startswith(pre)}


def dnn(x1, q, block_depth, heads, mm):
  """jet.py:34-65 -> (bias, raw) of [n, T, c]."""
  h = O.dense(x1, q["init_proj/kernel"], q["init_proj/bias"], mm) + O.rnd(q["posemb"], mm)
  h = O.rnd(h, mm)
  enc = O.rnd(O.encoder(h, O.sub(q, "vit/"), block_depth, heads, mm), mm)
  out = O.dense(enc, q["final_proj/kernel"], q["final_proj/bias"], mm)
  return out.chunk(2, dim=-1)


def _coupling(p, x, i, kind, cfg, inverse, mm):
  x1, x2 = split(x, kind, p[CH][i], p[SP][i])
  bias, raw = dnn(x1, coupling_params(p, i), cfg["block_depth"], cfg["num_heads"], mm)
  sf = cfg.get("scale_factor", 2.0)
  s = torch.sigmoid(raw) * sf
  ld = (torch.nn.functional.logsigmoid(raw) + math.log(sf)).sum(dim=(1, 2))
  x2 = x2 / s - bias if inverse else (x2 + bias) * s
  return merge(x1, x2, kind, p[CH][i], p[SP][i]), (-ld if inverse else ld)


def forward(p, image, cfg, mm="float32"):
  """jet.py:232-246 -> (z [n, H, W, C], logdet [n]).  cfg: depth, block_depth, num_heads, ps, kinds
  (scale_factor)."""
  x = patchify(image, cfg["ps"])
  logdet = torch.zeros(image.shape[0], dtype=image.dtype)
  for i, kind in enumerate(kinds_of(cfg["depth"], cfg["kinds"], (), ())):
    x, ld = _coupling(p, x, i, kind, cfg, False, mm)
    logdet = logdet + ld
  return unpatchify(x, image.shape, cfg["ps"]), logdet


def inverse(p, z, cfg, mm="float32"):
  """jet.py:248-262: the couplings in reverse order, each inverted."""
  x = patchify(z, cfg["ps"])
  logdet = torch.zeros(z.shape[0], dtype=z.dtype)
  kinds = kinds_of(cfg["depth"], cfg["kinds"], (), ())
  for i in reversed(range(cfg["depth"])):
    x, ld = _coupling(p, x, i, kinds[i], cfg, True, mm)
    logdet = logdet + ld
  return unpatchify(x, z.shape, cfg["ps"]), logdet


def bits_per_dim(z, logdet):
  """train.py:272-285 with reduce=False -> (bits, nll, logdet) per example, each / (D ln 2)."""
  D = z[0].numel()
  nll = (0.5 * z * z + 0.5 * math.log(2 * math.pi) + math.log(127.5)).reshape(z.shape[0], -1).sum(1)
  norm = math.log(2) * D
  return (nll - logdet) / norm, nll / norm, logdet / norm


def value_and_grad(np_tree, images, cfg, mm="float32"):
  """(mean bits, per-example (bits, nll, logdet), z, {name: float64 numpy gradient}) of the training loss on
  `images` (already dequantized).  The masks get no gradient (they are frozen)."""
  p = O.to_f64_tree({k: v for k, v in np_tree.items() if k not in (CH, SP)}, requires_grad=True)
  p.update(O.to_f64_tree({k: np_tree[k] for k in (CH, SP)}))
  z, logdet = forward(p, torch.as_tensor(np.asarray(images)).to(F64), cfg, mm)
  bits, nll, ld = bits_per_dim(z, logdet)
  loss = bits.mean()
  loss.backward()
  grads = {k: (v.grad.numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in p.items()}
  rows = np.stack([t.detach().numpy() for t in (bits, nll, ld)])
  return float(loss.detach()), rows, z.detach().numpy(), grads
