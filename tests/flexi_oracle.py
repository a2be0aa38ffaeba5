"""TEST INFRASTRUCTURE: the FlexiViT forward (big_vision/models/proj/flexi/vit.py) in float64 on torch-CPU
autograd, on top of oracle/bv_oracle.py's ViT.  The two resize matrices are built here independently of the
library: by resizing one-hot basis images with torch's F.interpolate (bilinear, half-pixel centres), without
antialias for the patch-embedding kernel (tf.image.resize "bilinear") and with it for the position embedding
(jax.image.resize "linear").  The flexi forward is then the ViT forward with the resampled kernel and
position embedding in place of the stored ones (flexi/vit.py:73-103, 131-141)."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import bv_oracle as O

F64 = torch.float64


def resize_matrix(n_in, n_out, antialias):
  """[n_out^2, n_in^2]: the bilinear resize of n_in x n_in images to n_out x n_out (row-major pixels)."""
  eye = torch.eye(n_in * n_in, dtype=F64).view(-1, 1, n_in, n_in)
  out = F.interpolate(eye, size=(n_out, n_out), mode="bilinear", align_corners=False, antialias=antialias)
  return out.reshape(n_in * n_in, n_out * n_out).T.contiguous()


def patch_matrix(p0, p):
  """pinv(R^T) of flexi/vit.py:59-66 for R the patch resize p0 -> p."""
  return torch.linalg.pinv(resize_matrix(p0, p, antialias=False).T)


def resample_kernel(kernel, p):
  """kernel [p0, p0, C, d] -> [p, p, C, d] (flexi/vit.py:68-71); unchanged at p == p0."""
  p0, _, C, d = kernel.shape
  if p == p0:
    return kernel
  return (patch_matrix(p0, p) @ kernel.reshape(p0 * p0, C * d)).reshape(p, p, C, d)


def resample_posemb(pe, posemb_size, seqhw):
  """pe [1, gh * gw, d] -> [1, seqhw^2, d] (flexi/vit.py:135-139); unchanged when the grid already fits."""
  if (seqhw, seqhw) == tuple(posemb_size):
    return pe
  assert posemb_size[0] == posemb_size[1]
  return (resize_matrix(posemb_size[0], seqhw, antialias=True) @ pe.reshape(-1, pe.shape[-1]))[None]


def flexi_forward(p, image, cfg, seqhw, mm="float32"):
  """flexi _Model.__call__ at `seqhw`.  cfg: dict(depth, num_heads, pool_type, posemb, posemb_size,
  num_classes); p: flat dict of float64 tensors with the reference names."""
  H = image.shape[1]
  kernel = p["embedding/kernel"]
  d = kernel.shape[-1]
  q = dict(p)
  q["embedding/kernel"] = resample_kernel(kernel, H // seqhw)
  if cfg.get("posemb", "learn") == "learn":
    pe = p["pos_embedding"]
  else:     # vit.get_posemb(..., "sincos2d", posemb_size): a fixed table at the base grid, then resized
    pe = torch.from_numpy(O.posemb_sincos_2d(*cfg["posemb_size"], d)).to(F64)
  q["pos_embedding"] = resample_posemb(pe, cfg["posemb_size"], seqhw)
  return O.vit_forward(q, image, {**cfg, "posemb": "learn", "rep_size": False}, mm)


def value_and_grad(np_tree, image, labels, cfg, seqhw, loss="sigmoid_xent", mm="float32"):
  """(loss, {name: float64 numpy gradient}) of the mean classification loss on the global batch."""
  p = O.to_f64_tree(np_tree, requires_grad=True)
  logits = flexi_forward(p, torch.as_tensor(np.asarray(image)), cfg, seqhw, mm)
  loss_fn = O.sigmoid_xent if loss == "sigmoid_xent" else O.softmax_xent
  val = loss_fn(logits, torch.as_tensor(np.asarray(labels)).to(F64))
  val.backward()
  return float(val.detach()), {k: (v.grad.numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in p.items()}
