"""float64 restatement of big_vision/models/bit_paper.py in torch (CPU), over a flat {name: array} tree of
the reference's names.  Line numbers cite the reference file.

With bf16=True the forward rounds to bf16 where the kernels store bf16 (the stem's patches, the standardised
kernels, every convolution and GroupNorm + ReLU output; a residual sum after its convolution output is
rounded), passing the gradient straight through each rounding.  Its ReLU and max-pool decisions are then the
kernels', so its gradients differ from theirs by accumulation order and gradient rounding only."""
import numpy as np
import torch
import torch.nn.functional as F


def block_desc(depth):
  if isinstance(depth, list):
    depth = tuple(depth)
  return {26: [2, 2, 2, 2], 50: [3, 4, 6, 3], 101: [3, 4, 23, 3], 152: [3, 8, 36, 3],
          200: [3, 24, 36, 3]}.get(depth, depth)


BF16 = [False]


def rnd(x):
  """x rounded to bf16 in the forward (bf16 mode), the identity in the backward."""
  if not BF16[0]:
    return x
  return x + (x.to(torch.bfloat16).to(torch.float64) - x).detach()


def standardize(x, axis, eps):                          # :29-32
  x = x - x.mean(dim=axis, keepdim=True)
  return x / torch.sqrt((x * x).mean(dim=axis, keepdim=True) + eps)


def group_norm(x, scale, bias, ngroups=32):             # :37-58 (NHWC)
  n, h, w, c = x.shape
  g = standardize(x.reshape(n, h, w, ngroups, c // ngroups), axis=(1, 2, 4), eps=1e-5).reshape(n, h, w, c)
  return g * scale + bias


def std_conv(x, kernel, stride, pad):                    # :61-67 (StdConv), flax nn.Conv with explicit padding
  k = rnd(standardize(kernel, axis=(0, 1, 2), eps=1e-10))
  y = F.conv2d(x.permute(0, 3, 1, 2), k.permute(3, 2, 0, 1), stride=stride, padding=pad)
  return rnd(y.permute(0, 2, 3, 1))


def gn_relu(x, scale, bias):
  return rnd(torch.relu(group_norm(x, scale, bias)))


def max_pool(x):                                         # :78 nn.max_pool(x, (3, 3), (2, 2), padding 1) pads -inf
  return F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, padding=1).permute(0, 2, 3, 1)


def unit(p, x, pre, stride):                             # :83-111
  nout = p[pre + "conv3/kernel"].shape[-1]
  residual = x
  x = gn_relu(x, p[pre + "gn1/scale"], p[pre + "gn1/bias"])
  if pre + "conv_proj/kernel" in p:
    residual = std_conv(x, p[pre + "conv_proj/kernel"], stride, 0)
  x = std_conv(x, p[pre + "conv1/kernel"], 1, 0)
  x = gn_relu(x, p[pre + "gn2/scale"], p[pre + "gn2/bias"])
  x = std_conv(x, p[pre + "conv2/kernel"], stride, 1)
  x = gn_relu(x, p[pre + "gn3/scale"], p[pre + "gn3/bias"])
  x = std_conv(x, p[pre + "conv3/kernel"], 1, 0)
  assert x.shape[-1] == nout
  return rnd(x + residual)


def forward(p, image, depth):
  """p: {name: float64 tensor}; image NHWC.  -> logits (or pre_logits without a head)  (:122-156)."""
  x = max_pool(std_conv(rnd(image), p["root_block/conv_root/kernel"], 2, 3))   # :76-78
  for b, size in enumerate(block_desc(depth)):                                 # :132-137
    for u in range(size):
      x = unit(p, x, f"block{b + 1}/unit{u + 1:02d}/", 2 if (b > 0 and u == 0) else 1)
  x = gn_relu(x, p["norm-pre-head/scale"], p["norm-pre-head/bias"])              # :144-145
  x = x.mean(dim=(1, 2))                                                        # :146
  if "head/kernel" in p:
    x = rnd(x) @ rnd(p["head/kernel"]) + p["head/bias"]                         # :149-154
  return x


def value_and_grads(tree, image, depth, dlogits, bf16=False):
  """(logits, {name: gradient of <logits, dlogits>}) in float64 (bf16: with the kernels' roundings)."""
  BF16[0] = bf16
  try:
    return _value_and_grads(tree, image, depth, dlogits)
  finally:
    BF16[0] = False


def _value_and_grads(tree, image, depth, dlogits):
  p = {k: torch.tensor(np.asarray(v), dtype=torch.float64, requires_grad=True) for k, v in tree.items()}
  out = forward(p, torch.as_tensor(np.asarray(image), dtype=torch.float64), depth)
  grads = torch.autograd.grad(out, list(p.values()), torch.as_tensor(np.asarray(dlogits), dtype=torch.float64))
  return out.detach().numpy(), {k: g.numpy() for k, g in zip(p, grads)}
