"""TEST INFRASTRUCTURE: one float64 reference per kind of backward stage (engine.Stage) of the models, built
from oracle/bv_oracle.py's pieces with mm="float32" (plain high-precision math).  Each function takes the
stage's input and its parameters, `p`: a dict of float64 tensors under the reference names relative to the
stage's root (the stage's own prefix, or the model prefix for the embeddings), and returns the stage's output;
torch autograd then gives d input and the parameter gradients under the same names.

Chained bottom-up they are the whole models of the oracle (tests/test_stage_oracle.py checks that), so a stage
checked against its reference on the inputs the CUDA path actually gave it is checked against the pinned
oracle, one stage at a time."""
import torch

import flexi_oracle as FO
from oracle import bv_oracle as O

MM = "float32"


def patch_embedding(image, p, name, pos=None, cls=False):
  """vit.PatchEmbedding (and the MLP-Mixer's stem): image [n, H, W, C] -> [n, N, d].  p: `name`/kernel
  [ph, pw, C, d], `name`/bias, and `cls` [1, 1, d] with `cls`; `pos`: the [N0, d] position table added to
  every image (None: no position embedding)."""
  x = O.patch_embed(image, p[name + "/kernel"], p[name + "/bias"], MM)
  if pos is not None:
    x = x + pos.reshape(x.shape[1:])
  if cls:
    x = torch.cat([p["cls"].expand(x.shape[0], -1, -1), x], dim=1)
  return x


def flexi_patch_embedding(image, p, seqhw, posemb_size, pos=None, cls=False):
  """FlexiPatchEmbedding at `seqhw`: the kernel resampled to patch H // seqhw and the [gh * gw, d] table `pos`
  (the learned one, or the fixed sincos table) resized to seqhw x seqhw, by tests/flexi_oracle.py's
  matrices; then the plain patch embedding."""
  kernel, patch = p["embedding/kernel"], image.shape[1] // seqhw
  p0, _, C, d = kernel.shape
  q = dict(p)
  if patch != p0:
    M = FO.patch_matrix(p0, patch).to(kernel.device)
    q["embedding/kernel"] = (M @ kernel.reshape(p0 * p0, C * d)).reshape(patch, patch, C, d)
  if pos is not None and (seqhw, seqhw) != tuple(posemb_size):
    assert posemb_size[0] == posemb_size[1]
    pos = FO.resize_matrix(posemb_size[0], seqhw, antialias=True).to(pos.device) @ pos.reshape(-1, d)
  return patch_embedding(image, q, "embedding", pos, cls)


def text_embed(ids, p):
  """text _Embed: Embed_0 of ids [n, L] plus the learned position embedding -> [n, L, d]."""
  return p["Embed_0/embedding"][ids.long()] + p["pos_embedding"]


def encoder_block(x, p, heads):
  """vit.EncoderBlock: x [n, N, d] -> [n, N, d]."""
  return O.encoder_block(x, p, heads, MM)


def mixer_block(x, p, masks=None):
  """mlp_mixer.MixerBlock: x [n, N, d] -> [n, N, d]; `masks` (token-mixing [n], channel-mixing [n]) gate each
  sample's residual branches.  The block body of O.mixer_forward."""
  y = O.layer_norm(x, p["LayerNorm_0/scale"], p["LayerNorm_0/bias"]).transpose(1, 2)
  tm = O.sub(p, "token_mixing/")
  h = O.gelu_tanh(O.dense(y, tm["Dense_0/kernel"], tm["Dense_0/bias"], MM))
  y = O.dense(h, tm["Dense_1/kernel"], tm["Dense_1/bias"], MM).transpose(1, 2)
  if masks is not None:
    y = y * masks[0][:, None, None]
  x = x + y
  y = O.layer_norm(x, p["LayerNorm_1/scale"], p["LayerNorm_1/bias"])
  y = O.mlp_block(y, O.sub(p, "channel_mixing/"), MM)
  if masks is not None:
    y = y * masks[1][:, None, None]
  return x + y


def norm_pool(x, p, pool, select=None):
  """vit.NormPool: the LayerNorm `scale` / `bias` of x [n, N, d], then the pool: "mean", "first", "last", "max"
  -> [n, d]; None -> [n, N, d].  The max pool averages the tokens that tie for the maximum of each column,
  and `select` [n, N, d] (default: the normalised x itself) is where that maximum is looked for: the CUDA
  path looks for it in its bf16 LayerNorm output."""
  y = O.layer_norm(x, p["scale"], p["bias"])
  if pool is None:
    return y
  if pool == "mean":
    return y.mean(1)
  if pool == "first":
    return y[:, 0]
  if pool == "last":
    return y[:, -1]
  if pool == "max":
    s = (y if select is None else select).detach()
    hit = (s == s.amax(1, keepdim=True)).to(y.dtype)
    return (y * hit).sum(1) / hit.sum(1)
  raise ValueError(pool)


def map_head(x, p, heads):
  """vit.MAPHead: x [n, N, d] -> [n, d]."""
  return O.map_head(x, p, heads, MM)


def dense(x, p, tanh=False):
  """common.Dense: x [rows, fan_in] -> [rows, fan_out] (tanh(x W + b) with `tanh`)."""
  y = O.dense(x, p["kernel"], p["bias"], MM)
  return torch.tanh(y) if tanh else y


class Tap(torch.overrides.TorchFunctionMode):
  """Exposes the gradient that reaches a bias before it is summed: where the bias `leaf` is reshaped or added
  in a reference, under this mode the result gets `self.tap` added, a zero tensor of `shape` (the rows the
  bias is broadcast over, then the bias's own width), whose gradient is then the per-row gradient the
  bias gradient is the sum of.  Used for the gradients that are zero in exact arithmetic, whose CUDA value is
  bounded by the sums of the |per-row gradients| it rounded: the key bias (softmax is invariant to a
  per-query shift) and the MLP-Mixer's token-mixing output bias (a per-token shift that every LayerNorm
  after it removes)."""

  def __init__(self, leaf, shape):
    super().__init__()
    self.leaf = leaf
    self.tap = torch.zeros(shape, dtype=leaf.dtype, device=leaf.device, requires_grad=True)

  def __torch_function__(self, func, types, args=(), kwargs=None):
    out = func(*args, **(kwargs or {}))
    if func in (torch.Tensor.reshape, torch.Tensor.add) and any(a is self.leaf for a in args):
      out = out + self.tap
    return out

  def floor(self):
    """sum of |per-row gradient| over the rows, shaped like the bias"""
    return self.tap.grad.abs().sum(tuple(range(self.tap.dim() - 1))).view(self.leaf.shape)


class ScoreGrad(torch.overrides.TorchFunctionMode):
  """Records, in a reference's attention, the queries and keys q, k [B, h, N, dh] of the score product
  s = q k^T / sqrt(dh) and, after the backward, dS = d s.  The CUDA attention backward feeds dS to the tensor
  cores in bf16, next to bf16 q and k: dq = dS k / sqrt(dh) and dk = dS^T q / sqrt(dh) each take two operands
  rounded with unit roundoff 2^-9, so |dq - dq_ref| <= 2^-8 |dS| |k| / sqrt(dh) to first order (dk alike).
  And dS = P (dP - D) takes D_i = sum_e dO_ie O_ie from the bf16 dO and the bf16 saved output O: an error of
  up to 2^-8 sum_e |dO_ie O_ie| in D_i, times P_ij, in every element of the row.
  Exact dS has zero row sums; when a query's keys share a large common component (deep blocks, where the
  tokens are nearly alike; the MAP head over the final tokens) that cancellation is what the rounding spoils,
  and this bound is the only honest scale for dq and dk there."""

  def __init__(self):
    super().__init__()
    self.q = self.k = self.s = self.P = self.o = None

  def __torch_function__(self, func, types, args=(), kwargs=None):
    out = func(*args, **(kwargs or {}))
    if func is torch.Tensor.matmul and self.q is None and args[0].dim() == 4:
      self.q, self.k = args[0], args[1].transpose(-1, -2)
    elif func is torch.softmax and self.s is None:
      self.s, self.P = args[0], out
      self.s.retain_grad()
    elif func is torch.Tensor.matmul and self.o is None and args[0] is self.P:
      self.o = out
      self.o.retain_grad()
    return out

  def floors(self):
    """(dq, dk) bounds [B, N, h * dh] of what the bf16 operands of dS k and dS^T q can change."""
    dh = self.q.shape[-1]
    d_err = 2.0 ** -8 * (self.o.grad * self.o).detach().abs().sum(-1, keepdim=True)
    dS = self.s.grad.abs() + self.P.detach() * d_err
    c = 2.0 ** -8 / dh ** 0.5
    fq = c * dS @ self.k.detach().abs()
    fk = c * dS.transpose(-1, -2) @ self.q.detach().abs()
    flat = lambda t: t.transpose(1, 2).reshape(t.shape[0], t.shape[2], -1)
    return flat(fq), flat(fk)
