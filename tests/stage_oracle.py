"""TEST INFRASTRUCTURE: one float64 reference per kind of backward stage (engine.Stage) of the models, built
from the pieces of oracle/bv_oracle.py (mm="float32": plain high-precision math) and of tests/bit_oracle.py
(in its float64 mode).  Each function takes the stage's input and its parameters, `p`: a dict of float64
tensors under the reference names relative to the stage's root (the stage's own prefix, or the model prefix
for the embeddings), and returns the stage's output; torch autograd then gives d input and the parameter
gradients under the same names.

Chained bottom-up they are the whole models of the oracle (tests/test_stage_oracle.py checks that), so a stage
checked against its reference on the inputs the CUDA path actually gave it is checked against the pinned
oracle, one stage at a time.

Where a stage's discrete decision (a ReLU's sign, a max pool's route) is taken on a value the kernels rounded
to bf16 inside the stage, a reference can be handed that decision instead of taking its own: within a bf16
rounding of the threshold the two would decide differently and move a whole gradient term, which says nothing
about the kernels.  Without it each reference decides on its own float64 values."""
import math

import torch
import torch.nn.functional as F

import bit_oracle as BO
import flexi_oracle as FO
from oracle import bv_oracle as O

MM = "float32"
BERT_EPS = 1e-12      # models/proj/flaxformer/bert.py LN_EPS


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


# ---- BERT (models/proj/flaxformer/bert.py) ----------------------------------------------------------------
def bert_embed(ids, p, keep=None):
  """bert._Embed: ids [n, N] -> the token row + position row (< N) + segment row 0, then the embedding
  LayerNorm (eps 1e-12) -> [n, N, d]; `keep` (the scaled EMBED dropout mask [n, N, d]) multiplies it."""
  N = ids.shape[1]
  x = (p["embedders_token_ids/embedding"][ids.long()] + p["embedders_position_ids/embedding"][:N]
       + p["embedders_segment_ids/embedding"][0])
  y = O.layer_norm(x, p["layer_norm/scale"], p["layer_norm/bias"], eps=BERT_EPS)
  return y if keep is None else y * keep


def bert_attention(x, p, heads, key_mask, probs=None):
  """BERT's self-attention of x [n, N, d] with the key mask [n, N] (True = attend; every sample attends at
  least one key) and `probs` (the scaled dropout mask [n, heads, N, N] of the probabilities, or None).  The
  softmax is torch.softmax of the -inf-masked scores, where ScoreGrad finds it."""
  n, N, d = x.shape
  dh = d // heads

  def proj(name):
    y = O.dense(x, p[name + "/kernel"].reshape(d, d), p[name + "/bias"].reshape(d), MM)
    return y.reshape(n, N, heads, dh).transpose(1, 2)

  q, k, v = proj("query"), proj("key"), proj("value")
  s = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
  w = torch.softmax(s.masked_fill(~key_mask[:, None, None, :], -math.inf), dim=-1)
  if probs is not None:
    w = w * probs
  o = (w @ v).transpose(1, 2).reshape(n, N, d)
  return O.dense(o, p["out/kernel"].reshape(d, d), p["out/bias"], MM)


def bert_layer(x, p, heads, key_mask, masks=None):
  """bert._Layer: x [n, N, d] -> the post-LN layer x1 = LN(x + Attn(x)), LN(x1 + MLP(x1)).  `masks`: None, or
  the scaled dropout masks (probabilities [n, heads, N, N], attention output [n, N, d], MLP output [n, N, d])."""
  probs, attn, mlp = (None, None, None) if masks is None else masks
  y = bert_attention(x, O.sub(p, "self_attention/"), heads, key_mask, probs)
  if attn is not None:
    y = y * attn
  x = O.layer_norm(x + y, p["attention_layer_norm/scale"], p["attention_layer_norm/bias"], eps=BERT_EPS)
  y = O.mlp_block(x, O.sub(p, "mlp/"), MM)
  if mlp is not None:
    y = y * mlp
  return O.layer_norm(x + y, p["output_layer_norm/scale"], p["output_layer_norm/bias"], eps=BERT_EPS)


def cls_pool(x):
  """bert._ClsPool: x [n, N, d] -> the [CLS] token x[:, 0]."""
  return x[:, 0]


# ---- BiT ResNet-v2 (models/bit_paper.py) -------------------------------------------------------------------
def _windows(t, ho, wo):
  """The 3 x 3 / 2 windows of t [n, h + 2, w + 2, C] (padded by one): [9, n, ho, wo, C], row-major order."""
  return torch.stack([t[:, i:i + 2 * ho - 1:2, j:j + 2 * wo - 1:2] for i in range(3) for j in range(3)])


def bit_root(image, p, route=None):
  """bit_paper.RootBlock: image [n, H, W, 3] -> StdConv 7 x 7 / 2 (padding 3), then the -inf-padded 3 x 3 / 2
  max pool -> [n, ho, wo, C].  Each window takes its first maximum in row-major window order of `route`
  [n, h, w, C] (default: the convolution output itself); the CUDA path routes by its bf16 convolution output."""
  y = BO.std_conv(image, p["conv_root/kernel"], 2, 3)
  h, w = y.shape[1], y.shape[2]
  ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
  pad = lambda t: F.pad(t, (0, 0, 1, 1, 1, 1), value=-math.inf)
  first = _windows(pad((y if route is None else route).detach()), ho, wo).argmax(0)   # the first maximum
  return _windows(pad(y), ho, wo).gather(0, first[None])[0]


def _gn_relu(x, p, prefix, keep=None):
  """The GroupNorm under `prefix` of x, then the ReLU, or the given ReLU decision `keep` (True = positive)."""
  y = BO.group_norm(x, p[prefix + "scale"], p[prefix + "bias"])
  return torch.relu(y) if keep is None else y * keep


def bit_unit(x, p, stride, relu_masks=None):
  """bit_paper.ResidualUnit: x [n, h, w, cin] -> the pre-activation bottleneck [n, ho, wo, 4 nmid], with the
  projection when p has conv_proj.  `relu_masks`: None, or the ReLU decisions of gn2 and gn3 (bool, shaped like
  their outputs); the CUDA path decides them on its bf16 conv1 and conv2 outputs."""
  m2, m3 = (None, None) if relu_masks is None else relu_masks
  a1 = _gn_relu(x, p, "gn1/")
  res = BO.std_conv(a1, p["conv_proj/kernel"], stride, 0) if "conv_proj/kernel" in p else x
  h = _gn_relu(BO.std_conv(a1, p["conv1/kernel"], 1, 0), p, "gn2/", m2)
  h = _gn_relu(BO.std_conv(h, p["conv2/kernel"], stride, 1), p, "gn3/", m3)
  return BO.std_conv(h, p["conv3/kernel"], 1, 0) + res


def bit_prehead(x, p):
  """bit_paper.PreHead: x [n, h, w, C] -> GroupNorm + ReLU, then the mean over the pixels -> [n, C]."""
  return _gn_relu(x, p, "").mean(dim=(1, 2))


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
