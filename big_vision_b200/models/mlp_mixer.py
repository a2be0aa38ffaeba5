"""MLP-Mixer on the H100 kernels -- mirror of big_vision/models/mlp_mixer.py:30-124.

Same factory / fields / parameter names (`stem`, `MixerBlock_{i}/{LayerNorm_0,LayerNorm_1,
token_mixing,channel_mixing}/Dense_{0,1}`, `pre_head_layer_norm`, `head`; mlp_mixer.py:145-165).
The reference is fp32-only; BASELINE.json config 3 asks for bf16 matmuls (fp32 accumulate), which
is what runs here.  Token mixing applies the MLP along the token axis (mlp_mixer.py:49-51): the
activations are transposed to [n*d, tokens] (tokens padded to a multiple of 8 for TMA strides), run
through the same wgmma GEMMs, and transposed back fused with the residual add.
Stochastic depth (mlp_mixer.py:52,55,76,173-177): block i drops each residual branch per sample with
probability i/(L-1)*stoch_depth, no 1/(1-p) rescale.  The 0/1 masks are an INPUT of fwd
(`masks` fp32 [num_blocks, 2, n]; parity tests feed the same masks to the oracle) or, with train=True,
are drawn from the numpy Generator passed as `rng` (the reference draws them from JAX's threefry
stream, which cannot be reproduced without JAX).
The model is a list of backward stages (engine.Staged): the stem (vit.PatchEmbedding without a position
embedding), one MixerBlock per block, pre_head_layer_norm with the mean pool (vit.NormPool) and the head.
"""
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

from big_vision_b200 import engine as E
from big_vision_b200 import lib as L
from big_vision_b200 import ops
from big_vision_b200.models import common
from big_vision_b200.models import vit


class MixerBlock(E.Stage):
  """MixerBlock_{i} (mlp_mixer.py:40-55): x + token-mixing MLP over the tokens of LayerNorm_0(x), then
  x + channel-mixing MLP over LayerNorm_1(x).  With the forward's stochastic-depth masks (geom.masks)
  each residual branch is dropped per sample."""

  def __init__(self, i, N, d, tokens_mlp_dim, channels_mlp_dim):
    self.i, self.N, self.Np = i, N, (N + 7) // 8 * 8
    self.d, self.T, self.C = d, tokens_mlp_dim, channels_mlp_dim
    self.p = p = f"MixerBlock_{i}/"
    self.tm, self.cm = tm, cm = p + "token_mixing/", p + "channel_mixing/"
    self.prefixes = (p,)
    self.ready = p + "LayerNorm_0/scale"
    specs, aliases = vit.ln_specs(p + "LayerNorm_0/", d) + vit.ln_specs(p + "LayerNorm_1/", d), []
    # flax nn.Dense defaults: lecun_normal kernel, zero bias.  Token-mixing Dense_1 writes [n*d, N] in
    # rows of Np elements: its storage is padded.
    for nm, fi, fo, sc in ((tm + "Dense_0/", N, self.T, None),
                           (tm + "Dense_1/", self.T, N, self.Np),
                           (cm + "Dense_0/", d, self.C, None),
                           (cm + "Dense_1/", self.C, d, None)):
      s, a = common.dense_specs(nm, fi, fo, E.lecun_normal(fi), sc)
      specs += s
      aliases += a
    self._specs = specs, aliases
    self.k1, self.b1 = (s.name for s in specs if s.name.startswith(tm + "Dense_1/"))

  def specs(self):
    return self._specs

  def fwd(self, P, x, geom, save=True):
    """save=False (forward only): same output bits; every intermediate is released as soon as the
    next op has consumed it, GELU's pre-activations are not written and saved is None."""
    n, N, masks = geom.n, geom.N, geom.masks
    d, p, tm = self.d, self.p, self.tm
    y, mean1, rstd1 = ops.layernorm_fwd(x, P.f(p + "LayerNorm_0/scale"), P.f(p + "LayerNorm_0/bias"))
    yt = ops.transpose_tokens(y, n, N, d)                                   # [n*d, Np]
    del y
    if save:
      hact, hpre = ops.gemm(yt, P.h(tm + "Dense_0/kernel"), b_mn=True, bias=P.f(tm + "Dense_0/bias"),
                            epilogue=L.EPI_BIAS_GELU, K=N)
    else:
      del mean1, rstd1
      hact = ops.gemm(yt, P.h(tm + "Dense_0/kernel"), b_mn=True, bias=P.f(tm + "Dense_0/bias"),
                      epilogue=L.EPI_BIAS_GELU_ACT, K=N)
      del yt
    ot = torch.empty((n * d, self.Np), dtype=torch.bfloat16, device=x.device)
    ops.gemm(hact, P.h(self.k1), b_mn=True, bias=P.f(self.b1), out=ot, N=N)
    if not save:
      del hact
    x1 = ops.untranspose_add(ot, x, n, N, d)
    del ot
    if masks is not None:
      x1 = ops.row_select(x1, x, masks[self.i, 0], n, N)                    # x + mask * branch
    y2, mean2, rstd2 = ops.layernorm_fwd(x1, P.f(p + "LayerNorm_1/scale"), P.f(p + "LayerNorm_1/bias"))
    if not save:
      del mean2, rstd2
    x2, mlp_saved = vit.mlp_fwd(vit.Scope(P, self.cm), y2, x1, save=save)
    if masks is not None:
      x2 = ops.row_select(x2, x1, masks[self.i, 1], n, N)
    if not save:
      return x2, None
    return x2, (x, mean1, rstd1, yt, hact, hpre, x1, mean2, rstd2, mlp_saved)

  def sink(self, P, geom):
    """colsum(d block-output) is the gradient of channel_mixing/Dense_1/bias -- but not with stochastic
    depth: the gradient entering the branch is then mask * d block-output, and bwd sums it itself."""
    return P.g(self.cm + "Dense_1/bias") if geom.masks is None else None

  def bwd(self, P, dx, saved, geom, sink, need_dx=True):
    """dx: bf16 [n*N, d] grad of the block output.  Returns the grad of the block input; colsum of it is
    accumulated into `sink`.  need_dx changes nothing: LayerNorm_0's gradients need the full chain."""
    n, N, masks = geom.n, geom.N, geom.masks
    d, p, tm = self.d, self.p, self.tm
    x, mean1, rstd1, yt, hact, hpre, x1, mean2, rstd2, mlp_saved = saved
    # channel mixing
    dbr = dx if masks is None else ops.row_select(dx, None, masks[self.i, 1], n, N)
    dy2 = vit.mlp_bwd(vit.Scope(P, self.cm), dbr, mlp_saved, want_bias2_grad=self.sink(P, geom) is None)
    dx1 = ops.layernorm_bwd(dy2, x1, P.f(p + "LayerNorm_1/scale"), mean2, rstd2, dres=dx,
                            dscale=P.g(p + "LayerNorm_1/scale"), dbias=P.g(p + "LayerNorm_1/bias"))
    # token mixing
    dbr = dx1 if masks is None else ops.row_select(dx1, None, masks[self.i, 0], n, N)
    dot = ops.transpose_tokens(dbr, n, N, d)                                # [n*d, Np], pad = 0
    ops.colsum(dot, P.g(self.b1))
    ops.gemm(hact, dot, a_mn=True, b_mn=True, out=P.g(self.k1), reduce_out=True, N=N)
    dhpre = ops.gemm(dot, P.h(self.k1), aux=hpre, epilogue=L.EPI_DGELU, K=N)    # [n*d, T]
    # separate column-sum pass: with n*d rows over only T columns the GEMM epilogue's fused bias
    # gradient is all atomic contention (measured 2.62 vs 1.26 + 0.07 ms per call)
    ops.colsum(dhpre, P.g(tm + "Dense_0/bias"))
    ops.gemm(yt, dhpre, a_mn=True, b_mn=True, out=P.g(tm + "Dense_0/kernel"), reduce_out=True, M=N)
    dyt = torch.empty((n * d, self.Np), dtype=torch.bfloat16, device=dx.device)
    ops.gemm(dhpre, P.h(tm + "Dense_0/kernel"), out=dyt, N=N)
    dyl = ops.untranspose_add(dyt, None, n, N, d)
    return ops.layernorm_bwd(dyl, x, P.f(p + "LayerNorm_0/scale"), mean1, rstd1, dres=dx1,
                             dscale=P.g(p + "LayerNorm_0/scale"), dbias=P.g(p + "LayerNorm_0/bias"),
                             dx_colsum=sink)


@dataclass
class MlpMixer(E.Staged):
  """Fields as mlp_mixer.MlpMixer (mlp_mixer.py:58-68)."""
  patch_size: Tuple[int, int] = (16, 16)
  num_classes: Optional[int] = None
  num_blocks: int = 12
  hidden_dim: int = 768
  tokens_mlp_dim: int = 384
  channels_mlp_dim: int = 3072
  model_name: Optional[str] = None
  stoch_depth: float = 0.0

  def drop_p(self, i):
    """mlp_mixer.py:76"""
    return (i / max(self.num_blocks - 1, 1)) * self.stoch_depth

  def draw_masks(self, rng, n, device):
    """1 - Bernoulli(drop_p_i) per block, branch and sample (mlp_mixer.py:173-177) from a numpy
    Generator; fp32 [num_blocks, 2, n] on `device`."""
    p = np.array([self.drop_p(i) for i in range(self.num_blocks)], dtype=np.float64)[:, None, None]
    keep = (rng.random((self.num_blocks, 2, n)) >= p).astype(np.float32)
    return torch.from_numpy(keep).to(device)

  def specs(self, image_hw, in_ch=3):
    """Builds the backward stages for [n, *image_hw, in_ch] images -> (specs, aliases)."""
    d = self.hidden_dim
    self.head = common.Dense("head/", d, self.num_classes, E.zeros, pad=True) if self.num_classes else None
    # bottom-up; the blocks' token-mixing MLPs are as wide as the stem's token count
    stem = vit.PatchEmbedding("", "stem", image_hw, self.patch_size, in_ch, d, None, False)
    stages = ([stem] + [MixerBlock(i, stem.tokens, d, self.tokens_mlp_dim, self.channels_mlp_dim)
                        for i in range(self.num_blocks)]
              + [vit.NormPool("pre_head_layer_norm/", d, "mean", torch.float32)])
    if self.head is not None:
      stages.append(self.head)
    return self._build(stages)

  def init(self, seed, image_shape, device="cuda"):
    specs, aliases = self.specs(image_shape[1:3], image_shape[3])
    return E.FlatParams(specs, aliases, device).init(seed)

  def fwd(self, P, image, *, train=False, rng=None, masks=None, frozen=None):
    """image [n,H,W,C] fp32 -> (x fp32 [n, out], saved).  `masks` fp32 [num_blocks, 2, n], or drawn from
    `rng` with train=True.  `frozen` as in vit._Model.fwd: the stages below the cut run forward-only and
    save nothing."""
    n = image.shape[0]
    if masks is None and train and self.stoch_depth:
      if rng is None:
        raise ValueError("stoch_depth > 0 in training needs an rng (numpy Generator) or explicit masks")
      masks = self.draw_masks(rng, n, image.device)
    return self._stages_fwd(P, image, E.Geom(n, self._stages[0].tokens, masks), frozen)

  def bwd(self, P, dout, saved):
    self._stages_bwd(P, dout, saved)

  def apply(self, variables, image, *, train=False):
    x, _ = self.fwd(variables["params"], image, frozen=True)     # no backward follows: forward-only, same bits
    return x, {"logits" if self.num_classes else "pre_logits": x}


def Model(num_classes=None, *, variant=None, **kw):  # pylint: disable=invalid-name
  """Factory function to easily create a Model variant like "L/16" (mlp_mixer.py:87-124)."""
  if variant is not None:
    model_size, patch = variant.split("/")
    kw.setdefault("patch_size", (int(patch), int(patch)))
    config = {
        "S": {"hidden_dim": 512, "num_blocks": 8, "channels_mlp_dim": 2048, "tokens_mlp_dim": 256},
        "B": {"hidden_dim": 768, "num_blocks": 12, "channels_mlp_dim": 3072, "tokens_mlp_dim": 384},
        "L": {"hidden_dim": 1024, "num_blocks": 24, "channels_mlp_dim": 4096, "tokens_mlp_dim": 512},
        "H": {"hidden_dim": 1280, "num_blocks": 32, "channels_mlp_dim": 5120, "tokens_mlp_dim": 640},
    }[model_size]
    for k, v in config.items():
      kw.setdefault(k, v)
  return MlpMixer(num_classes=num_classes, **kw)
