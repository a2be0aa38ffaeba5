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


def _dense_specs(p, fan_in, fan_out, store_cols=None):
  """flax nn.Dense defaults: lecun_normal kernel, zeros bias.  `store_cols` pads the stored
  kernel/bias columns (TMA row strides must be multiples of 16 bytes)."""
  lec = E.lecun_normal(fan_in)
  sc = store_cols or fan_out
  if sc == fan_out:
    return [E.ParamSpec(p + "kernel", (fan_in, fan_out), lec),
            E.ParamSpec(p + "bias", (fan_out,), E.zeros)], []
  pad = sc - fan_out
  specs = [E.ParamSpec(p + "kernel_pad", (fan_in, sc),
                       lambda rng, shape: np.concatenate([lec(rng, (fan_in, fan_out)),
                                                          np.zeros((fan_in, pad))], 1)),
           E.ParamSpec(p + "bias_pad", (sc,), E.zeros)]
  aliases = [E.Alias(p + "kernel", p + "kernel_pad", lambda t: t[:, :fan_out]),
             E.Alias(p + "bias", p + "bias_pad", lambda t: t[:fan_out])]
  return specs, aliases


@dataclass
class MlpMixer:
  """Fields as mlp_mixer.MlpMixer (mlp_mixer.py:58-68)."""
  patch_size: Tuple[int, int] = (16, 16)
  num_classes: Optional[int] = None
  num_blocks: int = 12
  hidden_dim: int = 768
  tokens_mlp_dim: int = 384
  channels_mlp_dim: int = 3072
  model_name: Optional[str] = None
  stoch_depth: float = 0.0

  def __post_init__(self):
    self._geom = None
    self.head = common.ClassifierHead("", self.hidden_dim, self.num_classes, E.zeros) if self.num_classes else None

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
    ph, pw = self.patch_size
    self._geom = (image_hw[0] // ph, image_hw[1] // pw)
    N = self._geom[0] * self._geom[1]
    Np = (N + 7) // 8 * 8
    d = self.hidden_dim
    K = ph * pw * in_ch
    Kp = (K + 7) // 8 * 8
    lec = E.lecun_normal(K)
    specs = [E.ParamSpec("stem/kernel_flat", (Kp, d),
                         lambda rng, shape: np.concatenate([lec(rng, (K, d)), np.zeros((Kp - K, d))], 0)),
             E.ParamSpec("stem/bias", (d,), E.zeros)]
    aliases = [E.Alias("stem/kernel", "stem/kernel_flat", lambda t: t[:K].unflatten(0, (ph, pw, in_ch)))]
    for i in range(self.num_blocks):
      p = f"MixerBlock_{i}/"
      specs += vit.ln_specs(p + "LayerNorm_0/", d) + vit.ln_specs(p + "LayerNorm_1/", d)
      for nm, fi, fo, sc in ((p + "token_mixing/Dense_0/", N, self.tokens_mlp_dim, None),
                             (p + "token_mixing/Dense_1/", self.tokens_mlp_dim, N, Np),
                             (p + "channel_mixing/Dense_0/", d, self.channels_mlp_dim, None),
                             (p + "channel_mixing/Dense_1/", self.channels_mlp_dim, d, None)):
        s, a = _dense_specs(nm, fi, fo, sc)
        specs += s
        aliases += a
    specs += vit.ln_specs("pre_head_layer_norm/", d)
    if self.head is not None:
      s, a = self.head.specs()
      specs += s
      aliases += a
    self._N, self._Np = N, Np
    return specs, aliases

  def init(self, seed, image_shape, device="cuda"):
    specs, aliases = self.specs(image_shape[1:3], image_shape[3])
    return E.FlatParams(specs, aliases, device).init(seed)

  @staticmethod
  def _store(P, p, what):
    """Name of the stored kernel/bias (padded storage if it exists)."""
    return p + what + ("_pad" if (p + what + "_pad") in P.offsets else "")

  def fwd(self, P, image, *, train=False, rng=None, masks=None):
    n = image.shape[0]
    d, N, Np, T = self.hidden_dim, self._N, self._Np, self.tokens_mlp_dim
    if masks is None and train and self.stoch_depth:
      if rng is None:
        raise ValueError("stoch_depth > 0 in training needs an rng (numpy Generator) or explicit masks")
      masks = self.draw_masks(rng, n, image.device)
    patches = ops.patchify(image, self.patch_size[0])
    x = ops.gemm(patches, P.h("stem/kernel_flat"), b_mn=True, bias=P.f("stem/bias"))
    saved = {"patches": patches, "n": n, "blocks": [], "masks": masks}
    for i in range(self.num_blocks):
      p = f"MixerBlock_{i}/"
      tm, cm = p + "token_mixing/", p + "channel_mixing/"
      y, mean1, rstd1 = ops.layernorm_fwd(x, P.f(p + "LayerNorm_0/scale"), P.f(p + "LayerNorm_0/bias"))
      yt = ops.transpose_tokens(y, n, N, d)                                   # [n*d, Np]
      hact, hpre = ops.gemm(yt, P.h(tm + "Dense_0/kernel"), b_mn=True, bias=P.f(tm + "Dense_0/bias"),
                            epilogue=L.EPI_BIAS_GELU, K=N)
      ot = torch.empty((n * d, Np), dtype=torch.bfloat16, device=x.device)
      ops.gemm(hact, P.h(self._store(P, tm + "Dense_1/", "kernel")), b_mn=True,
               bias=P.f(self._store(P, tm + "Dense_1/", "bias")), out=ot, N=N)
      x1 = ops.untranspose_add(ot, x, n, N, d)
      if masks is not None:
        x1 = ops.row_select(x1, x, masks[i, 0], n, N)                         # x + mask * branch
      y2, mean2, rstd2 = ops.layernorm_fwd(x1, P.f(p + "LayerNorm_1/scale"), P.f(p + "LayerNorm_1/bias"))
      x2, mlp_saved = vit.mlp_fwd(vit.Scope(P, cm), y2, x1)
      if masks is not None:
        x2 = ops.row_select(x2, x1, masks[i, 1], n, N)
      saved["blocks"].append((x, mean1, rstd1, yt, hact, hpre, x1, mean2, rstd2, mlp_saved))
      x = x2
    y, mean, rstd = ops.layernorm_fwd(x, P.f("pre_head_layer_norm/scale"), P.f("pre_head_layer_norm/bias"))
    saved["norm"] = (x, mean, rstd)
    out = ops.pool_fwd(y, n, N, 0, out_dtype=torch.float32)
    if self.head is not None:
      out, saved["head_in"] = self.head.fwd(P, out)
    return out, saved

  def bwd(self, P, dout, saved):
    n = saved["n"]
    d, N, Np, T = self.hidden_dim, self._N, self._Np, self.tokens_mlp_dim
    if self.head is not None:
      dout = self.head.bwd(P, dout, saved["head_in"])
    dy = ops.pool_bwd(dout, n, N, 0)
    x, mean, rstd = saved["norm"]
    masks = saved.get("masks")
    # with stochastic depth the gradient entering a branch is mask * dx, so the fused
    # "colsum(dx) -> the previous block's Dense_1 bias gradient" shortcut does not apply
    last = f"MixerBlock_{self.num_blocks - 1}/channel_mixing/Dense_1/bias"
    dx = ops.layernorm_bwd(dy, x, P.f("pre_head_layer_norm/scale"), mean, rstd,
                           dscale=P.g("pre_head_layer_norm/scale"), dbias=P.g("pre_head_layer_norm/bias"),
                           dx_colsum=P.g(last) if masks is None else None)
    for i in reversed(range(self.num_blocks)):
      p = f"MixerBlock_{i}/"
      tm, cm = p + "token_mixing/", p + "channel_mixing/"
      x, mean1, rstd1, yt, hact, hpre, x1, mean2, rstd2, mlp_saved = saved["blocks"][i]
      saved["blocks"][i] = None
      # channel mixing (colsum(dx) already went into this block's channel_mixing/Dense_1/bias)
      dbr = dx if masks is None else ops.row_select(dx, None, masks[i, 1], n, N)
      dy2 = vit.mlp_bwd(vit.Scope(P, cm), dbr, mlp_saved, want_bias2_grad=masks is not None)
      dx1 = ops.layernorm_bwd(dy2, x1, P.f(p + "LayerNorm_1/scale"), mean2, rstd2, dres=dx,
                              dscale=P.g(p + "LayerNorm_1/scale"), dbias=P.g(p + "LayerNorm_1/bias"))
      # token mixing
      k1, b1 = self._store(P, tm + "Dense_1/", "kernel"), self._store(P, tm + "Dense_1/", "bias")
      dbr = dx1 if masks is None else ops.row_select(dx1, None, masks[i, 0], n, N)
      dot = ops.transpose_tokens(dbr, n, N, d)                                # [n*d, Np], pad = 0
      ops.colsum(dot, P.g(b1))
      ops.gemm(hact, dot, a_mn=True, b_mn=True, out=P.g(k1), reduce_out=True, N=N)
      dhpre = ops.gemm(dot, P.h(k1), aux=hpre, epilogue=L.EPI_DGELU, K=N)    # [n*d, T]
      # separate column-sum pass: with n*d rows over only T columns the GEMM epilogue's fused bias
      # gradient is all atomic contention (measured 2.62 vs 1.26 + 0.07 ms per call)
      ops.colsum(dhpre, P.g(tm + "Dense_0/bias"))
      ops.gemm(yt, dhpre, a_mn=True, b_mn=True, out=P.g(tm + "Dense_0/kernel"), reduce_out=True, M=N)
      dyt = torch.empty((n * d, Np), dtype=torch.bfloat16, device=dx.device)
      ops.gemm(dhpre, P.h(tm + "Dense_0/kernel"), out=dyt, N=N)
      dyl = ops.untranspose_add(dyt, None, n, N, d)
      prev = (P.g(f"MixerBlock_{i - 1}/channel_mixing/Dense_1/bias") if i > 0 else P.g("stem/bias"))
      if masks is not None and i > 0:
        prev = None
      dx = ops.layernorm_bwd(dyl, x, P.f(p + "LayerNorm_0/scale"), mean1, rstd1, dres=dx1,
                             dscale=P.g(p + "LayerNorm_0/scale"), dbias=P.g(p + "LayerNorm_0/bias"),
                             dx_colsum=prev)
    ops.gemm(saved["patches"], dx, a_mn=True, b_mn=True, out=P.g("stem/kernel_flat"), reduce_out=True)

  def apply(self, variables, image, *, train=False):
    x, _ = self.fwd(variables["params"], image)
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
