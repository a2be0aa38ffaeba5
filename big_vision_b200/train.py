"""Classification training step -- mirror of `update_fn` in big_vision/train.py:271-315:

  logits = model(images) ; loss = getattr(u, config.loss)(logits, labels) (mean over batch)
  grads  = d loss / d params ; data-parallel mean over ranks ; fused Adam step.

Mixup (train.py:283-290, utils.py:1146-1158) runs per rank on that rank's shard, as the reference's
shard_map does.  Losses: sigmoid_xent / softmax_xent (utils.py:236-243, 276-281) as fused
loss+gradient kernels.
"""
import torch

from big_vision_b200 import ops
from big_vision_b200.trainers.proj.image_text.siglip import Dist

_LOSSES = {"sigmoid_xent": ops.sigmoid_xent, "softmax_xent": ops.softmax_xent}


def fwd_loss_bwd(model, P, images, loss_grad, dist_view=None, frozen=None, **fwd_kw):
  """Forward, `loss_grad`, backward on this rank's shard; P.grad holds the LOCAL gradient (callers average
  across ranks).  `loss_grad(flat, ld) -> dlogits [rows, ld]` gets the logits as [rows, classes] (row
  stride ld) and returns d loss / d logits with zeros in the columns past `classes`; the loss itself is
  its own business.  Returns the logits.

  `frozen` (storage names, optax.Chain.frozen()): parameters that get no gradient.  The model's backward
  stages below the lowest trained one run forward-only -- a linear probe (`head/.*` trained, the
  rest None) runs the backbone without a backward -- and the all-reduce covers the trained ranges only."""
  ranges = None
  if frozen:
    fwd_kw["frozen"] = frozen
    ranges = P.trained_ranges(frozen)
  P.zero_grad()
  logits, saved = model.fwd(P, images, **fwd_kw)
  # unpooled models (pool_type="none") give [n, N, classes]: the losses sum over the class axis and
  # average over all leading axes (utils.py:236-243,276-281), i.e. over the n*N rows.  A head with
  # padded storage returns a view of [rows, Cp] logits; the gradient is written [rows, Cp] with zero
  # padding columns, the layout the head's backward GEMMs take.
  flat = logits.reshape(-1, logits.shape[-1])
  ld = flat.stride(0)
  dlogits = loss_grad(flat, ld).view(*logits.shape[:-1], ld)
  if dist_view is None:
    model.bwd(P, dlogits, saved)
  else:      # gradient all-reduce (SUM; callers divide by world) overlapped with the backward
    from big_vision_b200.trainers.proj.image_text.siglip import all_reduce_grads
    all_reduce_grads(P, dist_view, lambda: model.bwd(P, dlogits, saved), ranges=ranges)
  return logits


def loss_and_grads(model, P, images, labels, loss_name="sigmoid_xent", dist_view=None, frozen=None, **fwd_kw):
  """value_and_grad(loss_fn)(params) of train.py:295-303 on this rank's shard, the LOCAL-mean loss
  (fwd_loss_bwd)."""
  if loss_name not in _LOSSES:
    raise NotImplementedError(f"loss {loss_name}")
  loss = torch.zeros(1, dtype=torch.float32, device=images.device)
  logits = fwd_loss_bwd(
      model, P, images, lambda flat, ld: _LOSSES[loss_name](flat, labels.reshape(flat.shape), loss, dlogits_cols=ld),
      dist_view, frozen, **fwd_kw)
  return loss, logits


def make_update_fn(model, tx, config):
  mixup_p = (config.get("mixup") or {}).get("p")
  loss_name = config.get("loss", "sigmoid_xent")
  d = Dist()
  frozen = tx.frozen() if hasattr(tx, "frozen") else frozenset()

  def update_fn(train_state, rng, batch, **fwd_kw):
    """`fwd_kw`: extra keyword arguments of the model's forward (a FlexiViT step's seqhw)."""
    P, opt = train_state["params"], train_state["opt"]
    images, labels = batch["image"], batch["labels"]
    if mixup_p:
      from big_vision_b200 import utils as u
      if rng is None:
        raise ValueError("mixup needs an rng (numpy Generator)")
      rng, (images, labels), _ = u.get_mixup(rng, mixup_p)(images, labels)
    # stochastic depth (Mixer, mlp_mixer.py:173-177) draws its masks from the step's rng like the
    # reference's `rngs={"dropout": rng}` (train.py:296-299)
    kw = dict(train=True, rng=rng) if getattr(model, "stoch_depth", 0.0) else {}
    loss, _ = loss_and_grads(model, P, images, labels, loss_name, dist_view=d, frozen=frozen, **kw, **fwd_kw)
    # the loss is the mean over the GLOBAL batch: sum the per-rank means and divide by world
    d.all_reduce_sum(loss)
    sc = tx.update(P, opt, grad_mult=1.0 / d.world)
    measurements = {
        "training_loss": loss[0] / d.world,
        "l2_grads": sc[0].sqrt() / d.world,
        "l2_params": sc[2].sqrt(),
        "l2_updates": sc[1].sqrt(),
    }
    return train_state, measurements

  return update_fn
