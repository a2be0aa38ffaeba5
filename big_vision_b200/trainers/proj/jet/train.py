"""Jet training -- mirror of `update_fn` and `eval_loss_fn` in big_vision/trainers/proj/jet/train.py:272-333,
398-409 (config: configs/proj/jet/imagenet64.py):

  images = image + U[0, 1/127.5)  (the step's noise: key config.seed, counter = the optimizer's step count)
  z, logdet = model.forward(images) ; loss = mean over the global batch of (nll - logdet) / (D ln 2)
  grads = d loss / d params ; data-parallel mean over ranks ; fused Adam step.

The noise is the counter-based stream of bv_jet_dequantize_patchify, indexed by the element's position in the
GLOBAL batch, so a step's noise does not depend on how many ranks share the batch.  Not built: the
class-conditional model (a `label` in the batch, jet.py:50-56) and trained masks.
"""
import math


from big_vision_b200 import ops
from big_vision_b200.models.proj.jet import jet
from big_vision_b200.trainers.proj.image_text.siglip import Dist
from big_vision_b200.trainers.proj.image_text.siglip import all_reduce_grads

MEASUREMENTS = ("training_loss", "bits", "nll", "logdet", "l2_grads", "l2_params", "l2_updates")


def _refuse_context(batch):
  if "label" in batch or "context" in batch:
    raise NotImplementedError("class-conditional Jet (a label / context in the batch) is not built")


def loss_and_grads(model, P, images, noise, dist_view=None, frozen=jet.MASKS):
  """Forward, bits and backward on this rank's shard: -> (rows fp32 [3, n], means fp32 [3]) of
  (bits, nll, logdet) / (D ln 2), the means over the LOCAL batch.  P.grad holds the gradient of the local mean
  (summed over ranks when dist_view has peers)."""
  n = images.shape[0]
  P.zero_grad()
  (z, logdet), saved = model.fwd(P, images, frozen=frozen, noise=noise)
  grad_scale = 1.0 / (n * (z.numel() // n) * math.log(2.0))
  rows, means, dz = ops.jet_bits(z, logdet, grad_scale)
  del z
  run = lambda: model.bwd(P, dz, -grad_scale, saved)
  if dist_view is None:
    run()
  else:
    all_reduce_grads(P, dist_view, run, ranges=P.trained_ranges(frozen))
  return rows, means


def make_update_fn(model, tx, config):
  """-> update_fn(train_state, rng, batch): one step on this rank's shard of the global batch.  `rng` is not
  used: the step's noise comes from config.seed and the step count."""
  frozen = tx.frozen() if hasattr(tx, "frozen") else frozenset()
  if not jet.MASKS <= frozen:
    raise NotImplementedError("the coupling masks must be frozen by the schedule (('.*FREEZE_ME.*', None)): "
                              "training them through the permutation einsum is not built")
  seed = int(config.get("seed", 0))
  d = Dist()

  def update_fn(train_state, rng, batch):
    del rng
    _refuse_context(batch)
    P, opt = train_state["params"], train_state["opt"]
    images = batch["image"]
    _, means = loss_and_grads(model, P, images, (seed, opt["count"], d.rank * images.numel()), d, frozen)
    # the means are over the GLOBAL batch: sum the per-rank means and divide by world
    d.all_reduce_sum(means)
    sc = tx.update(P, opt, grad_mult=1.0 / d.world)
    means = means / d.world
    measurements = {
        "training_loss": means[0],
        "bits": means[0],
        "nll": means[1],
        "logdet": means[2],
        "l2_grads": sc[0].sqrt() / d.world,
        "l2_params": sc[2].sqrt(),
        "l2_updates": sc[1].sqrt(),
    }
    return train_state, measurements

  return update_fn


def make_predict_fns(model, config):
  """{"loss": fn(params, batch, seed, counter, offset=0) -> {"bits", "nll", "logdet"}}: per-example values
  (each / (D ln 2)) of the forward on the batch plus its dequantization noise, as eval_loss_fn
  (train.py:398-409)."""
  del config

  def loss_fn(params, batch, seed, counter, offset=0):
    _refuse_context(batch)
    (z, logdet), _ = model.fwd(params, batch["image"], frozen=True, noise=(seed, counter, offset))
    rows, _ = ops.jet_bits(z, logdet)
    return {"bits": rows[0], "nll": rows[1], "logdet": rows[2]}

  return {"loss": loss_fn}
