"""GSAM classification training step -- mirror of `update_fn` in big_vision/trainers/proj/gsam/train.py:188-222
(config: configs/proj/gsam/vit_i1k_gsam_no_aug.py):

  mixup (per rank, as train.py)  ->  gsam_gradient on this rank's shard (both passes local)
  ->  pmean(loss, g): one all-reduce of the combined gradient  ->  tx.update

The learning rate that sets rho is `sched_fns[0](count) * lr` at the count the optimizer evaluates its
own schedule with.  Measurements: the CLEAN loss, l2_grads of the averaged g, l2_params, l2_updates.
"""
from big_vision_b200 import train as T
from big_vision_b200.trainers.proj.gsam import gsam as G
from big_vision_b200.trainers.proj.image_text.siglip import Dist


def make_update_fn(model, tx, config):
  mixup_p = (config.get("mixup") or {}).get("p")
  loss_name = config.get("loss", "sigmoid_xent")
  kw = G.parse_config(config.get("gsam"))
  if hasattr(tx, "frozen") and tx.frozen():
    # The reference perturbs by, and takes its norms over, the frozen parameters' clean gradients too;
    # this library computes no gradient for frozen stages.  Refuse rather than compute something else.
    raise NotImplementedError("GSAM with frozen parameters (a schedule entry of None)")
  if len(tx.sched_fns) != 1:
    raise NotImplementedError("GSAM supports one global learning-rate schedule (train.py:182)")
  d = Dist()
  twin = {}
  seed = int(config.get("seed", 0))

  def update_fn(train_state, rng, batch):
    P, opt = train_state["params"], train_state["opt"]
    images, labels = batch["image"], batch["labels"]
    if mixup_p:
      from big_vision_b200 import utils as u
      if rng is None:
        raise ValueError("mixup needs an rng (numpy Generator)")
      rng, (images, labels), _ = u.get_mixup(rng, mixup_p)(images, labels)
    fwd_kw = {}
    if getattr(model, "stoch_depth", 0.0):
      # one draw for both passes: the reference's loss_fn reuses the same dropout rng (train.py:198-206)
      if rng is None:
        raise ValueError("stoch_depth > 0 in training needs an rng (numpy Generator)")
      fwd_kw["masks"] = model.draw_masks(rng, images.shape[0], images.device)
    if getattr(model, "dropout", 0.0):      # one key for both passes, as for the masks above
      fwd_kw["dropout"] = T.dropout_key(seed, opt, d, images.shape[0])
    if "P" not in twin or twin["P"][0] is not P:
      twin["P"] = (P, P.twin())
    lr = tx.sched_fns[0](opt["count"]) * tx.lr
    loss = G.gsam_gradient(model, P, images, labels, lr=lr, loss_name=loss_name, P_sam=twin["P"][1], **kw,
                           **fwd_kw)
    # train.py:211: pmean of the clean loss and of the combined per-worker gradients
    d.all_reduce_sum(P.grad)
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
