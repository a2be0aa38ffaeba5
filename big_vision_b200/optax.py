"""Optimizer factory -- the chain `big_vision/optax.py:75-149` builds, executed as fused CUDA
launches over the flat parameter buffer:

  clip_by_global_norm(grad_clip_norm)          (norm over the NON-frozen gradients, :104-113)
  -> inner transform `config.optax_name`       scale_by_adam (fused, `bv_adam_step`) | scale (`bv_scale_step`)
  -> scale(lr) [* lr_mults, first match]       (:120-129)
  -> add_decayed_weights(wd * wd_mults)        (first match; default mask ".*/kernel$", :136-145)
  -> scale_by_schedule, one per config.schedule pattern (first match; None = frozen, :79-101)
  -> scale(-1), applied to the parameters in place (optax.apply_updates).

Every stored parameter gets (schedule index | frozen, lr multiplier, weight decay) from the regex
lists exactly like `u.make_mask_trees` assigns them (FIRST matching pattern wins, full match on the
reference name "a/b/c"); neighbours in the flat layout with the same setting are merged into one
launch -- two launches for the default config (decayed kernels | everything else).  Frozen ranges
get no launch and no optimizer state (optax_test.py:301-317) and do not count towards the clipping
norm or `l2_grads` (optax_test.py:206-299, siglip.py:315-321).

`big_vision.scale_by_adafactor` (optax.py:187-214) is the third inner transform: one `bv_adafactor_step`
per reference tensor (factored second moments over the two largest axes when the second largest is
>= min_dim_size_to_factor, bf16 momentum), see `_AdafactorTensor`.  Not built: clipping_threshold
(clip_by_block_rms) and per-example clipping raise instead of silently doing something else.
"""
import re

import torch

from big_vision_b200 import ops
from big_vision_b200 import utils as u


class _AdafactorTensor:
  """One reference tensor (a stored parameter or a named view of a fused one) as bv_adafactor_step sees
  it: the strided view [A, L, M, H] of the flat buffers with {L, H} = optax's factored dims
  (`_factored_dims`: the two largest axes, provided the second largest is >= min_dim_size_to_factor),
  or a flat/2-D view for an unfactored tensor."""

  def __init__(self, name, view, min_dim_size_to_factor):
    import numpy as np
    self.name, self.offset = name, view.storage_offset()
    shape, stride = list(view.shape), list(view.stride())
    self.numel = int(np.prod(shape))
    order = np.argsort(shape, kind="stable")
    if len(shape) < 2 or shape[order[-2]] < min_dim_size_to_factor:
      self.mode = 0
      if view.is_contiguous():
        self.dims, self.strides = (1, 1, 1, self.numel), (0, 0, 0)
      elif len(shape) == 2 and stride[1] == 1:
        self.dims, self.strides = (1, shape[0], 1, shape[1]), (0, stride[0], 0)
      elif len(shape) == 3 and stride[2] == 1:     # e.g. a scan-stacked q / k / v bias [depth, heads, dh]
        self.dims, self.strides = (shape[0], shape[1], 1, shape[2]), (stride[0], stride[1], 0)
      else:
        raise NotImplementedError(f"adafactor: unfactored strided tensor {name} {shape} {stride}")
      return
    d1, d0 = int(order[-2]), int(order[-1])          # optax: (second largest, largest)
    lo, hi = min(d0, d1), max(d0, d1)
    if hi != len(shape) - 1 or stride[hi] != 1:
      raise NotImplementedError(f"adafactor: factored axes of {name} {shape} are not (.., L, .., H)")

    def merged(axes):                                # (size, stride) of a run of axes read as one
      size = int(np.prod([shape[i] for i in axes])) if axes else 1
      for i, j in zip(axes, axes[1:]):
        if stride[i] != stride[j] * shape[j]:
          raise NotImplementedError(f"adafactor: axes {axes} of {name} do not merge")
      return size, (stride[axes[-1]] if axes else 0)

    (A, sA), (M, sM) = merged(list(range(lo))), merged(list(range(lo + 1, hi)))
    self.dims, self.strides = (A, shape[lo], M, shape[hi]), (sA, stride[lo], sM)
    self.mode = 1 if d0 == hi else 2

  def state_sizes(self):
    A, L, M, H = self.dims
    return {"vfull": self.numel} if self.mode == 0 else {"red_h": A * L * M, "red_l": A * M * H, "nrm": A * M}


def _first_match(patterns, names):
  """Index of the first pattern that fully matches ALL reference names of one stored parameter
  (a fused q|k|v kernel carries three names); None if no pattern matches any of them.  Names of one
  storage that would be assigned differently cannot be honoured and raise."""
  hits = set()
  for name in names:
    hit = next((i for i, p in enumerate(patterns) if p.fullmatch(name)), None)
    hits.add(hit)
  if len(hits) > 1:
    raise NotImplementedError(f"{sorted(names)} share one fused storage tensor but match different "
                              "optimizer patterns")
  return hits.pop()


class Chain:
  """tx-like object: init(P) -> opt state, update(P, opt, ...) applies one step in place."""

  def __init__(self, config, P, sched_kw):
    name = config.get("optax_name", "scale_by_adam")
    kw = dict(config.get("optax", {}) or {})
    if name == "scale_by_adam":
      self.b1, self.b2, self.eps = kw.pop("b1", 0.9), kw.pop("b2", 0.999), kw.pop("eps", 1e-8)
      mu_dtype = kw.pop("mu_dtype", None)
      self.mu_dtype = torch.bfloat16 if mu_dtype in ("bfloat16", torch.bfloat16) else torch.float32
      if kw.pop("eps_root", 0.0):
        raise NotImplementedError("eps_root")
      self.step_size = None
    elif name == "scale":
      self.step_size = float(kw.pop("step_size"))
    elif name == "big_vision.scale_by_adafactor":
      self.af = dict(min_dim_size_to_factor=kw.pop("min_dim_size_to_factor", 32), decay_rate=kw.pop("decay_rate", 0.8),
                     decay_offset=kw.pop("decay_offset", 0), beta2_cap=kw.pop("beta2_cap", 0.999),
                     momentum=kw.pop("momentum", 0.9), eps=kw.pop("eps", 1e-30))
      if kw.pop("clipping_threshold", None):
        raise NotImplementedError("adafactor clipping_threshold (optax.clip_by_block_rms)")
      if kw.pop("dtype_momentum", "bfloat16") not in ("bfloat16", torch.bfloat16):
        raise NotImplementedError("adafactor momentum accumulator other than bfloat16")
      self.step_size = None
    else:
      raise NotImplementedError(f"optax_name={name}: built are scale_by_adam, scale, big_vision.scale_by_adafactor")
    if kw:
      raise NotImplementedError(f"{name} options {sorted(kw)}")
    if config.get("grad_clip_per_example"):
      raise NotImplementedError("grad_clip_per_example")
    if not config.get("weight_decay_decouple", True):
      raise AssertionError("Coupled weight decay not supported anymore.")
    self.inner = name
    self.lr = float(config.get("lr", 1e-3))
    self.clip = float(config.get("grad_clip_norm", 0.0) or 0.0)

    # ---- schedules (first match; None = frozen) ------------------------------------------------
    schedule = config.get("schedule", {})
    if not isinstance(schedule, (tuple, list)):
      schedule = [(".*", schedule)]
    sched_pat = u.check_and_compile_patterns([p for p, _ in schedule])
    self.sched_fns, sched_slot = [], []
    for _, sc in schedule:
      if sc is None:
        sched_slot.append(None)
      else:
        sc = dict(sc)
        if "base" in sc:
          raise AssertionError(sc)
        sched_slot.append(len(self.sched_fns))
        self.sched_fns.append(u.create_learning_rate_schedule(base=sc.pop("mult", 1.0), **sched_kw, **sc))
    lr_mults = list(config.get("lr_mults") or [])
    if not all(m > 0 for _, m in lr_mults):
      raise AssertionError(f"Use schedule=None for parameter freezing instead of lr_mults={lr_mults}")
    lr_pat = u.check_and_compile_patterns([p for p, _ in lr_mults]) if lr_mults else []
    wd = float(config.get("wd", 0.0) or 0.0)
    wd_mults = list(config.get("wd_mults", [(".*/kernel$", 1.0)])) if wd else []
    wd_pat = u.check_and_compile_patterns([p for p, _ in wd_mults]) if wd_mults else []

    # ---- per stored parameter -> merged launch ranges over the flat layout -----------------------
    names_of = {}
    for a in P.aliases.values():
      names_of.setdefault(a.storage, []).append(a.name)
    uncovered, self.ranges = [], []      # ranges: [lo, hi, sched slot | None, lr mult, wd]
    self.per_storage = []                # (storage, sched slot | None, lr mult, wd)
    for storage, (off, shape) in sorted(P.offsets.items(), key=lambda kv: kv[1][0]):
      names = names_of.get(storage, [storage])
      si = _first_match(sched_pat, names)
      if si is None:
        uncovered += names
        continue
      li = _first_match(lr_pat, names) if lr_pat else None
      wi = _first_match(wd_pat, names) if wd_pat else None
      key = (sched_slot[si], 1.0 if li is None else float(lr_mults[li][1]),
             0.0 if wi is None else wd * float(wd_mults[wi][1]))
      self.per_storage.append((storage, *key))
      n = 1
      for dim in shape:
        n *= dim
      hi = off + (n + 7) // 8 * 8          # engine.ALIGN: the padding belongs to its parameter
      if self.ranges and tuple(self.ranges[-1][2:]) == key and self.ranges[-1][1] == off:
        self.ranges[-1][1] = hi
      else:
        self.ranges.append([off, hi, *key])
    if uncovered:
      raise AssertionError(f"All params must be covered (use `None` for freezing): {uncovered}")
    # optimizer state only for what is trained, packed in range order
    self.state_off, n_state = [], 0
    for lo, hi, slot, _, _ in self.ranges:
      self.state_off.append(n_state if slot is not None else None)
      if slot is not None:
        n_state += hi - lo
    self.n_state = n_state
    # adafactor works tensor by tensor on the REFERENCE tensors (the named views of fused storage)
    self.tensors = []
    if self.inner == "big_vision.scale_by_adafactor":
      views_of = {}
      for a in P.aliases.values():
        views_of.setdefault(a.storage, []).append(a)
      for storage, slot, lr_mult, wd in self.per_storage:
        if slot is None:
          continue
        base = P.f(storage)
        for nm, view in ([(a.name, a.view(base)) for a in views_of[storage]] if storage in views_of
                         else [(storage, base)]):
          self.tensors.append((_AdafactorTensor(nm, view, self.af["min_dim_size_to_factor"]), slot, lr_mult, wd))

  def frozen(self):
    """frozenset of the storage names whose schedule is None.  The models' forward takes it
    (`frozen=`) to run the stages that hold no trained parameter forward-only, and the gradient
    all-reduce skips their ranges."""
    return frozenset(storage for storage, slot, *_ in self.per_storage if slot is None)

  def init(self, P):
    dev = P.flat.device
    state = {"count": 0, "scalars": torch.zeros(4, dtype=torch.float32, device=dev)}   # [gnorm_sq, upd_sq, param_sq]
    if self.inner == "scale_by_adam":
      state["mu"] = torch.zeros(self.n_state, dtype=self.mu_dtype, device=dev)
      state["nu"] = torch.zeros(self.n_state, dtype=torch.float32, device=dev)
    if self.inner == "big_vision.scale_by_adafactor":
      state["af"] = []
      for t, *_ in self.tensors:
        st = {k: torch.zeros(n, dtype=torch.float32, device=dev) for k, n in t.state_sizes().items()}
        if self.af["momentum"]:
          st["momentum"] = torch.zeros(t.numel, dtype=torch.bfloat16, device=dev)
        state["af"].append(st)
    return state

  def update(self, P, opt, grad_mult=1.0):
    """Applies one step in place; returns the device tensor [gnorm_sq, upd_sq, param_sq, 0]."""
    sc = opt["scalars"]
    sc.zero_()
    trained = [(r, so) for r, so in zip(self.ranges, self.state_off) if r[2] is not None]
    for (lo, hi, *_), _ in trained:                      # norm over the non-frozen gradients only
      ops.sumsq(P.grad[lo:hi], sc[0:1])
    scheds = [fn(opt["count"]) for fn in self.sched_fns]   # evaluated at the pre-increment count
    step = opt["count"] + 1
    if self.inner == "big_vision.scale_by_adafactor":
      # second-moment decay of this step (optax.py:196-199): min(beta2_cap, 1 - (t + 1)^-decay_rate), float32
      import numpy as np
      t = np.float32(opt["count"] - self.af["decay_offset"]) + np.float32(1.0)
      decay = float(min(np.float32(self.af["beta2_cap"]), np.float32(1.0) - t ** np.float32(-self.af["decay_rate"])))
      for (tens, slot, lr_mult, wd), st in zip(self.tensors, opt["af"]):
        ops.adafactor_step(P, tens, st, decay=decay, eps=self.af["eps"], beta=self.af["momentum"] or 0.0,
                           lr_eff=scheds[slot] * self.lr * lr_mult, wd_eff=scheds[slot] * wd, grad_mult=grad_mult,
                           clip_norm=self.clip, gnorm_sq=sc[0:1], upd_sq=sc[1:2], param_sq=sc[2:3])
      trained = []
    for (lo, hi, slot, lr_mult, wd), so in trained:
      sched = scheds[slot]
      common = dict(wd_eff=sched * wd, grad_mult=grad_mult, clip_norm=self.clip, gnorm_sq=sc[0:1],
                    upd_sq=sc[1:2], param_sq=sc[2:3])
      if self.inner == "scale_by_adam":
        ops.adam_step(P.flat[lo:hi], P.grad[lo:hi], opt["mu"][so:so + hi - lo], opt["nu"][so:so + hi - lo],
                      P.half[lo:hi], lr_eff=sched * self.lr * lr_mult, b1=self.b1, b2=self.b2, eps=self.eps,
                      step=step, **common)
      else:
        ops.scale_step(P.flat[lo:hi], P.grad[lo:hi], P.half[lo:hi],
                       lr_eff=sched * self.lr * lr_mult * self.step_size, **common)
    frozen = [r for r in self.ranges if r[2] is None]
    for lo, hi, *_ in frozen:                            # l2_params covers every parameter
      ops.sumsq(P.flat[lo:hi], sc[2:3])
    opt["count"] = step
    return sc


FusedAdam = Chain     # name used by round-1 callers


def make(config, params, *, sched_kw):
  """Returns (tx, schedule_fns) like optax.py:75 `make`; `params` is the model's FlatParams."""
  if "optim" in config:
    raise AssertionError("Deprecated option, use config.optax.")
  if "weight_decay" in config:
    raise AssertionError("Deprecated option. Use wd and schedule.")
  tx = Chain(config, params, sched_kw)
  return tx, list(tx.sched_fns)
