"""SigLIP training step -- mirror of `update_fn` in
big_vision/trainers/proj/image_text/siglip.py:271-323, written out in its explicit
data-parallel form (_deprecated_contrastive.py:117-141, :343):

  zimg, ztxt = two_towers(images, labels)                       (local batch n)
  ztxt_all   = all_gather(ztxt)                                 C1  [B, D]
  loss       = (1/B) sum_i sum_j -log_sigmoid(+-(zimg_i.ztxt_j * exp(t) + b))
  dztxt      = reduce_scatter(d loss / d ztxt_all)              C2
  grads      = all_reduce_sum(local grads)                      C3 (+ loss, dt, db: C4)
  params    += fused Adam step

One process per GPU; collectives go through torch.distributed (NCCL over NVLink on the
GPU box, gloo in the CPU tests).  The loss is normalised by the GLOBAL batch B
(siglip.py:306), so per-rank partial losses/gradients are SUMMED across ranks.
"""
import math
import os

import torch
import torch.distributed as dist

from big_vision_b200 import engine as E
from big_vision_b200 import ops


class Dist:
  """Thin view of the default process group (world size 1 when not initialised)."""

  def __init__(self):
    self.on = dist.is_available() and dist.is_initialized()
    self.world = dist.get_world_size() if self.on else 1
    self.rank = dist.get_rank() if self.on else 0

  def all_gather_rows(self, x):
    if self.world == 1:
      return x
    out = torch.empty((self.world * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    self._timed("nccl_all_gather", lambda: dist.all_gather_into_tensor(out, x.contiguous()))
    return out

  def reduce_scatter_rows(self, x):
    if self.world == 1:
      return x
    out = torch.empty((x.shape[0] // self.world,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    self._timed("nccl_reduce_scatter",
                lambda: dist.reduce_scatter_tensor(out, x.contiguous(), op=dist.ReduceOp.SUM))
    return out

  def broadcast_rows(self, x, src):
    """Every rank receives rank `src`'s x (same shape on all ranks)."""
    if self.world == 1:
      return x
    buf = x.contiguous().clone() if self.rank == src else torch.empty_like(x)
    self._timed("nccl_broadcast", lambda: dist.broadcast(buf, src=src))
    return buf

  def reduce_rows(self, x, dst):
    """Sum over ranks delivered to rank `dst` (the other ranks' return value is scratch)."""
    if self.world > 1:
      x = x.contiguous()
      self._timed("nccl_reduce", lambda: dist.reduce(x, dst=dst, op=dist.ReduceOp.SUM))
    return x

  def all_reduce_sum(self, x):
    if self.world > 1:
      self._timed("nccl_all_reduce", lambda: dist.all_reduce(x, op=dist.ReduceOp.SUM))
    return x

  @staticmethod
  def _timed(name, fn):
    """Runs a collective; under bench.py --profile-calls it is bracketed by CUDA events like
    every C-ABI call (NCCL kernels run on the current stream for the default process group)."""
    from big_vision_b200 import lib as L
    if L.PROFILE is None:
      fn()
      return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    L.PROFILE.append((name, e0, e1, 0.0))


class BucketedGradAllReduce:
  """C3 overlapped with the backward pass (the reference's `lax.pmean` of the gradients,
  _deprecated_contrastive.py:343, which XLA schedules under the backward as well).

  Gradients complete in the REVERSE of the parameter-spec order (the loss scalars first, then the
  text tower from its head down to its embedding, then the image tower likewise), and the flat
  gradient buffer is laid out in spec order inside each of its two groups (decayed kernels | the
  rest).  So the finished part of each group grows from the group's end towards its start: whenever
  the backward reports "everything from spec `name` on is done" (`P.on_ready`, called by the stage
  runner engine.Staged after every unstacked encoder block) and at least `bucket_elems` new elements are final, that slice
  is all-reduced asynchronously -- NCCL's stream waits for the kernels enqueued so far, the main
  stream carries on with the next block -- and `finish()` reduces what is left and joins.
  Elementwise SUM over the same values as one big all-reduce: results are identical."""

  def __init__(self, P, d, bucket_elems=8 << 20, ranges=None):
    self.P, self.d, self.bucket = P, d, bucket_elems
    self.ranges = ranges                   # trained [lo, hi) slices (None: the whole buffer)
    idx = {s.name: i for i, s in enumerate(P.specs)}
    self.idx = idx
    self.groups = []                       # (lo, hi, [spec index ...], [offset ...]) in layout order
    for lo, hi in ((0, P.n_decay), (P.n_decay, P.total)):
      members = sorted((off, idx[name]) for name, (off, _) in P.offsets.items() if lo <= off < hi)
      self.groups.append((lo, hi, [m[1] for m in members], [m[0] for m in members]))
    self.front, self.handles = None, []

  def begin(self):
    self.front = [hi for _, hi, _, _ in self.groups]
    self.handles = []
    self.P.on_ready = self.ready

  def _launch(self, lo, hi):
    for a, b in ([(lo, hi)] if self.ranges is None else
                 [(max(lo, r0), min(hi, r1)) for r0, r1 in self.ranges]):
      if b > a:
        h = dist.all_reduce(self.P.grad[a:b], op=dist.ReduceOp.SUM, async_op=True)
        self.handles.append(h)

  def ready(self, name):
    """Everything at or after storage parameter `name` in spec order has its final gradient."""
    k = self.idx[name]
    for gi, (lo, hi, spec_idx, offs) in enumerate(self.groups):
      # layout order == spec order inside a group: first member whose spec index is >= k
      import bisect
      j = bisect.bisect_left(spec_idx, k)
      new = offs[j] if j < len(offs) else hi
      if self.front[gi] - new >= self.bucket:
        self._launch(new, self.front[gi])
        self.front[gi] = new

  def finish(self):
    self.P.on_ready = None
    for gi, (lo, hi, _, _) in enumerate(self.groups):
      self._launch(lo, self.front[gi])
      self.front[gi] = lo
    for h in self.handles:
      h.wait()                             # the current stream waits for NCCL's
    self.handles = []


def all_reduce_grads(P, d, run_backward, ranges=None):
  """Runs `run_backward()` and all-reduces (SUM) the flat gradient buffer when there are peers.
  `ranges` (FlatParams.trained_ranges) restricts the reduction to those [lo, hi) slices: frozen
  parameters have no gradient to reduce, and their slices stay as the backward left them.

  Default: ONE all-reduce after the backward (one per range).  BV_GRAD_ALLREDUCE=overlap selects the bucketed form
  that runs under the backward (BucketedGradAllReduce).  Which of the two is faster on H100 has not
  been measured: an NCCL kernel that holds a few SMs delays the GEMM tiles running beside it, so the
  overlapped form pays for part of the collective anyway, plus the extra launches."""
  if d.world == 1:
    run_backward()
    return
  if os.environ.get("BV_GRAD_ALLREDUCE") != "overlap":
    run_backward()
    if ranges is None:
      d.all_reduce_sum(P.grad)
    else:
      for lo, hi in ranges:
        d.all_reduce_sum(P.grad[lo:hi])
    return
  red = BucketedGradAllReduce(P, d, ranges=ranges)
  red.begin()
  try:
    run_backward()
  finally:
    red.finish()


def sigmoid_loss_fwd_bwd(P, zimg, ztxt, d, scal, img_grad=True, txt_grad=True):
  """Pairwise sigmoid loss + gradients for the local image rows against ALL text rows.

  scal: fp32 device tensor [>=1]; scal[0] += this rank's share of the loss.
  dt/db are accumulated straight into the gradient slots of `t` and `b`.
  Returns (dzimg [n,D] fp32, dztxt_local [n,D] fp32); img_grad / txt_grad = False (a wholly frozen
  tower) skips that embedding's gradient, its GEMM and its collective, and returns None for it.
  """
  n, D = zimg.shape
  ztxt_all = d.all_gather_rows(ztxt)                       # C1
  B = ztxt_all.shape[0]
  zi16 = ops.cast(zimg, torch.empty_like(zimg, dtype=torch.bfloat16))
  zt16 = ops.cast(ztxt_all, torch.empty_like(ztxt_all, dtype=torch.bfloat16))
  dots = ops.gemm(zi16, zt16, out_dtype=torch.float32)     # [n, B] = zimg . ztxt_all^T
  has_b = "b" in P.offsets
  G = ops.siglip_loss(dots, d.rank * n, P.f("t"), P.f("b") if has_b else None, B,
                      scal[0:1], P.g("t"), P.g("b") if has_b else None)
  dzimg = dztxt = None
  if img_grad:
    dzimg = ops.gemm(G, zt16, b_mn=True, out_dtype=torch.float32)                  # G . ztxt_all
  if txt_grad:
    dztxt_all = ops.gemm(G, zi16, a_mn=True, b_mn=True, out_dtype=torch.float32)   # G^T . zimg
    dztxt = d.reduce_scatter_rows(dztxt_all)               # C2
  return dzimg, dztxt


def chunked_sigmoid_loss_fwd_bwd(P, zimg, ztxt, d, scal, img_grad=True, txt_grad=True):
  """The memory-lean variant of the same loss: section 3.1 of arxiv.org/abs/2303.15343,
  `chunked_sigmoid_loss` in _deprecated_contrastive.py:168-200.  G rounds; round r scores the local
  images against rank r's texts only, so the live slab is [n, n] instead of [n, B].  Positives sit
  on the diagonal of the round r == rank; every other round is all negatives (row_offset = -n puts
  the positive column outside the block).  The reference gathers the chunk with a masked psum;
  here it is a broadcast from its owner, and the chunk's gradient is reduced back to the owner.
  Same arguments and return values as sigmoid_loss_fwd_bwd; same loss value and gradients."""
  n, D = zimg.shape
  B = n * d.world
  zi16 = ops.cast(zimg, torch.empty_like(zimg, dtype=torch.bfloat16))
  has_b = "b" in P.offsets
  dzimg = torch.zeros((n, D), dtype=torch.float32, device=zimg.device) if img_grad else None
  dztxt = None
  for r in range(d.world):
    chunk = d.broadcast_rows(ztxt, src=r)                          # C1, one peer per round
    zc16 = ops.cast(chunk, torch.empty_like(chunk, dtype=torch.bfloat16))
    dots = ops.gemm(zi16, zc16, out_dtype=torch.float32)           # [n, n]
    G = ops.siglip_loss(dots, 0 if r == d.rank else -n, P.f("t"), P.f("b") if has_b else None, B,
                        scal[0:1], P.g("t"), P.g("b") if has_b else None)
    if img_grad:
      ops.gemm(G, zc16, b_mn=True, out=dzimg, reduce_out=True)     # dzimg += G . chunk
    if txt_grad:
      dzc = ops.gemm(G, zi16, a_mn=True, b_mn=True, out_dtype=torch.float32)   # G^T . zimg  [n, D]
      dzc = d.reduce_rows(dzc, dst=r)                              # C2, delivered to the owner
      if r == d.rank:
        dztxt = dzc
  return dzimg, dztxt


def softmax_loss_fwd_bwd(P, zimg, ztxt, d, scal, img_grad=True, txt_grad=True):
  """The CLIP softmax loss, `softmax_loss` of _deprecated_contrastive.py:80-101 (config.loss_fn="softmax"):
  0.5 * (image->text + text->image) InfoNCE, each direction a softmax of the local rows against ALL
  gathered columns with the positive on this rank's diagonal block; temperature only (no bias).
  Global semantics: mean over the global batch of both directions (the reference's per-device means
  followed by pmean).  scal[0] += loss share, scal[1] / scal[2] += number of correct i2t / t2i
  retrievals on this rank (the reference's `i2t_acc` / `t2i_acc` times n).
  Same arguments and return values as sigmoid_loss_fwd_bwd."""
  n, D = zimg.shape
  zimg_all = d.all_gather_rows(zimg)                       # t2i needs the gathered image embeddings too
  ztxt_all = d.all_gather_rows(ztxt)
  B = ztxt_all.shape[0]
  cast16 = lambda x: ops.cast(x, torch.empty_like(x, dtype=torch.bfloat16))
  zi16, zt16, zia16, zta16 = cast16(zimg), cast16(ztxt), cast16(zimg_all), cast16(ztxt_all)
  off = d.rank * n
  # image -> text: local images against all texts
  dots = ops.gemm(zi16, zta16, out_dtype=torch.float32)                          # [n, B]
  G1 = ops.softmax_contrastive_loss(dots, off, P.f("t"), B, 0.5, scal[0:1], P.g("t"), scal[1:2])
  # text -> image: local texts against all images
  dots = ops.gemm(zt16, zia16, out_dtype=torch.float32)                          # [n, B]
  G2 = ops.softmax_contrastive_loss(dots, off, P.f("t"), B, 0.5, scal[0:1], P.g("t"), scal[2:3])
  # contributions to the OTHER ranks' rows (the gathered operand of each direction), summed back
  dzimg = dztxt = None
  if txt_grad:
    dztxt = ops.gemm(G2, zia16, b_mn=True, out_dtype=torch.float32)              # G2 . zimg_all
    dztxt_all = ops.gemm(G1, zi16, a_mn=True, b_mn=True, out_dtype=torch.float32)  # G1^T . zimg [B, D]
    dztxt = ops.axpby(dztxt, d.reduce_scatter_rows(dztxt_all), 1.0, 1.0) if d.world > 1 else \
        ops.axpby(dztxt, dztxt_all, 1.0, 1.0)
  if img_grad:
    dzimg = ops.gemm(G1, zta16, b_mn=True, out_dtype=torch.float32)              # G1 . ztxt_all
    dzimg_all = ops.gemm(G2, zt16, a_mn=True, b_mn=True, out_dtype=torch.float32)  # G2^T . ztxt [B, D]
    dzimg = ops.axpby(dzimg, d.reduce_scatter_rows(dzimg_all), 1.0, 1.0) if d.world > 1 else \
        ops.axpby(dzimg, dzimg_all, 1.0, 1.0)
  return dzimg, dztxt


_LOSS_FNS = {"sigmoid": sigmoid_loss_fwd_bwd, "chunked_sigmoid": chunked_sigmoid_loss_fwd_bwd,
             "softmax": softmax_loss_fwd_bwd}


def _loss_fn(config):
  """config.loss_fn as in _deprecated_contrastive.py:322-331 ('sigmoid' is what siglip.py runs)."""
  name = (config or {}).get("loss_fn", "sigmoid")
  if name not in _LOSS_FNS:
    raise NotImplementedError(f"Unrecognized loss config.loss_fn={name!r} (built: {sorted(_LOSS_FNS)})")
  return _LOSS_FNS[name]


def make_update_fn(model, tx, config=None):
  """Returns update_fn(train_state, rng, batch) -> (train_state, measurements), the
  signature of siglip.py:275.  train_state = {"params": FlatParams, "opt": opt_state};
  it is updated IN PLACE (the reference donates it, siglip.py:273).

  Parameters whose schedule is None (tx.frozen(), e.g. the image tower under SigLiT's
  `schedule=[("img/.*", None), (".*", ...)]`) get no gradient: the stages that hold only frozen
  parameters run forward-only, a wholly frozen tower gets no embedding gradient from the loss, and
  the gradient all-reduce covers the trained ranges only."""
  d = Dist()
  loss_fwd_bwd = _loss_fn(config)
  frozen = tx.frozen() if hasattr(tx, "frozen") else frozenset()
  plan = {}

  seed = int((config or {}).get("seed", 0))

  def update_fn(train_state, rng, batch):
    del rng  # the dropout masks come from config.seed and the step count
    P, opt = train_state["params"], train_state["opt"]
    images, labels = batch["image"], batch["labels"]
    if id(P) not in plan:
      plan.clear()
      plan[id(P)] = _frozen_plan(model, P, frozen)
    fz, ranges, (img_frozen, txt_frozen) = plan[id(P)]
    P.zero_grad()
    scal = torch.zeros(4, dtype=torch.float32, device=P.flat.device)
    key = E.DropoutKey(seed, int(opt["count"]), d.rank * images.shape[0])
    zimg, ztxt, saved = model.fwd(P, images, labels, frozen=fz, dropout=key)
    dzimg, dztxt = loss_fwd_bwd(P, zimg, ztxt, d, scal, img_grad=not img_frozen, txt_grad=not txt_frozen)
    # C3 (+ dt, db inside the flat buffer), bucketed and overlapped with the backward
    all_reduce_grads(P, d, lambda: model.bwd(P, dzimg, dztxt, saved), ranges=ranges)
    d.all_reduce_sum(scal)                                 # C4: loss
    sc = tx.update(P, opt, grad_mult=1.0)
    measurements = {
        "training_loss": scal[0],
        "l2_grads": sc[0].sqrt(),
        "l2_params": sc[2].sqrt(),
        "l2_updates": sc[1].sqrt(),
    }
    return train_state, measurements

  return update_fn


def _frozen_plan(model, P, frozen):
  """(frozen for the forward or None, trained ranges for the all-reduce or None, (image tower wholly
  frozen, text tower wholly frozen)); all None / False when nothing is frozen: today's path."""
  if not frozen:
    return None, None, (False, False)
  return frozen, P.trained_ranges(frozen), model.tower_frozen(P, frozen)


def loss_and_grads(model, P, images, labels, loss_fn="sigmoid", frozen=None, dropout=None):
  """value_and_grad(loss_fn)(params) of siglip.py:287-311 without the optimizer: returns the
  global loss (device scalar) with P.grad holding d loss / d params (summed over ranks).  `frozen`
  (storage names, optax.Chain.frozen()) as in make_update_fn: their gradients are not computed.
  `dropout`: the step's engine.DropoutKey, or None (no dropout)."""
  d = Dist()
  sigmoid_loss_fwd_bwd = _loss_fn({"loss_fn": loss_fn})   # pylint: disable=redefined-outer-name
  fz, ranges, (img_frozen, txt_frozen) = _frozen_plan(model, P, frozen)
  P.zero_grad()
  scal = torch.zeros(4, dtype=torch.float32, device=P.flat.device)
  zimg, ztxt, saved = model.fwd(P, images, labels, frozen=fz, dropout=dropout)
  dzimg, dztxt = sigmoid_loss_fwd_bwd(P, zimg, ztxt, d, scal, img_grad=not img_frozen,
                                      txt_grad=not txt_frozen)
  all_reduce_grads(P, d, lambda: model.bwd(P, dzimg, dztxt, saved), ranges=ranges)
  d.all_reduce_sum(scal)
  return scal[0], {"zimg": zimg, "ztxt": ztxt, "dzimg": dzimg, "dztxt": dztxt}
