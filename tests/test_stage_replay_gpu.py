"""Per-stage float64 replay of the model backward.

One real forward + backward of a model runs with every backward stage (engine.Stage) instance wrapped, and
each block of a ScanEncoder too.  The wrappers record each stage's input, Geom, output, incoming dy, the sink
it was handed and the dx it returned; before the backward the gradient buffer is filled with a seeded random
pattern, not zeros.  Right after each stage's backward, top stage first:
  1. dx matches the stage's float64 reference (tests/stage_oracle.py) on the recorded input and dy;
  2. every parameter the stage owns equals seed + reference gradient (a sink-delivered bias is final then);
  3. the stage was handed the sink of the stage below, and that range equals seed + colsum(reference dx);
  4. every other element of the buffer is what it was: the seed, or the value it had when it became final;
     padding columns, alignment gaps and the stages below included.  Bit for bit;
  5. a ScanEncoder block recomputed in the backward gives the bits of its forward (output and saved tensors);
  6. with a frozen cut, the stages below it are never called and the stage at it gets need_dx=False.
The `ready` announcements (P.on_ready) are recorded with BucketedGradAllReduce's own slice mapping: each slice
announced final must hold its final bits.

Bounds (checks 1-3), per tensor with reference R and result G: ||G - R||_2 <= tau ||R||_2 and
max|G - R| <= tau_max max|R|, per stage kind (TOL).  The gradients that are zero in exact arithmetic (EXACT_ZERO)
get the floor |G - R| <= ZERO_FLOOR * colsum(|per-row gradient|) per element instead."""
import json
import math

import numpy as np
import pytest
import torch

import stage_oracle as S

pytestmark = pytest.mark.gpu

F64 = torch.float64
# (tau, tau_max) per stage kind: at most 4x the worst normwise / element-wise value measured on the clean path
# (the comments; H100 80GB HBM3 at a 700 W power limit), never above 2^-6 / 2^-4
TOL = {
    "PatchEmbedding": (2 ** -19, 2 ** -18),        # measured 7.2e-7, 1.2e-6 (fp32 sums of bf16 products)
    "FlexiPatchEmbedding": (2 ** -21, 2 ** -19),   # 3.1e-7, 6.8e-7
    "_Embed": (2 ** -22, 2 ** -22),                # 9.5e-8, 9.3e-8
    "EncoderBlock": (2 ** -6, 2 ** -4),            # 1.4e-2, 2.0e-2
    "MixerBlock": (2 ** -6, 2 ** -6),              # 6.0e-3, 6.3e-3
    "NormPool": (2 ** -7, 2 ** -6),                # 2.4e-3, 4.5e-3
    "MAPHead": (2 ** -6, 2 ** -5),                 # 8.4e-3, 1.1e-2
    "Dense": (2 ** -7, 2 ** -7),                   # 2.4e-3, 2.8e-3
}
ZERO_FLOOR = 2 ** -6
# gradients that are zero in exact arithmetic -> the per-row shape of the tap that gives their floor: the key
# bias (softmax is invariant to a per-query shift of the scores) and the Mixer's token-mixing output bias (a
# per-token shift, which every LayerNorm after it removes)
KEY_BIAS = "MultiHeadDotProductAttention_0/key/bias"
EXACT_ZERO = {
    "EncoderBlock": (KEY_BIAS, lambda st, n, N: (n, N, st.d)),
    "MAPHead": (KEY_BIAS, lambda st, n, N: (n, N, st.d)),
    "MixerBlock": ("token_mixing/Dense_1/bias", lambda st, n, N: (n, st.d, N)),
}

# the gradients computed from the attention backward's dq and dk, which get the bound of stage_oracle.ScoreGrad
# (the bf16 operands of dS k and dS^T q) on top of TOL: dq, dk propagated through the weight-gradient sums
QK = ("MultiHeadDotProductAttention_0/query/kernel", "MultiHeadDotProductAttention_0/query/bias",
      "MultiHeadDotProductAttention_0/key/kernel")
QK_FLOOR = ("EncoderBlock", "MAPHead")
# Open finding: the MAP head of ViT-B/16 (one probe query against 196 nearly alike final tokens) leaves its
# query / key gradients 1.6x past that first-order bound (11 % normwise); the bf16 operands of dq, dk and D do
# not account for all of it.  That case alone allows 2x the bound for those three tensors of the MAP head
# (CASES "qk_allow"); every other check of the case is as strict as elsewhere.

NC = 13      # C % 8 != 0: the padded class head
TINY = dict(width=64, depth=2, mlp_dim=128, num_heads=1)

# name -> (model kind, model keyword arguments, input shape, extra)
CASES = {
    "vit_tok": ("vit", dict(pool_type="tok", rep_size=32), (4, 40, 40, 3), {}),
    "vit_gap_sincos": ("vit", dict(pool_type="gap", posemb="sincos2d"), (4, 40, 40, 3), {}),
    "vit_map": ("vit", dict(pool_type="map"), (4, 40, 40, 3), {}),
    "vit_0": ("vit", dict(pool_type="0"), (4, 40, 40, 3), {}),
    "vit_none": ("vit", dict(pool_type="none"), (4, 40, 40, 3), {}),
    "vit_tok_scan": ("vit", dict(pool_type="tok", rep_size=32, scan=True, depth=3), (4, 40, 40, 3), {}),
    "vit_map_scan": ("vit", dict(pool_type="map", scan=True, depth=3), (4, 40, 40, 3), {}),
    "vit_hd72": ("vit", dict(pool_type="map", width=144, num_heads=2, mlp_dim=288), (4, 40, 40, 3), {}),
    "vit_b16_tok": ("vit_b16", dict(pool_type="tok", rep_size=True), (4, 224, 224, 3), {}),
    "vit_b16_map": ("vit_b16", dict(pool_type="map"), (4, 224, 224, 3), dict(qk_allow={"MAPHead": 2.0})),
    "mixer": ("mixer", {}, (4, 56, 56, 3), {}),
    "mixer_stoch": ("mixer", dict(stoch_depth=0.5), (4, 56, 56, 3), dict(masks=True)),
    "text_last": ("text", dict(pool_type="last"), (4, 16), {}),
    "text_first": ("text", dict(pool_type="first"), (4, 16), {}),
    "text_max": ("text", dict(pool_type="max"), (4, 16), dict(ties=True)),
    "text_mean": ("text", dict(pool_type="mean"), (4, 16), {}),
    "text_map": ("text", dict(pool_type="map"), (4, 16), {}),
    "text_last_nohead": ("text", dict(pool_type="last", num_classes=None), (4, 16), {}),
    "text_map_nohead": ("text", dict(pool_type="map", num_classes=None), (4, 16), {}),
    "flexi_resample": ("flexi", dict(pool_type="tok"), (4, 56, 56, 3), dict(seqhw=4)),
    "flexi_base_sincos": ("flexi", dict(pool_type="gap", posemb="sincos2d"), (4, 56, 56, 3), dict(seqhw=7)),
    "vit_frozen_cut": ("vit", dict(pool_type="gap"), (4, 40, 40, 3), dict(frozen=1)),
    "text_frozen_cut": ("text", dict(pool_type="last"), (4, 16), dict(frozen=1)),
}


def build_model(case):
  """The case's model with its stages built (specs() called): no device needed."""
  kind, kw, shape, _ = CASES[case]
  if kind in ("vit", "vit_b16"):
    from big_vision_b200.models import vit
    model = (vit.Model(1000, variant="B/16", **kw) if kind == "vit_b16" else
             vit.Model(NC, patch_size=(8, 8), **{**TINY, **kw}))
    model.specs(shape[1:3], shape[3])
  elif kind == "mixer":
    from big_vision_b200.models import mlp_mixer
    model = mlp_mixer.Model(NC, patch_size=(8, 8), num_blocks=3, hidden_dim=64, tokens_mlp_dim=32,
                            channels_mlp_dim=128, **kw)
    model.specs(shape[1:3], shape[3])
  elif kind == "text":
    from big_vision_b200.models.proj.image_text import text_transformer
    model = text_transformer.Model(**{"num_classes": 32, **kw}, **TINY, vocab_size=64)
    model.specs(shape[1])
  else:
    from big_vision_b200.models.proj.flexi import vit as fv
    model = fv.Model(NC, patch_size=(8, 8), **{**TINY, **kw})
    model.specs(shape[1:3], shape[3])
  return model


# ---- set-up -------------------------------------------------------------------------------------------
def _params(model, case, seed=0):
  """FlatParams with every all-zero initial tensor replaced by small random values (padding stays zero)."""
  from big_vision_b200 import engine as E
  _, _, shape, extra = CASES[case]
  specs, aliases = (model.specs(shape[1]) if CASES[case][0] == "text" else model.specs(shape[1:3], shape[3]))
  P = E.FlatParams(specs, aliases, "cuda").init(seed)
  rng = np.random.default_rng(seed + 1)
  tree = {k: ((rng.standard_normal(v.shape) * 0.05).astype(np.float32) if not np.any(v) else v)
          for k, v in P.numpy_tree("f").items()}
  if extra.get("ties"):            # tokens 4 and 9 identical in every layer: exact ties in the max pool
    tree["pos_embedding"][:, 9] = tree["pos_embedding"][:, 4]
  P.load_tree(tree)
  return P


def _inputs(model, case, seed=0):
  kind, _, shape, extra = CASES[case]
  rng = np.random.default_rng(seed + 2)
  if kind == "text":
    ids = rng.integers(0, 64, size=shape).astype(np.int32)
    if extra.get("ties"):
      ids[:, 9] = ids[:, 4]
    x = torch.from_numpy(ids).cuda()
  else:
    x = torch.from_numpy(rng.uniform(-1, 1, size=shape).astype(np.float32)).cuda()
  kw = {}
  if kind == "mixer" and extra.get("masks"):
    masks = np.ones((3, 2, shape[0]), np.float32)
    masks[1, 0, 1] = masks[1, 1, 3] = 0     # single samples dropped
    masks[2, 0, :] = 0                     # a branch dropped for the whole batch: its gradients are exactly 0
    masks[2, 1, 2] = 0
    kw["masks"] = torch.from_numpy(masks).cuda()
  if kind == "flexi":
    kw["seqhw"] = extra["seqhw"]
  return x, kw


def frozen_set(model, P, case):
  """The storages of the stages below stage `frozen` + 1 (the embedding and the first block): the cut is
  mid-model, at the second block."""
  k = CASES[case][3].get("frozen")
  if not k:
    return None
  prefixes = tuple(p for s in model.stages()[:k + 1] for p in s)
  return frozenset(n for n in P.offsets if n.startswith(prefixes))


def _dout(model, out, seed=0):
  from big_vision_b200.models import common
  top = model._stages[-1]   # pylint: disable=protected-access
  cols = top.Cp if isinstance(top, common.Dense) else out.shape[-1]
  g = torch.Generator(device="cuda").manual_seed(seed + 3)
  dout = torch.randn(tuple(out.shape[:-1]) + (cols,), generator=g, device="cuda")
  dout[..., out.shape[-1]:] = 0
  return dout


def _run(model, P, x, kw, frozen, dout=None, before_bwd=None):
  out, saved = model.fwd(P, x, frozen=frozen, **kw)
  if dout is None:
    dout = _dout(model, out)
  if before_bwd is not None:
    before_bwd()
  model.bwd(P, dout, saved)
  torch.cuda.synchronize()
  return dout


# ---- the recorder of `ready` announcements ---------------------------------------------------------------
def ready_recorder(P, ranges=None):
  """BucketedGradAllReduce with a bucket of one element whose collective is a snapshot of the slice."""
  from big_vision_b200.trainers.proj.image_text import siglip

  class Recorder(siglip.BucketedGradAllReduce):
    def _launch(self, lo, hi):
      for a, b in ([(lo, hi)] if self.ranges is None else
                   [(max(lo, r0), min(hi, r1)) for r0, r1 in self.ranges]):
        if b > a:
          self.snaps.append((a, b, self.P.grad[a:b].clone()))

    def broken(self):
      """The announced slices that changed afterwards."""
      return [(a, b) for a, b, s in self.snaps if not torch.equal(s, self.P.grad[a:b])]

  rec = Recorder(P, None, bucket_elems=1, ranges=ranges)
  rec.snaps = []
  return rec


# ---- the replay harness ------------------------------------------------------------------------------------
def _index_tree(P):
  """name -> flat-buffer indices, through the same storage and alias views as P.tree()."""
  I = torch.arange(P.total, device=P.device)
  aliased = {a.storage for a in P.aliases.values()}

  def view(name):
    off, shape = P.offsets[name]
    return I[off:off + int(np.prod(shape))].view(shape)

  out = {s.name: view(s.name) for s in P.specs if s.name not in aliased}
  out.update({a.name: a.view(view(a.storage)) for a in P.aliases.values()})
  return out


def _flat(t):
  if t is None:
    return []
  if isinstance(t, (tuple, list)):
    return [u for v in t for u in _flat(v)]
  return [t]


def _sink_of(st, P, geom):
  """The gradient buffer that equals the column sum of stage st's output gradient, which the stage above must
  accumulate that sum into (None: there is none): the MlpBlock Dense_1 bias of an encoder block, the
  channel-mixing Dense_1 bias of a Mixer block without stochastic depth (with it, the gradient entering the
  branch is mask * d output), the patch-embedding bias without [cls]."""
  from big_vision_b200.models import mlp_mixer, vit
  if isinstance(st, vit.ScanEncoder):
    st = st.blocks[-1]
  if isinstance(st, vit.EncoderBlock):
    g = P.g(st.p + "MlpBlock_0/Dense_1/bias")
    return g if st.index is None else g[st.index]
  if isinstance(st, mlp_mixer.MixerBlock):
    return None if geom.masks is not None else P.g(st.p + "channel_mixing/Dense_1/bias")
  if isinstance(st, vit.PatchEmbedding):
    return None if st.cls else P.g(st.w + "bias")
  return None


class Replay:
  """Wraps the stages of `model` for one forward + backward on P and checks each stage's backward.
  Faults for the planted-fault tests: `sink_from` {label: stage index whose sink is handed instead},
  `op_fault` {label: (ops function name, wrapper factory)} active during that stage's backward, `after`
  {label: fn()} run right after that stage's backward.  Labels: "i" for stage i, "i.j" for block j of a
  ScanEncoder at stage i."""

  def __init__(self, model, P, frozen=None, sink_from=None, op_fault=None, after=None, qk_allow=None):
    from big_vision_b200.models import vit
    self.model, self.P, self.frozen = model, P, frozen
    self.stages = model._stages   # pylint: disable=protected-access
    self.cut = model.cut(P, frozen)
    self.sink_from, self.op_fault, self.after = sink_from or {}, op_fault or {}, after or {}
    self.qk_allow = qk_allow or {}
    self.idx = _index_tree(P)
    self.failures, self.worst, self.calls, self.fwds = [], {}, [], {}
    self.checking = False
    self._wrapped = []
    for i, st in enumerate(self.stages):
      self._wrap(st, str(i), self._expected_sink(i))
      if isinstance(st, vit.ScanEncoder):
        for j, b in enumerate(st.blocks):
          self._wrap(b, f"{i}.{j}", None)

  # ---- wrapping
  def _expected_sink(self, i):
    """The sink the runner should hand stage i (from the model's structure, not the stages' sink methods)."""
    if i - 1 < self.cut:
      return lambda geom: None
    below = self.stages[i - 1]
    return lambda geom: _sink_of(below, self.P, geom)

  def _wrap(self, st, label, expected_sink):
    from big_vision_b200 import ops
    from big_vision_b200.models import vit
    fwd, bwd = st.fwd, st.bwd

    def wfwd(P, x, geom, save=True):
      y, saved = fwd(P, x, geom, save)
      if self.checking:
        self.fwds.setdefault(label, []).append((x, geom, y, saved))
      return y, saved

    def wbwd(P, dy, saved, geom, sink, need_dx=True):
      self.calls.append((label, need_dx))
      if not self.checking:
        return bwd(P, dy, saved, geom, sink, need_dx)
      if isinstance(st, vit.ScanEncoder):        # its blocks check themselves; hand block 0 the expected sink
        self._scan_sink = expected_sink(geom)
        self._scan_stage = st
      if label in self.sink_from:
        j = self.sink_from[label]
        sink = _sink_of(self.stages[j], P, geom)
      dy_in = dy.clone()
      patched = None
      if label in self.op_fault:
        name, make = self.op_fault[label]
        patched = (name, getattr(ops, name))
        setattr(ops, name, make(patched[1]))
      try:
        dx = bwd(P, dy, saved, geom, sink, need_dx)
      finally:
        if patched:
          setattr(ops, *patched)
      if label in self.after:
        self.after[label]()
      if not isinstance(st, vit.ScanEncoder):
        want = expected_sink(geom) if expected_sink is not None else self._block_sink(st, geom)
        self._check(label, st, self.fwds[label][-1][0], geom, dy_in, saved, sink, want, need_dx, dx)
      return dx

    st.fwd, st.bwd = wfwd, wbwd
    self._wrapped.append(st)

  def _block_sink(self, b, geom):
    blocks = self._scan_stage.blocks
    return _sink_of(blocks[b.index - 1], self.P, geom) if b.index else self._scan_sink

  def unwrap(self):
    for st in self._wrapped:
      del st.fwd, st.bwd

  # ---- running
  def run(self, x, kw, dout, ready=True):
    """Pass 1 (zeroed buffer, unchecked) sizes the seed of each storage to its gradient; pass 2 is the
    checked one."""
    P = self.P
    P.zero_grad()
    _run(self.model, P, x, kw, self.frozen, dout)
    scale = torch.ones(P.total, device=P.device)
    for name, (off, shape) in P.offsets.items():
      n = int(np.prod(shape))
      m = P.grad[off:off + n].abs().max()
      if float(m) > 0:
        scale[off:off + n] = m
    g = torch.Generator(device="cuda").manual_seed(7)
    mag = torch.rand(P.total, generator=g, device="cuda") * 0.5 + 0.5
    sign = torch.randint(0, 2, (P.total,), generator=g, device="cuda") * 2 - 1
    self.seed = mag * sign * scale
    self.seed64 = self.seed.to(F64)
    self.exp = self.seed.clone()
    self.final = torch.zeros(P.total, dtype=torch.bool, device=P.device)
    self.calls = []
    self.rec = ready_recorder(P, P.trained_ranges(self.frozen) if self.frozen else None) if ready else None

    def seed():
      P.grad.copy_(self.seed)
      if self.rec is not None:
        self.rec.begin()

    self.checking = True
    try:
      _run(self.model, P, x, kw, self.frozen, dout, before_bwd=seed)
    finally:
      self.checking = False
      if self.rec is not None:
        self.rec.finish()
    self._after_backward()
    return self

  def _after_backward(self):
    if not torch.equal(self.P.grad, self.exp):
      self._fail(4, "end", f"{int((self.P.grad != self.exp).sum())} elements changed outside the final ranges")
    # 5: remat
    for label, recs in self.fwds.items():
      if "." in label:
        if len(recs) != 2:
          self._fail(5, label, f"{len(recs)} forward calls, want forward + recompute")
          continue
        (_, _, y0, s0), (_, _, y1, s1) = recs
        if not all(torch.equal(a, b) for a, b in zip([y0] + _flat(s0), [y1] + _flat(s1))):
          self._fail(5, label, "the recomputed block differs from its forward")
    # 6: the frozen cut
    called = {}
    for label, need_dx in self.calls:
      called.setdefault(label.split(".")[0], need_dx)
    for i in range(len(self.stages)):
      if i < self.cut and str(i) in called:
        self._fail(6, str(i), "stage below the frozen cut ran a backward")
      if i >= self.cut and str(i) not in called:
        self._fail(6, str(i), "stage above the cut ran no backward")
    if self.cut and called.get(str(self.cut)) is not False:
      self._fail(6, str(self.cut), "the stage at the cut was asked for dx")
    if self.rec is not None:
      for a, b in self.rec.broken():
        self._fail("ready", "-", f"slice [{a}, {b}) changed after it was announced final")

  def _fail(self, check, label, msg):
    self.failures.append((check, label, msg))

  # ---- one stage's checks
  def _note(self, kind, key, v):
    w = self.worst.setdefault(kind, {})
    w[key] = max(w.get(key, 0.0), v)

  def _compare(self, check, label, kind, what, got, ref, floor=None):
    """The bounds of the module docstring; `floor` (shaped like ref) is added per element to the element-wise
    bound, and its norm to the normwise one."""
    tau, tau_max = TOL[kind]
    got, ref = got.reshape(ref.shape).to(F64), ref.detach()
    if not bool(torch.isfinite(got).all()):
      self._fail(check, label, f"{what}: {int((~torch.isfinite(got)).sum())} non-finite elements")
      return
    err = got - ref
    rn, rm = float(ref.norm()), float(ref.abs().max()) if ref.numel() else 0.0
    en, em = float(err.norm()), float(err.abs().max()) if err.numel() else 0.0
    if rn == 0.0:
      if en != 0.0:
        self._fail(check, label, f"{what}: {en:.3g} where the reference is exactly zero")
      return
    self._note(kind, "norm", en / rn)
    self._note(kind, "max", em / rm)
    if floor is not None:
      floor = floor.reshape(ref.shape)
      r = float((err.abs() / (tau_max * rm + floor)).max())
      self._note(kind, "qk_floor", max(r, en / (tau * rn + float(floor.norm()))))
      allow = self.qk_allow.get(kind, 1.0)
      if not (en <= allow * (tau * rn + float(floor.norm())) and r <= allow):
        self._fail(check, label, f"{what}: normwise {en / rn:.3g}, max {em / rm:.3g}; {r:.3g} x its bound with the dS floor")
      return
    if not (en <= tau * rn and em <= tau_max * rm):
      self._fail(check, label, f"{what}: normwise {en / rn:.3g} (tau {tau:.3g}), max {em / rm:.3g} "
                               f"(tau_max {tau_max:.3g})")

  def _names(self, st):
    """(root, {name relative to the stage's root: flat-buffer indices}) of the tree names the stage owns."""
    root = st.p
    own = {}
    for name, ix in self.idx.items():
      if name.startswith(st.prefixes):
        if getattr(st, "index", None) is not None:
          ix = ix[st.index]
        own[name[len(root):]] = ix
    return root, own

  def _check(self, label, st, x, geom, dy, saved, sink, want_sink, need_dx, dx):
    from big_vision_b200.models import common, mlp_mixer, vit
    from big_vision_b200.models.proj.flexi import vit as fv
    from big_vision_b200.models.proj.image_text import text_transformer as tt
    P, n, N = self.P, geom.n, geom.N
    kind = type(st).__name__
    root, own = self._names(st)
    g = P.grad.to(F64)
    # --- the reference, on what the kernels read
    resampled = False
    if isinstance(st, fv.FlexiPatchEmbedding):
      seqhw = math.isqrt(N - st.cls)
      resampled = x.shape[1] // seqhw != st.patch_size[0] or (seqhw, seqhw) != st.posemb_size
    h = P.tree("h")
    f = P.tree("f")

    def value(rel):
      full = root + rel
      use_h = rel.endswith("kernel") or rel == "probe" or (rel == "pos_embedding" and isinstance(st, vit.PatchEmbedding))
      t = (f if resampled or not use_h else h)[full]
      if getattr(st, "index", None) is not None:
        t = t[st.index]
      return t.to(F64).clone().requires_grad_(True)

    p = {rel: value(rel) for rel in own}
    xin = None
    tap = None
    scores = S.ScoreGrad()
    if kind in EXACT_ZERO:
      zname, zshape = EXACT_ZERO[kind]
      tap = S.Tap(p[zname], zshape(st, n, N))
    if isinstance(st, (vit.PatchEmbedding, tt._Embed)):     # pylint: disable=protected-access
      xin = x if isinstance(st, tt._Embed) else x.to(torch.bfloat16).to(F64)   # pylint: disable=protected-access
    else:
      xin = (common.to16(x) if isinstance(st, common.Dense) else x).to(F64).requires_grad_(True)
    if isinstance(st, fv.FlexiPatchEmbedding):
      pos = p.get("pos_embedding")
      if st.posemb == "sincos2d":
        pos = (st._sincos32 if resampled else st._sincos).to(F64)   # pylint: disable=protected-access
      y = S.flexi_patch_embedding(xin, p, math.isqrt(N - st.cls), st.posemb_size, pos, st.cls)
    elif isinstance(st, vit.PatchEmbedding):
      pos = p.get("pos_embedding")
      if st.posemb == "sincos2d":
        pos = st._sincos.to(F64)   # pylint: disable=protected-access
      y = S.patch_embedding(xin, p, st.w[len(root):-1], pos, st.cls)
    elif isinstance(st, tt._Embed):   # pylint: disable=protected-access
      y = S.text_embed(xin, p)
    elif isinstance(st, vit.EncoderBlock):
      with tap, scores:
        y = S.encoder_block(xin.view(n, N, -1), p, st.heads)
    elif isinstance(st, mlp_mixer.MixerBlock):
      m = None if geom.masks is None else (geom.masks[st.i, 0].to(F64), geom.masks[st.i, 1].to(F64))
      with tap:
        y = S.mixer_block(xin.view(n, N, -1), p, m)
    elif isinstance(st, vit.NormPool):
      sel = saved[3].view(n, N, -1).to(F64) if st.pool == "max" else None
      y = S.norm_pool(xin.view(n, N, -1), p, st.pool, sel)
    elif isinstance(st, vit.MAPHead):
      with tap, scores:
        y = S.map_head(xin.view(n, N, -1), p, st.heads)
    elif isinstance(st, common.Dense):
      y = S.dense(xin, p, st.tanh)
      dy = dy[:, :st.C]
    else:
      raise NotImplementedError(f"no reference for stage {kind}")
    y.backward(dy.to(F64).reshape(y.shape))
    dx_ref = xin.grad
    bound = {}
    if kind in QK_FLOOR:
      fq, fk = scores.floors()
      if kind == "EncoderBlock":
        ln1 = saved[1].to(F64).abs().view(n * N, -1)
        fq, fk = fq.reshape(n * N, -1), fk.reshape(n * N, -1)
        bound = {QK[0]: ln1.T @ fq, QK[1]: fq.sum(0), QK[2]: ln1.T @ fk}
      else:
        fq1 = fq.reshape(n, -1).sum(0)
        bound = {QK[0]: p["probe"].detach().abs().reshape(-1, 1) * fq1, QK[1]: fq1,
                 QK[2]: xin.detach().abs().view(n * N, -1).T @ fk.reshape(n * N, -1),
                 "probe": p[QK[0]].detach().abs().reshape(st.d, st.d) @ fq1}
    # 1. dx
    if need_dx and dx_ref is not None:
      if dx is None:
        self._fail(1, label, "no dx returned")
      else:
        self._compare(1, label, kind, "dx", dx, dx_ref)
    # 2. own parameters
    allowed = torch.zeros_like(self.final)
    for rel, ix in own.items():
      ref = p[rel].grad if p[rel].grad is not None else torch.zeros_like(p[rel])
      got = g[ix] - self.seed64[ix]
      if tap is not None and rel == EXACT_ZERO[kind][0]:
        e, fl = (got - ref).abs(), ZERO_FLOOR * tap.floor()
        r = float(torch.where(fl > 0, e / fl.clamp_min(1e-300), torch.where(e > 0, math.inf, 0.0)).max())
        self._note(kind, "zero_floor", r)
        if not r <= 1:
          self._fail(2, label, f"{rel}: {r:.3g} x the floor")
      else:
        self._compare(2, label, kind, rel, got, ref, bound.get(rel))
      allowed[ix.reshape(-1)] = True
    allowed &= ~self.final
    # 3. the sink
    ptr = lambda t: None if t is None else t.data_ptr()
    if ptr(sink) != ptr(want_sink):
      self._fail(3, label, "handed a sink other than the stage below's")
    if want_sink is not None:
      a = (want_sink.data_ptr() - P.grad.data_ptr()) // 4
      b = a + want_sink.numel()
      self._compare(3, label, kind, "sink", g[a:b] - self.seed64[a:b], dx_ref.reshape(-1, b - a).sum(0))
      allowed[a:b] = True
    # 4. nothing else moved
    moved = (P.grad != self.exp) & ~allowed
    if bool(moved.any()):
      self._fail(4, label, f"{int(moved.sum())} elements written outside the stage's own range and its sink")
    self.exp[allowed] = P.grad[allowed]
    self.final |= allowed


def _replay(case, **faults):
  model = build_model(case)
  P = _params(model, case)
  x, kw = _inputs(model, case)
  frozen = frozen_set(model, P, case)
  out, _ = model.fwd(P, x, frozen=True, **kw)
  dout = _dout(model, out)
  rep = Replay(model, P, frozen, qk_allow=CASES[case][3].get("qk_allow"), **faults)
  try:
    return rep.run(x, kw, dout)
  finally:
    rep.unwrap()


def _report(case, rep):
  print(json.dumps({f"stage_replay_{case}": {k: {m: float(f"{v:.4g}") for m, v in w.items()}
                                             for k, w in sorted(rep.worst.items())}}))


@pytest.mark.parametrize("case", list(CASES))
def test_every_stage_matches_its_fp64_reference(case):
  rep = _replay(case)
  _report(case, rep)
  assert not rep.failures, rep.failures[:10]
  kinds = {type(s).__name__ for s in rep.stages[rep.cut:]}
  assert set(rep.worst) >= kinds - {"ScanEncoder"}, (kinds, set(rep.worst))


def test_siglip_two_tower_ready_announcements_hold_their_final_bits():
  """Both towers in one FlatParams (spec order: image, text, t, b): every slice announced during
  siglip.loss_and_grads' backward is final."""
  import common
  from big_vision_b200.models.proj.image_text import two_towers
  from big_vision_b200.trainers.proj.image_text import siglip
  model = two_towers.Model(**common.TINY)
  P = model.init(0, common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE, device="cuda")
  image, text = common.synthetic_batch(common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE, 64)
  rec = ready_recorder(P)
  rec.begin()
  siglip.loss_and_grads(model, P, torch.from_numpy(image).cuda(), torch.from_numpy(text).cuda())
  rec.finish()
  torch.cuda.synchronize()
  assert len(rec.snaps) >= 4           # two blocks per tower, then the rest
  assert not rec.broken()


# ---- planted faults: each is caught by the check named, and the clean run passes ------------------------------
def _checks(rep):
  return {c for c, _, _ in rep.failures}


def _once(pred, change):
  """A wrapper factory for an ops function: the first call that satisfies pred(kwargs) gets change(...)."""
  def make(fn):
    done = [False]

    def wrapped(*args, **kw):
      if not done[0] and pred(kw):
        done[0] = True
        return change(fn, args, kw)
      return fn(*args, **kw)
    return wrapped
  return make


# Each fault runs on a case whose clean run is test_every_stage_matches_its_fp64_reference[case].
def test_fault_wrong_sink_is_caught():
  # block 1 (stage 2) handed the patch embedding's bias (stage 0's sink) instead of block 0's
  rep = _replay("vit_gap_sincos", sink_from={"2": 0})
  assert _checks(rep) & {3, 4}, rep.failures


def test_fault_missing_dres_is_caught():
  rep = _replay("vit_tok", op_fault={"2": ("layernorm_bwd", _once(lambda kw: kw.get("dres") is not None,
                                                                 lambda fn, a, kw: fn(*a, **{**kw, "dres": None})))})
  assert 1 in _checks(rep), rep.failures


def test_fault_overwriting_wgrad_is_caught():
  """Without the seed this fault is invisible: the buffer would start at zero."""
  rep = _replay("mixer", op_fault={"2": ("gemm", _once(lambda kw: kw.get("reduce_out"),
                                                      lambda fn, a, kw: fn(*a, **{**kw, "reduce_out": False})))})
  assert 2 in _checks(rep), rep.failures


def test_fault_colsum_twice_is_caught():
  def twice(fn, a, kw):
    fn(*a, **kw)
    return fn(*a, **kw)
  # the MAP head's first column sum (its MlpBlock's Dense_1 bias), counted twice
  rep = _replay("vit_map", op_fault={"4": ("colsum", _once(lambda kw: True, twice))})
  assert 2 in _checks(rep), rep.failures


def test_fault_write_after_ready_is_caught():
  holder = {}

  def bump():
    a = holder["rep"].rec.snaps[-1][0]       # the first element of the slice announced last
    P = holder["rep"].P
    P.grad[a] = torch.nextafter(P.grad[a], torch.tensor(math.inf, device=P.device))

  # after block 1 (stage 2) announced its slice, block 0's backward adds one ulp to it
  model = build_model("vit_tok")
  P = _params(model, "vit_tok")
  x, kw = _inputs(model, "vit_tok")
  out, _ = model.fwd(P, x, frozen=True)
  rep = holder["rep"] = Replay(model, P, None, after={"1": bump})
  try:
    rep.run(x, kw, _dout(model, out))
  finally:
    rep.unwrap()
  assert "ready" in _checks(rep), rep.failures


def test_fault_mixer_sink_kept_under_stochastic_depth_is_caught():
  """MixerBlock_1 (stage 2) drops sample 3's channel-mixing branch.  Kept as a sink, its channel-mixing Dense_1
  bias gets colsum(d output) from the block above instead of colsum(mask * d output): wrong by sample 3's rows."""
  model = build_model("mixer_stoch")
  P = _params(model, "mixer_stoch")
  x, kw = _inputs(model, "mixer_stoch")
  assert float(kw["masks"][1, 1].min()) == 0.0
  out, _ = model.fwd(P, x, frozen=True, **kw)
  block = model._stages[2]     # pylint: disable=protected-access
  block.sink = lambda P_, geom: P_.g(block.cm + "Dense_1/bias")
  rep = Replay(model, P, None)
  try:
    rep.run(x, kw, _dout(model, out))
  finally:
    rep.unwrap()
    del block.sink
  assert 3 in _checks(rep), rep.failures
  # and numerically, not only by which buffer was handed over
  assert any(c == 2 and lbl == "2" and m.startswith("channel_mixing/Dense_1/bias:") for c, lbl, m in rep.failures), \
      rep.failures
