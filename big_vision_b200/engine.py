"""Flat parameter storage shared by the models, the backward pass and the optimizer.

All parameters of a model live in ONE fp32 buffer (`flat`), their gradients in a second
buffer of the same layout (`grad`) and a bf16 shadow copy (`half`) that the tensor-core
GEMMs read.  One flat layout means: one fused optimizer launch per parameter group, one
bucketed NCCL all-reduce over `grad`, one zero-fill per step.  Parameters are addressed
by the reference's tree names (`img/Transformer/encoderblock_0/...`, see SURVEY.md 8b);
fused storage (q|k|v in one [d, 3d] matrix) is exposed through strided views so the
reference names and shapes still resolve.
"""
import re
from dataclasses import dataclass
from typing import Callable, Dict, List, NamedTuple, Optional, Tuple

import numpy as np
import torch


@dataclass
class ParamSpec:
  name: str                      # storage name ("a/b/c")
  shape: Tuple[int, ...]         # storage shape
  init: Callable                 # init(rng: np.random.Generator, shape) -> np.ndarray (fp32)


@dataclass
class Alias:
  """A reference-named view into a stored parameter."""
  name: str
  storage: str
  view: Callable                 # torch storage tensor -> torch view with the reference shape


ALIGN = 8  # elements: 32 B in fp32, 16 B in bf16 (TMA base alignment)


class FlatParams:
  """fp32 master params + grads + bf16 shadow in three flat device buffers."""

  def __init__(self, specs: List[ParamSpec], aliases: List[Alias], device, decay_regex=r".*/kernel$"):
    self.specs = specs
    self.aliases = {a.name: a for a in aliases}
    self.device = torch.device(device)
    # decayed parameters first, so weight decay is one contiguous launch range
    # (optax.py:133 default mask `.*/kernel$`).
    rx = re.compile(decay_regex) if decay_regex else None
    alias_by_storage: Dict[str, List[str]] = {}
    for a in aliases:
      alias_by_storage.setdefault(a.storage, []).append(a.name)

    def decayed(s):
      if rx is None:
        return False
      names = alias_by_storage.get(s.name, [s.name])
      return any(rx.match(n) for n in names)

    order = [s for s in specs if decayed(s)] + [s for s in specs if not decayed(s)]
    self.offsets: Dict[str, Tuple[int, Tuple[int, ...]]] = {}
    off = 0
    for s in order:
      self.offsets[s.name] = (off, tuple(s.shape))
      n = int(np.prod(s.shape))
      off += (n + ALIGN - 1) // ALIGN * ALIGN
      if decayed(s):
        self.n_decay = off
    if not hasattr(self, "n_decay"):
      self.n_decay = 0
    self.total = off
    self.flat = torch.zeros(self.total, dtype=torch.float32, device=self.device)
    self.grad = torch.zeros(self.total, dtype=torch.float32, device=self.device)
    self.half = torch.zeros(self.total, dtype=torch.bfloat16, device=self.device)
    self._views = {}

  def twin(self):
    """A second parameter set with the same specs, aliases and flat layout but its own zeroed `flat`,
    `grad` and `half` buffers (10 bytes per element): model code runs on it unchanged, e.g. on the
    perturbed weights of a GSAM / SAM step."""
    t = object.__new__(FlatParams)
    t.specs, t.aliases, t.device = self.specs, self.aliases, self.device
    t.offsets, t.n_decay, t.total = self.offsets, self.n_decay, self.total
    t.flat = torch.zeros_like(self.flat)
    t.grad = torch.zeros_like(self.grad)
    t.half = torch.zeros_like(self.half)
    t._views = {}
    return t

  def drop_grad(self):
    """Releases the gradient buffer, 4 of the 10 bytes per parameter, of a model that only ever runs
    forward (`fwd(..., frozen=True)` / `apply()`), e.g. a distillation teacher."""
    self.grad = None
    self._views = {k: v for k, v in self._views.items() if k[0] != "g"}
    return self

  # ---- raw views ------------------------------------------------------------------
  def _view(self, buf, name):
    off, shape = self.offsets[name]
    n = int(np.prod(shape))
    return buf[off:off + n].view(shape)

  def f(self, name):
    """fp32 master view of storage parameter `name`."""
    key = ("f", name)
    if key not in self._views:
      self._views[key] = self._view(self.flat, name)
    return self._views[key]

  def g(self, name):
    key = ("g", name)
    if key not in self._views:
      self._views[key] = self._view(self.grad, name)
    return self._views[key]

  def h(self, name):
    key = ("h", name)
    if key not in self._views:
      self._views[key] = self._view(self.half, name)
    return self._views[key]

  # ---- init / interchange ---------------------------------------------------------
  def init(self, seed=0):
    rng = np.random.default_rng(seed)
    host = np.zeros(self.total, dtype=np.float32)
    for s in self.specs:
      off, shape = self.offsets[s.name]
      n = int(np.prod(shape))
      host[off:off + n] = np.asarray(s.init(rng, tuple(shape)), dtype=np.float32).reshape(-1)
    self.flat.copy_(torch.from_numpy(host))
    self.sync_half()
    return self

  def sync_half(self):
    """Refreshes the bf16 shadow from the fp32 master (the optimizer kernel does this itself)."""
    if self.flat.is_cuda:
      from big_vision_b200 import ops
      ops.cast(self.flat, self.half)
    else:
      self.half.copy_(self.flat)

  def tree(self, which="f"):
    """dict: reference name -> tensor view (params 'f', grads 'g')."""
    out = {}
    aliased = {a.storage for a in self.aliases.values()}
    get = {"f": self.f, "g": self.g, "h": self.h}[which]
    for s in self.specs:
      if s.name not in aliased:
        out[s.name] = get(s.name)
    for a in self.aliases.values():
      out[a.name] = a.view(get(a.storage))
    return out

  def load_tree(self, tree: Dict[str, "np.ndarray"]):
    """Copies a reference-named tree (numpy / torch, reference shapes) into the flat buffer."""
    views = self.tree("f")
    missing = [k for k in views if k not in tree]
    if missing:
      raise KeyError(f"missing parameters: {missing[:5]}{'...' if len(missing) > 5 else ''}")
    for k, v in views.items():
      src = torch.as_tensor(np.asarray(tree[k], dtype=np.float32)).to(self.device)
      v.copy_(src.reshape(v.shape))
    self.sync_half()
    return self

  def numpy_tree(self, which="f"):
    return {k: v.detach().float().cpu().numpy().copy() for k, v in self.tree(which).items()}

  def zero_grad(self):
    self.grad.zero_()

  def trained_ranges(self, frozen):
    """[(lo, hi), ...]: the flat-buffer slices of every stored parameter NOT in `frozen` (storage
    names), each with its alignment padding, neighbours merged, in layout order."""
    out = []
    for name, (off, shape) in sorted(self.offsets.items(), key=lambda kv: kv[1][0]):
      if name in frozen:
        continue
      hi = off + (int(np.prod(shape)) + ALIGN - 1) // ALIGN * ALIGN
      if out and out[-1][1] == off:
        out[-1][1] = hi
      else:
        out.append([off, hi])
    return [tuple(r) for r in out]


def stage_cut(storages, stages, frozen):
  """Index of the lowest of `stages` (bottom-up; each a tuple of storage-name prefixes) that holds a
  storage not in `frozen`: a backward that stops there still reaches every trained parameter.
  len(stages) when everything is frozen; 0 when nothing is (`frozen` empty or None).  `frozen=True`
  means every storage."""
  if frozen is True:
    return len(stages)
  if not frozen:
    return 0
  for i, prefixes in enumerate(stages):
    if any(s.startswith(prefixes) and s not in frozen for s in storages):
      return i
  return len(stages)


class Geom(NamedTuple):
  """What every stage of one forward sees besides its input: n samples of N tokens each, and the
  MLP-Mixer's stochastic-depth masks of that forward (None: no residual branch is dropped)."""
  n: int
  N: int
  masks: Optional[torch.Tensor] = None


class Stage:
  """Defaults of a backward stage (see Staged)."""
  ready = None

  def sink(self, P, geom):
    return None


class Staged:
  """A model built as `self._stages`, a bottom-up list of backward stages (Stage), which the model's
  specs() builds once the input geometry is known (_build).  Each stage has
    `prefixes`: the storage-name prefixes of its parameters;
    `specs() -> (specs, aliases)`: its parameters;
    `fwd(P, x, geom, save) -> (y, saved)`: `geom` is the forward's Geom; with save=False it keeps
        nothing (saved is None) and frees each intermediate once it has been consumed;
    `bwd(P, dy, saved, geom, sink, need_dx) -> dx`: accumulates its parameter gradients; `sink` (or
        None) receives colsum(dx), and with need_dx=False dx is not computed and None is returned;
    `sink(P, geom)`: the gradient buffer that equals the column sum of the stage's output gradient, or
        None;
    `ready`: None, or the storage name from which on (in spec order) every gradient is final once the
        stage's backward has run (P.on_ready, the bucketed gradient all-reduce)."""

  def _build(self, stages):
    """Makes `stages` the model's stage list -> (specs, aliases) of all their parameters, in stage order."""
    self._stages = stages
    specs, aliases = [], []
    for stage in stages:
      s, a = stage.specs()
      specs += s
      aliases += a
    return specs, aliases

  def stages(self):
    """The stages' storage-name prefixes, bottom-up."""
    return [s.prefixes for s in self._stages]

  def cut(self, P, frozen):
    """Index into stages() of the lowest stage with a trained parameter (stage_cut): the backward stops
    there and everything below runs forward-only.  len(stages()) = wholly frozen."""
    cache = self.__dict__.setdefault("_cuts", {})
    key = frozen if frozen is True or frozen is None else frozenset(frozen)
    if key not in cache:
      cache[key] = stage_cut(P.offsets, self.stages(), frozen)
    return cache[key]

  def _stages_fwd(self, P, x, geom, frozen):
    """Runs every stage; those below the cut save nothing.  -> (output, saved for _stages_bwd)."""
    cut = self.cut(P, frozen)
    saved = []
    for i, stage in enumerate(self._stages):
      x, s = stage.fwd(P, x, geom, i >= cut)
      saved.append(s)
    return x, {"stages": saved, "geom": geom, "cut": cut}

  def _stages_bwd(self, P, dy, saved):
    """Runs the backward from the top stage down to the cut, dropping each stage's saved tensors once
    its backward is done."""
    stages, kept, geom, cut = self._stages, saved["stages"], saved["geom"], saved["cut"]
    on_ready = getattr(P, "on_ready", None)
    for i in reversed(range(cut, len(stages))):
      sink = stages[i - 1].sink(P, geom) if i - 1 >= cut else None
      dy = stages[i].bwd(P, dy, kept[i], geom, sink, i > cut)
      kept[i] = None
      if on_ready is not None and stages[i].ready is not None:
        on_ready(stages[i].ready)


# ---- initialisers (numpy; same distributions as the reference's, see SURVEY.md 3.4) -------
def xavier_uniform(fan_in, fan_out):
  def init(rng, shape):
    lim = np.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-lim, lim, size=shape)
  return init


def lecun_normal(fan_in):
  def init(rng, shape):
    # flax lecun_normal = variance_scaling(1.0, "fan_in", "truncated_normal")
    std = np.sqrt(1.0 / fan_in) / 0.87962566103423978
    x = rng.standard_normal(size=shape)
    bad = np.abs(x) > 2
    while bad.any():
      x[bad] = rng.standard_normal(size=int(bad.sum()))
      bad = np.abs(x) > 2
    return x * std
  return init


def normal(std):
  return lambda rng, shape: rng.standard_normal(size=shape) * std


def zeros(rng, shape):
  return np.zeros(shape, dtype=np.float32)


def ones(rng, shape):
  return np.ones(shape, dtype=np.float32)


def constant(v):
  return lambda rng, shape: np.full(shape, v, dtype=np.float32)
