"""CPU: BERT dropout.  The attention-dropout arguments of include/bv_dropout.h (every refusal before any
launch; their layout and the BV_ATTN_DROPOUT mirror are checked with the other headers' in
tests/test_abi.py), the numpy restatement of the attention mask stream (numpy's Philox in 16-bit lanes, its
realized rate, and its separation from every bv_dropout counter and from Jet's), the float64 BERT oracle
with given masks pinned against `transformers.BertModel` in train mode with the same masks, and what the
BERT tower launches and keeps with dropout, recorded by tests/golden/make_model_traces.py's recorder."""
import ctypes
import importlib.util
import math
import os
import re

import numpy as np
import pytest
import torch

import bert_dropout_oracle as BD
import bert_oracle as BO
import dropout_oracle as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the C ABI -------------------------------------------------------------------------------------------
def _key(**kw):
  from big_vision_b200 import lib as L
  return L.DropoutKey(**{"seed": 1, "step": 2, "site": 3, "row0": 0, "rate": 0.1, **kw})


_MASK = (ctypes.c_uint8 * 64)(*([1] * 64))


@pytest.mark.parametrize("what,flags,kw,mask,message", [
    ("no key mask flag", 64, {}, True, "needs BV_ATTN_KEY_MASK"),
    ("head dim 72", 72 | 65536, {}, True, "head_dim 64 only"),
    ("head dim 104", 104 | 65536, {}, True, "head_dim 64 only"),
    ("site 0", 64 | 65536, dict(site=0), True, "site 0"),
    ("rate < 0", 64 | 65536, dict(rate=-0.1), True, "outside [0, 1)"),
    ("rate 1", 64 | 65536, dict(rate=1.0), True, "outside [0, 1)"),
    ("rate nan", 64 | 65536, dict(rate=float("nan")), True, "outside [0, 1)"),
    ("row0 < 0", 64 | 65536, dict(row0=-1), True, "row0"),
    ("null key mask", 64 | 65536, {}, False, "non-null key_mask"),
])
@pytest.mark.parametrize("direction", ["fwd", "bwd"])
def test_attention_dropout_refusals(what, flags, kw, mask, message, direction):
  """Every refusal returns BV_ERR_INVALID, names the entry point and launches nothing (no device here)."""
  from big_vision_b200 import lib as L
  lib = L.load()
  km = ctypes.cast(_MASK, ctypes.c_void_p) if mask else None
  if direction == "fwd":
    a = L.AttnDropoutArgs(masked=L.AttnMaskedArgs(key_mask=km, bsmask=64), drop=_key(**kw))
    rc, fn = lib.bv_attention_fwd_hd(ctypes.byref(a.masked.attn), flags | L.ATTN_DROPOUT, None), "bv_attention_fwd_hd"
  else:
    a = L.AttnDropoutBwdArgs(masked=L.AttnMaskedBwdArgs(key_mask=km, bsmask=64), drop=_key(**kw))
    rc, fn = lib.bv_attention_bwd_hd(ctypes.byref(a.masked.attn), flags | L.ATTN_DROPOUT, None), "bv_attention_bwd_hd"
  assert rc == -1, what
  err = lib.bv_last_error_string().decode()
  assert err.startswith(fn + ":") and message in err, err


def test_null_args_with_the_flag_are_refused():
  from big_vision_b200 import lib as L
  lib = L.load()
  for fn in ("bv_attention_fwd_hd", "bv_attention_bwd_hd"):
    assert getattr(lib, fn)(None, 64 | L.ATTN_KEY_MASK | L.ATTN_DROPOUT, None) == -1
    assert lib.bv_last_error_string().decode() == f"{fn}: null args"


def test_ops_refuse_dropout_without_a_key_mask():
  from big_vision_b200 import lib as L, ops
  q = torch.zeros((1, 16, 64), dtype=torch.bfloat16)
  with pytest.raises(L.BvError, match="key_mask"):
    ops.attention_fwd(q, q, q, 1, dropout=_key())


# ---- the attention mask stream --------------------------------------------------------------------------
def test_the_attention_stream_is_numpys_philox_in_16_bit_lanes():
  Nk = 40                                    # three blocks, the last one partly used
  raw = np.random.Philox(key=11, counter=[0, 4, 9, 6]).random_raw(12)   # row 5: counter word 3 = 6
  got = BD.attn_lanes(11, 4, 9, 5, Nk)
  assert got.shape == (Nk,)
  for k in range(Nk):
    assert got[k] == (int(raw[4 * (k // 16) + (k % 16) // 4]) >> (16 * (k % 4))) & 0xFFFF
  # block b sits at counter (b + 1, step, site, row + 1): numpy increments word 0 before each block
  w = np.random.Philox(key=11, counter=[2, 4, 9, 6]).random_raw(4)
  assert np.array_equal(w, raw[8:12])


def test_rows_follow_the_global_batch_layout():
  """Probability (b, h, q, k) is row row0 + (b H + h) Nq + q, so a slice of samples called with
  row0 = b0 H Nq draws that slice of the whole batch's masks."""
  B, H, N, rate = 4, 3, 20, 0.3
  whole = BD.attn_keep(7, 1, 5, 0, B, H, N, N, rate)
  assert np.array_equal(BD.attn_keep(7, 1, 5, 2 * H * N, 2, H, N, N, rate), whole[2:])
  assert np.array_equal(whole[1, 2, 3], BD.attn_lanes(7, 1, 5, (1 * H + 2) * N + 3, N) >= D.threshold(rate))


@pytest.mark.parametrize("rate", [0.1, 0.5])
def test_realized_rate_is_within_the_binomial_bound(rate):
  keep = BD.attn_keep(3, 9, 17, 0, 2, 12, 128, 512, rate)
  n = keep.size
  p = D.threshold(rate) / 65536
  assert abs(float((~keep).mean()) - p) <= 5 * math.sqrt(p * (1 - p) / n)


def test_no_attention_counter_meets_a_dropout_or_jet_counter():
  """bv_dropout draws at counter word 3 = 0 and Jet's noise at words 2 = 3 = 0; every attention counter has
  word 3 = row + 1 >= 1.  So the attention stream of a layer shares its DROP_ATTN site with the attention
  output's dropout and never draws its blocks."""
  from big_vision_b200 import engine as E
  site = E.dropout_site(1, 0, E.DROP_ATTN)
  attn = np.concatenate([BD.attn_lanes(5, 3, site, r, 64) for r in range(64)]).view("<u8")
  hidden = D.lanes(5, 3, site, 0, 64 * 64).view("<u8")
  jet = np.random.Philox(key=5, counter=[0, 3, 0, 0]).random_raw(attn.size)
  assert not set(attn.tolist()) & set(hidden.tolist())
  assert not set(attn.tolist()) & set(jet.tolist())


# ---- the float64 oracle with masks, pinned against transformers ------------------------------------------
TINY = dict(width=128, depth=2, num_heads=2, mlp_dim=256, vocab_size=97)
N_TOK, BATCH, CLASSES = 16, 6, 24


def _random_masks(rate, attn_rate, seed, n, N, d, heads, depth):
  """Scaled float64 masks of every site, from a numpy generator (any masks: the pin is on their placement)."""
  from big_vision_b200 import engine as E
  rng = np.random.default_rng(seed)
  hidden = {}
  for layer, kind in [(0, E.DROP_EMBED)] + [(i, k) for i in range(depth) for k in (E.DROP_ATTN, E.DROP_MLP)]:
    hidden[(layer, kind)] = BD.scaled(rng.random((n, N, d)) >= rate, rate)
  probs = [BD.scaled(rng.random((n, heads, N, N)) >= attn_rate, attn_rate) for _ in range(depth)]
  return BD.GivenMasks(hidden, probs)


def test_oracle_with_masks_matches_transformers_bert_in_train_mode(monkeypatch):
  """The same masks placed in `transformers.BertModel` (eager, train mode) by replacing its three nn.Dropout
  modules per layer and `nn.functional.dropout` on the attention probabilities: [CLS] output within 1e-9 and
  every parameter gradient within 1e-8 (relative to the tensor's max), float64, with padded captions."""
  pytest.importorskip("transformers")
  import test_bert as TB
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.flaxformer import bert
  model = bert.Model(dict(TINY, dropout_rate=0.1, attention_dropout_rate=0.1), num_classes=CLASSES,
                     head_zeroinit=False)
  tree = TB.random_tree(model, N_TOK, seed=3)
  text = torch.from_numpy(BO.padded_text(BATCH, N_TOK, TINY["vocab_size"], seed=4)).long()
  cot = torch.from_numpy(np.random.default_rng(5).standard_normal((BATCH, CLASSES)))
  cfg = dict(depth=TINY["depth"], num_heads=TINY["num_heads"], num_classes=CLASSES)
  masks = _random_masks(0.3, 0.2, 6, BATCH, N_TOK, TINY["width"], TINY["num_heads"], TINY["depth"])

  leaves = TB._leaves(tree)   # pylint: disable=protected-access
  ours = BD.bert_forward(leaves, text, cfg, masks)
  (ours * cot).sum().backward()
  # without the masks the output differs: they are applied
  assert (BO.bert_forward(TB._leaves(tree), text, cfg) - ours).abs().max() > 1e-3   # pylint: disable=protected-access

  hf, sd = TB._hf_model(tree, TINY, TINY["vocab_size"])   # pylint: disable=protected-access
  hf.train()

  class Given(torch.nn.Module):
    def __init__(self, m):
      super().__init__()
      self.m = m

    def forward(self, x):
      return x * self.m

  hf.embeddings.dropout = Given(masks.h[(0, E.DROP_EMBED)])
  for i, layer in enumerate(hf.encoder.layer):
    layer.attention.output.dropout = Given(masks.h[(i, E.DROP_ATTN)])
    layer.output.dropout = Given(masks.h[(i, E.DROP_MLP)])
  calls = []

  def probs_dropout(x, p=0.5, training=True, inplace=False):
    assert training and p == pytest.approx(0.1)
    calls.append(len(calls))
    return x * masks.p[calls[-1]]

  from transformers.models.bert import modeling_bert
  monkeypatch.setattr(modeling_bert.nn.functional, "dropout", probs_dropout)
  kernel, bias = (torch.tensor(np.asarray(tree[k], dtype=np.float64), requires_grad=True)
                  for k in ("head/kernel", "head/bias"))
  for layer in hf.encoder.layer:     # the rate the attention passes to nn.functional.dropout in train mode
    layer.attention.self.dropout.p = 0.1
  out = hf(input_ids=text, attention_mask=(text != 0).long(), token_type_ids=torch.zeros_like(text))
  assert calls == list(range(TINY["depth"]))
  theirs = out.last_hidden_state[:, 0] @ kernel + bias
  (theirs * cot).sum().backward()

  scale = theirs.abs().max().item()
  assert (ours - theirs).abs().max().item() <= 1e-9 * scale
  hf_params = dict(hf.named_parameters())
  theirs_g = {"head/kernel": kernel.grad, "head/bias": bias.grad}
  for name in sd:
    ref = TB.name_map(name)
    theirs_g[ref] = TB._to_ours(ref, hf_params[name].grad, leaves[ref].shape)   # pylint: disable=protected-access
  assert set(theirs_g) == set(tree), sorted(set(tree) ^ set(theirs_g))
  for ref, g in theirs_g.items():
    scale_of = ref.replace("key/bias", "value/bias")
    tol = 1e-8 * theirs_g[scale_of].abs().max().item()
    assert (leaves[ref].grad - g).abs().max().item() <= tol, ref


# ---- the tower's configuration --------------------------------------------------------------------------
def test_rates_follow_the_original_bert():
  from big_vision_b200.models.proj.flaxformer import bert
  for cfg in ("base", "large"):
    m = bert.Model(cfg)
    assert m.dropout_rate == m.attention_dropout_rate == 0.1
  m = bert.Model(dict(TINY))
  assert m.dropout_rate == m.attention_dropout_rate == 0.0
  m = bert.Model(dict(TINY, attention_dropout_rate=0.2))
  assert (m.dropout_rate, m.attention_dropout_rate) == (0.0, 0.2)
  for kw in (dict(dropout_rate=1.0), dict(attention_dropout_rate=-0.1)):
    with pytest.raises(ValueError):
      bert.Model(dict(TINY, **kw))


def test_apply_train_names_the_missing_key():
  from big_vision_b200.models.proj.flaxformer import bert
  with pytest.raises(NotImplementedError, match=r"dropout.*fwd\(\.\.\., dropout=key\)"):
    bert.Model("base").apply({"params": None}, None, train=True)


def test_two_towers_apply_train_refuses_bert_with_dropout():
  from big_vision_b200.models.proj.image_text import two_towers
  tt = two_towers.Model(image=dict(width=64, depth=1, mlp_dim=128, num_heads=1), text_model="proj.flaxformer.bert",
                        text=dict(config=dict(TINY, attention_dropout_rate=0.1)))
  with pytest.raises(ValueError, match="dropout key"):
    tt.apply({"params": None}, None, None, train=True)


# ---- what the tower launches and keeps -------------------------------------------------------------------
def _generator():
  spec = importlib.util.spec_from_file_location("make_model_traces", os.path.join(ROOT, "tests", "golden",
                                                                                   "make_model_traces.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def _count(lines, name):
  return sum(1 for line in lines if line.split(" ", 1)[0] == name)


DEPTH, N_TXT = 3, 16


def _bert(rate, attn_rate):
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.flaxformer import bert
  model = bert.Model(dict(TINY, depth=DEPTH, dropout_rate=rate, attention_dropout_rate=attn_rate), num_classes=8)
  return model, E.FlatParams(*model.specs(N_TXT), "cpu")


def _record_keys(mp, keys):
  """Appends the dropout key of every attention-dropout call to `keys` (the trace shows the attention
  arguments only)."""
  from big_vision_b200 import lib as L
  for name in ("AttnDropoutArgs", "AttnDropoutBwdArgs"):
    real = getattr(L, name)
    mp.setattr(L, name, lambda masked, drop, real=real: keys.append(drop) or real(masked=masked, drop=drop))


def _step(gen, mp, model, P, frozen=None, dropout=None, keys=None):
  text = torch.from_numpy(BO.padded_text(2, N_TXT, TINY["vocab_size"], seed=1))
  out = {}
  if keys is not None:
    _record_keys(mp, keys)

  def fwd():
    y, saved = model.fwd(P, text, frozen=frozen, dropout=dropout)
    out["y"], out["saved"] = y, saved
    return gen.saved_bytes(saved, P, text)

  f, nbytes = gen._run(P, mp.setattr, fwd)   # pylint: disable=protected-access
  b, _ = gen._run(P, mp.setattr, lambda: model.bwd(P, torch.zeros((2, 8)), out["saved"]))   # pylint: disable=protected-access
  return f, b, nbytes


def _attn_flags(lines):
  return [int(line.rsplit(" ", 2)[1]) for line in lines if line.startswith("bv_attention")]


def test_rate_zero_and_no_key_launch_what_bert_launched_before():
  from big_vision_b200 import engine as E
  gen = _generator()
  key = E.DropoutKey(seed=5, step=7, sample0=4)
  with pytest.MonkeyPatch.context() as mp:
    f0, b0, n0 = _step(gen, mp, *_bert(0.0, 0.0), dropout=key)
    fe, be, ne = _step(gen, mp, *_bert(0.1, 0.1))          # no key: the evaluation path
  assert (fe, be, ne) == (f0, b0, n0)
  assert not any(line.startswith("bv_dropout") for line in f0 + b0)
  assert set(_attn_flags(f0 + b0)) == {64 | 65536}
  assert _count(f0, "bv_gemm") == 4 * DEPTH + 1 and sum("epilogue=3 " in line for line in f0) == 2 * DEPTH


@pytest.mark.parametrize("rate,attn_rate", [(0.1, 0.1), (0.1, 0.0), (0.0, 0.2)])
def test_dropout_adds_the_expected_calls_and_no_saved_bytes(rate, attn_rate):
  from big_vision_b200 import engine as E
  gen = _generator()
  key = E.DropoutKey(seed=5, step=7, sample0=4, tower=1)
  keys = []
  with pytest.MonkeyPatch.context() as mp:
    f0, b0, n0 = _step(gen, mp, *_bert(0.0, 0.0), dropout=key)
    f1, b1, n1 = _step(gen, mp, *_bert(rate, attn_rate), dropout=key, keys=keys)
  assert n1 == n0
  hid = 1 if rate else 0
  # forward: the embedding, then per layer the attention output and the MLP output (residual adds)
  assert _count(f1, "bv_dropout") == hid and _count(f1, "bv_dropout_add") == 2 * DEPTH * hid
  # backward: the embedding's and two masked gradients per layer, each bias summed from its masked gradient
  assert _count(b1, "bv_dropout") == (1 + 2 * DEPTH) * hid and _count(b1, "bv_dropout_add") == 0
  assert _count(b1, "bv_colsum") == _count(b0, "bv_colsum") + 2 * DEPTH * hid
  assert _count(f1, "bv_gemm") == _count(f0, "bv_gemm") and _count(b1, "bv_gemm") == _count(b0, "bv_gemm")
  # the attention calls carry the flag and the key in both directions
  flags = 64 | 65536 | (131072 if attn_rate else 0)
  assert _attn_flags(f1 + b1) == [flags] * (2 * DEPTH)
  # forward layers bottom-up, then the backward top-down, each with the layer's key: the forward's
  H, n = TINY["num_heads"], 4
  assert len(keys) == (2 * DEPTH if attn_rate else 0)
  for k, layer in zip(keys, list(range(DEPTH)) + list(reversed(range(DEPTH)))):
    assert (k.seed, k.step, k.site, k.row0) == (5, 7, E.dropout_site(1, layer, E.DROP_ATTN), n * H * N_TXT)
    assert k.rate == pytest.approx(attn_rate)
  # every hidden mask is drawn at this rank's rows, at the tower's sites
  lines = [line for line in f1 + b1 if line.startswith("bv_dropout")]
  assert all(f"row0={n * N_TXT} " in line and "seed=5 " in line for line in lines)
  sites = {int(s) for s in re.findall(r"site=(\d+)", " ".join(lines))}
  want = ({E.dropout_site(1, 0, E.DROP_EMBED)} | {E.dropout_site(1, i, k) for i in range(DEPTH)
                                                  for k in (E.DROP_ATTN, E.DROP_MLP)}) if rate else set()
  assert sites == want


def test_frozen_stages_drop_and_save_nothing():
  from big_vision_b200 import engine as E
  gen = _generator()
  model, P = _bert(0.1, 0.1)
  text = torch.from_numpy(BO.padded_text(2, N_TXT, TINY["vocab_size"], seed=1))
  with pytest.MonkeyPatch.context() as mp:
    lines, saved = gen._run(P, mp.setattr,   # pylint: disable=protected-access
                            lambda: model.fwd(P, text, frozen=True, dropout=E.DropoutKey(1, 2))[1])
  assert all(s is None for s in saved["stages"])
  assert _count(lines, "bv_dropout") == 1 and _count(lines, "bv_dropout_add") == 2 * DEPTH
  assert _attn_flags(lines) == [64 | 65536 | 131072] * DEPTH


def test_two_towers_pass_the_key_to_bert_as_tower_1():
  import common
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.image_text import two_towers
  gen = _generator()
  model = two_towers.Model(image=common.TINY["image"], text_model="proj.flaxformer.bert",
                           text=dict(config=dict(TINY, depth=1, attention_dropout_rate=0.1)), out_dim=(None, 64))
  P = E.FlatParams(*model.specs(common.TINY_IMAGE_SHAPE, (2, N_TXT)), "cpu")
  text = torch.from_numpy(BO.padded_text(2, N_TXT, TINY["vocab_size"], seed=1))
  keys = []
  with pytest.MonkeyPatch.context() as mp:
    _record_keys(mp, keys)
    lines, _ = gen._run(P, mp.setattr,   # pylint: disable=protected-access
                        lambda: model.fwd(P, None, text, dropout=E.DropoutKey(1, 2)))
  assert _attn_flags(lines) == [64 | 65536 | 131072]
  assert [k.site for k in keys] == [E.dropout_site(1, 0, E.DROP_ATTN)]
