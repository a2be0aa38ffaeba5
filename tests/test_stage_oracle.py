"""CPU: the per-stage float64 references of tests/stage_oracle.py, chained bottom-up, are the whole-model
oracle (O.vit_forward, O.mixer_forward, O.text_forward, the FlexiViT forward, the BERT tower with and without
dropout, and the BiT ResNet-v2), outputs and autograd gradients to 1e-12; and every backward stage class of the
models is named with the replay cases of tests/test_stage_replay_gpu.py that check it."""
import importlib
import pkgutil

import numpy as np
import pytest
import torch

import flexi_oracle as FO
import stage_oracle as S
from oracle import bv_oracle as O

F64 = torch.float64
sub = O.sub


def _tree(specs_aliases, seed):
  """A random float64 leaf per reference name of the model's parameters (every tensor nonzero)."""
  from big_vision_b200 import engine as E
  P = E.FlatParams(*specs_aliases, "cpu").init(seed)
  rng = np.random.default_rng(seed)
  tree = {k: (v if np.any(v) else rng.standard_normal(v.shape) * 0.05) for k, v in P.numpy_tree("f").items()}
  return O.to_f64_tree(tree, requires_grad=True)


def _assert_same(chain, ref, p, inputs, scale_of=None):
  """The two forwards agree, and so do their gradients w.r.t. every parameter (and input) for one cotangent.
  `scale_of` {name: other name}: a gradient that is zero in exact arithmetic, held to the other's scale."""
  assert chain.shape == ref.shape
  assert float((chain - ref).abs().max()) <= 1e-12 * float(ref.detach().abs().max())
  leaves = list(p.values()) + list(inputs)
  dy = torch.randn(ref.shape, dtype=F64, generator=torch.Generator().manual_seed(0))
  g1 = torch.autograd.grad(chain, leaves, dy, allow_unused=True)
  g2 = torch.autograd.grad(ref, leaves, dy, allow_unused=True)
  grads = dict(zip(list(p) + ["input"] * len(inputs), g2))
  for name, a, b in zip(list(p) + ["input"] * len(inputs), g1, g2):
    assert (a is None) == (b is None), name
    if a is not None:
      scale = grads[(scale_of or {}).get(name, name)]
      assert float((a - b).abs().max()) <= 1e-12 * max(float(scale.abs().max()), 1e-300), name


# (O.vit_forward pool_type -> the NormPool pool)
_VIT_POOL = {"gap": "mean", "0": "first", "tok": "first", "map": None, "none": None}


def _vit_chain(p, image, cfg, heads, depth):
  d = p["embedding/bias"].shape[0]
  ph, pw = p["embedding/kernel"].shape[:2]
  if cfg["posemb"] == "learn":
    pos = p["pos_embedding"]
  else:
    pos = torch.from_numpy(O.posemb_sincos_2d(image.shape[1] // ph, image.shape[2] // pw, d)).to(F64)
  x = S.patch_embedding(image, p, "embedding", pos, cfg["pool_type"] == "tok")
  for i in range(depth):
    x = S.encoder_block(x, sub(p, f"Transformer/encoderblock_{i}/"), heads)
  x = S.norm_pool(x, sub(p, "Transformer/encoder_norm/"), _VIT_POOL[cfg["pool_type"]])
  if cfg["pool_type"] == "map":
    x = S.map_head(x, sub(p, "MAPHead_0/"), heads)
  if cfg.get("rep_size"):
    x = S.dense(x, sub(p, "pre_logits/"), tanh=True)
  return S.dense(x, sub(p, "head/"))


@pytest.mark.parametrize("pool,posemb,rep", [("tok", "learn", 16), ("gap", "sincos2d", False), ("map", "learn", False),
                                             ("0", "learn", 16), ("none", "sincos2d", False)])
def test_vit_chain_is_the_vit_oracle(pool, posemb, rep):
  from big_vision_b200.models import vit
  model = vit.Model(5, width=64, depth=2, mlp_dim=96, num_heads=1, patch_size=(8, 8), pool_type=pool, posemb=posemb,
                    rep_size=rep)
  p = _tree(model.specs((24, 16), 3), 1)
  image = torch.empty(2, 24, 16, 3, dtype=F64).uniform_(-1, 1, generator=torch.Generator().manual_seed(2))
  cfg = dict(depth=2, num_heads=1, pool_type=pool, posemb=posemb, rep_size=rep, num_classes=5)
  _assert_same(_vit_chain(p, image, cfg, 1, 2), O.vit_forward(p, image, cfg), p, [])


@pytest.mark.parametrize("masked", [False, True])
def test_mixer_chain_is_the_mixer_oracle(masked):
  from big_vision_b200.models import mlp_mixer
  model = mlp_mixer.Model(5, patch_size=(8, 8), num_blocks=3, hidden_dim=32, tokens_mlp_dim=16, channels_mlp_dim=48)
  p = _tree(model.specs((24, 24), 3), 3)
  image = torch.empty(3, 24, 24, 3, dtype=F64).uniform_(-1, 1, generator=torch.Generator().manual_seed(4))
  masks = None
  if masked:
    masks = torch.ones(3, 2, 3, dtype=F64)
    masks[0, 1, 2] = masks[1, 0, 0] = masks[2, 0, :] = 0
  x = S.patch_embedding(image, p, "stem")
  for i in range(3):
    x = S.mixer_block(x, sub(p, f"MixerBlock_{i}/"), None if masks is None else masks[i])
  x = S.dense(S.norm_pool(x, sub(p, "pre_head_layer_norm/"), "mean"), sub(p, "head/"))
  _assert_same(x, O.mixer_forward(p, image, dict(num_blocks=3, num_classes=5), masks=masks), p, [])


@pytest.mark.parametrize("pool,head", [("last", True), ("first", True), ("max", True), ("mean", False),
                                       ("map", True), ("map", False), ("max", False)])
def test_text_chain_is_the_text_oracle(pool, head):
  from big_vision_b200.models.proj.image_text import text_transformer
  C = 16 if head else None
  model = text_transformer.Model(C, width=64, depth=2, mlp_dim=96, num_heads=1, vocab_size=20, pool_type=pool)
  p = _tree(model.specs(7), 5)
  ids = torch.from_numpy(np.random.default_rng(6).integers(0, 20, size=(3, 7)).astype(np.int32))
  x = S.text_embed(ids, p)
  for i in range(2):
    x = S.encoder_block(x, sub(p, f"Encoder_0/encoderblock_{i}/"), 1)
  x = S.norm_pool(x, sub(p, "Encoder_0/encoder_norm/"), None if pool == "map" else pool)
  if pool == "map":
    x = S.map_head(x, sub(p, "MAPHead_0/"), 1)
  if head:
    x = S.dense(x, sub(p, "head/"))
  cfg = dict(depth=2, num_heads=1, pool_type=pool, num_classes=C)
  _assert_same(x, O.text_forward(p, ids, cfg), p, [])


BERT_TINY = dict(width=128, depth=2, num_heads=2, mlp_dim=96, vocab_size=20)


@pytest.mark.parametrize("head,dropout", [(True, False), (False, False), (True, True), (False, True)])
def test_bert_chain_is_the_bert_oracle(head, dropout):
  """Without masks the chain is bert_oracle.bert_forward; under given dropout masks (the embedding, each
  layer's probabilities, attention output and MLP output) it is bert_dropout_oracle.bert_forward."""
  import bert_dropout_oracle as BDO
  import bert_oracle as BO
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.flaxformer import bert
  C, n, N, d, H = (5 if head else None), 3, 7, 128, 2
  model = bert.Model(BERT_TINY, num_classes=C)
  p = _tree(model.specs(N), 5)
  ids = torch.from_numpy(BO.padded_text(n, N, 20, seed=6))
  assert (ids == 0).any()
  key_mask = ids != 0
  masks = None
  if dropout:
    rng = np.random.default_rng(7)
    keep = lambda *shape: torch.from_numpy(rng.random(shape) >= 0.1).to(F64) / 0.9
    masks = BDO.GivenMasks({(i, k): keep(n, N, d) for i in range(2) for k in (E.DROP_EMBED, E.DROP_ATTN, E.DROP_MLP)},
                           [keep(n, H, N, N) for _ in range(2)])
  x = S.bert_embed(ids, sub(p, "BertEncoder_0/embedder/"), masks and masks.h[(0, E.DROP_EMBED)])
  for i in range(2):
    m = masks and (masks.p[i], masks.h[(i, E.DROP_ATTN)], masks.h[(i, E.DROP_MLP)])
    x = S.bert_layer(x, sub(p, f"BertEncoder_0/encoder_layer_{i}/"), H, key_mask, m)
  x = S.cls_pool(x)
  if head:
    x = S.dense(x, sub(p, "head/"))
  cfg = dict(depth=2, num_heads=H, num_classes=C)
  ref = BO.bert_forward(p, ids.long(), cfg) if masks is None else BDO.bert_forward(p, ids.long(), cfg, masks)
  # the key bias (softmax is invariant to a per-query shift) at the value bias's scale: the two softmax forms
  # round differently
  _assert_same(x, ref, p, [], {k: k.replace("key/bias", "value/bias") for k in p if k.endswith("key/bias")})


@pytest.mark.parametrize("head", [True, False])
def test_bit_chain_is_the_bit_oracle(head):
  """Depth [2, 1, 1, 1]: a projection unit and an identity unit in block 1, stride 2 on odd sizes after."""
  import bit_oracle as BO
  from big_vision_b200.models import bit_paper
  depth = [2, 1, 1, 1]
  model = bit_paper.Model(5 if head else None, width=0.5, depth=depth)
  p = _tree(model.specs((26, 22), 3), 15)
  image = torch.empty(2, 26, 22, 3, dtype=F64).uniform_(-1, 1, generator=torch.Generator().manual_seed(16))
  x = S.bit_root(image, sub(p, "root_block/"))
  for b, size in enumerate(depth):
    for u in range(size):
      x = S.bit_unit(x, sub(p, f"block{b + 1}/unit{u + 1:02d}/"), 2 if (b > 0 and u == 0) else 1)
  x = S.bit_prehead(x, sub(p, "norm-pre-head/"))
  if head:
    x = S.dense(x, sub(p, "head/"))
  _assert_same(x, BO.forward(p, image, depth), p, [])


def test_bit_root_routes_to_the_first_maximum_of_route():
  """With a `route` whose windows tie, each window takes its first maximum in row-major order."""
  import bit_oracle as BO
  y = torch.randn(1, 5, 5, 2, dtype=F64, generator=torch.Generator().manual_seed(17))
  route = torch.zeros_like(y)          # every window ties: the first in-image element of each window wins
  kernel = torch.randn(7, 7, 3, 2, dtype=F64, generator=torch.Generator().manual_seed(18))
  image = torch.randn(1, 10, 10, 3, dtype=F64, generator=torch.Generator().manual_seed(19))
  out = S.bit_root(image, {"conv_root/kernel": kernel}, route=route)
  conv = BO.std_conv(image, kernel, 2, 3)
  assert out.shape == (1, 3, 3, 2)
  # window (i, j) covers rows 2i - 1 .. 2i + 1: its first in-image element is (max(2i - 1, 0), max(2j - 1, 0))
  first = [0, 1, 3]
  assert torch.equal(out, conv[:, first][:, :, first])


def test_max_pool_splits_ties_like_amax():
  """Tied maxima share the cotangent evenly, as torch.amax (and jnp.max) do."""
  x = torch.randn(2, 5, 8, dtype=F64)
  x[:, 3] = x[:, 1]
  x.requires_grad_(True)
  p = {"scale": torch.ones(8, dtype=F64), "bias": torch.zeros(8, dtype=F64)}
  dy = torch.randn(2, 8, dtype=F64)
  ga, = torch.autograd.grad(S.norm_pool(x, p, "max"), x, dy)
  gb, = torch.autograd.grad(torch.amax(O.layer_norm(x, p["scale"], p["bias"]), 1), x, dy)
  assert float((ga - gb).abs().max()) <= 1e-12


@pytest.mark.parametrize("pool,posemb,seqhw", [("tok", "learn", 3), ("gap", "sincos2d", 4), ("map", "learn", 2)])
def test_flexi_chain_is_the_flexi_oracle(pool, posemb, seqhw):
  from big_vision_b200.models.proj.flexi import vit as fv
  model = fv.Model(5, width=64, depth=1, mlp_dim=96, num_heads=1, patch_size=(4, 4), posemb_size=(3, 3),
                   pool_type=pool, posemb=posemb)
  p = _tree(model.specs(), 7)
  image = torch.empty(2, 12, 12, 3, dtype=F64).uniform_(-1, 1, generator=torch.Generator().manual_seed(8))
  pos = p["pos_embedding"] if posemb == "learn" else torch.from_numpy(O.posemb_sincos_2d(3, 3, 64)).to(F64)
  x = S.flexi_patch_embedding(image, p, seqhw, (3, 3), pos, pool == "tok")
  x = S.encoder_block(x, sub(p, "Transformer/encoderblock_0/"), 1)
  x = S.norm_pool(x, sub(p, "Transformer/encoder_norm/"), {"tok": "first", "gap": "mean", "map": None}[pool])
  if pool == "map":
    x = S.map_head(x, sub(p, "MAPHead_0/"), 1)
  x = S.dense(x, sub(p, "head/"))
  cfg = dict(depth=1, num_heads=1, pool_type=pool, posemb=posemb, posemb_size=(3, 3), num_classes=5)
  _assert_same(x, FO.flexi_forward(p, image, cfg, seqhw), p, [])


def test_key_grad_tap_is_the_key_gradient():
  """S.Tap on the key bias receives d key: its column sum is the key-bias gradient, and the forward is unchanged."""
  from big_vision_b200.models import vit
  model = vit.Model(None, width=64, depth=1, mlp_dim=96, num_heads=1, patch_size=(8, 8), pool_type="gap")
  p = _tree(model.specs((16, 16), 3), 9)
  q = sub(p, "Transformer/encoderblock_0/")
  x = torch.randn(2, 6, 64, dtype=F64, generator=torch.Generator().manual_seed(10))
  kb = q["MultiHeadDotProductAttention_0/key/bias"]
  tap = S.Tap(kb, (2, 6, 64))
  with tap:
    y = S.encoder_block(x, q, 1)
  y0 = S.encoder_block(x, q, 1)
  assert float((y - y0).abs().max()) == 0.0
  dy = torch.randn(y.shape, dtype=F64)
  dkey, dbias = torch.autograd.grad(y, [tap.tap, kb], dy)
  assert float((dkey.sum((0, 1)).view(dbias.shape) - dbias).abs().max()) <= 1e-12
  assert float(dkey.abs().sum()) > 1e3 * float(dbias.abs().max())    # zero in exact arithmetic


def test_score_grad_records_the_attention_scores():
  """S.ScoreGrad records the q, k of the score product and dS: dS rows sum to zero (softmax), dS k / sqrt(dh)
  is d query, and the floors have the queries' and keys' shapes."""
  from big_vision_b200.models import vit
  model = vit.Model(None, width=64, depth=1, mlp_dim=96, num_heads=1, patch_size=(8, 8), pool_type="gap")
  p = _tree(model.specs((16, 16), 3), 13)
  q = sub(p, "Transformer/encoderblock_0/")
  x = torch.randn(2, 6, 64, dtype=F64, generator=torch.Generator().manual_seed(14))
  qb = q["MultiHeadDotProductAttention_0/query/bias"]
  tap, rec = S.Tap(qb, (2, 6, 64)), S.ScoreGrad()
  with tap, rec:
    y = S.encoder_block(x, q, 1)
  y.backward(torch.randn(y.shape, dtype=F64, generator=torch.Generator().manual_seed(15)))
  assert float(rec.s.grad.sum(-1).abs().max()) <= 1e-12 * float(rec.s.grad.abs().max())
  dq = (rec.s.grad @ rec.k / 8.0).transpose(1, 2).reshape(2, 6, 64)
  assert float((dq - tap.tap.grad).abs().max()) <= 1e-12 * float(dq.abs().max())
  fq, fk = rec.floors()
  assert fq.shape == fk.shape == (2, 6, 64) and bool((fq > 0).all())


def test_mixer_token_mixing_output_bias_tap():
  """The token-mixing Dense_1 bias shifts each token's channels by one constant, which the next LayerNorm
  removes: its gradient is zero in exact arithmetic, and S.Tap's column sum is that gradient."""
  from big_vision_b200.models import mlp_mixer
  model = mlp_mixer.Model(5, patch_size=(8, 8), num_blocks=1, hidden_dim=32, tokens_mlp_dim=16, channels_mlp_dim=48)
  p = _tree(model.specs((24, 24), 3), 11)
  q = sub(p, "MixerBlock_0/")
  b = q["token_mixing/Dense_1/bias"]
  x = torch.randn(2, 9, 32, dtype=F64, generator=torch.Generator().manual_seed(12))
  tap = S.Tap(b, (2, 32, 9))
  with tap:
    y = S.mixer_block(x, q)
  y = O.layer_norm(y, torch.ones(32, dtype=F64), torch.zeros(32, dtype=F64))
  dtok, db = torch.autograd.grad(y, [tap.tap, b], torch.randn(y.shape, dtype=F64))
  assert float((dtok.sum((0, 1)) - db).abs().max()) <= 1e-12
  assert float(dtok.abs().sum()) > 1e3 * float(db.abs().max())


# ---- every backward stage class has replay cases ---------------------------------------------------------------
# stage class (module.qualname) -> the cases of test_stage_replay_gpu.CASES whose model holds one
COVERAGE = {
    "big_vision_b200.models.vit.PatchEmbedding": ["vit_tok", "vit_gap_sincos", "vit_map", "vit_0", "vit_none",
                                                  "vit_b16_tok", "mixer", "mixer_stoch"],
    "big_vision_b200.models.vit.EncoderBlock": ["vit_tok", "vit_map", "vit_hd72", "vit_b16_tok", "vit_b16_map",
                                                "text_last", "vit_frozen_cut", "text_frozen_cut"],
    "big_vision_b200.models.vit.ScanEncoder": ["vit_tok_scan", "vit_map_scan"],
    "big_vision_b200.models.vit.NormPool": ["vit_tok", "vit_gap_sincos", "vit_0", "vit_none", "text_last",
                                            "text_first", "text_max", "text_mean", "mixer"],
    "big_vision_b200.models.vit.MAPHead": ["vit_map", "vit_map_scan", "vit_hd72", "vit_b16_map", "text_map",
                                           "text_map_nohead"],
    "big_vision_b200.models.common.Dense": ["vit_tok", "vit_none", "vit_b16_tok", "mixer", "text_last"],
    "big_vision_b200.models.mlp_mixer.MixerBlock": ["mixer", "mixer_stoch"],
    "big_vision_b200.models.proj.image_text.text_transformer._Embed": ["text_last", "text_max", "text_frozen_cut"],
    "big_vision_b200.models.proj.flexi.vit.FlexiPatchEmbedding": ["flexi_resample", "flexi_base_sincos"],
    "big_vision_b200.models.proj.flaxformer.bert._Embed": ["bert", "bert_dropout", "bert_nohead"],
    "big_vision_b200.models.proj.flaxformer.bert._Layer": ["bert", "bert_dropout", "bert_nohead", "bert_frozen_cut"],
    "big_vision_b200.models.proj.flaxformer.bert._ClsPool": ["bert", "bert_dropout", "bert_nohead", "bert_frozen_cut"],
    "big_vision_b200.models.bit_paper.RootBlock": ["bit", "bit_nohead"],
    "big_vision_b200.models.bit_paper.ResidualUnit": ["bit", "bit_nohead", "bit_frozen_cut"],
    "big_vision_b200.models.bit_paper.PreHead": ["bit", "bit_nohead", "bit_frozen_cut"],
}


def _stage_classes():
  """Every engine.Stage subclass defined under big_vision_b200/models/ (after importing every module there)."""
  import big_vision_b200.models as models
  from big_vision_b200 import engine as E
  for m in pkgutil.walk_packages(models.__path__, models.__name__ + "."):
    importlib.import_module(m.name)
  out, todo = set(), [E.Stage]
  while todo:
    for c in todo.pop().__subclasses__():
      todo.append(c)
      if c.__module__.startswith("big_vision_b200.models."):
        out.add(f"{c.__module__}.{c.__qualname__}")
  return out


def test_every_stage_class_is_named_with_replay_cases():
  found = _stage_classes()
  assert len(found) >= 15
  missing, extra = found - set(COVERAGE), set(COVERAGE) - found
  assert not missing, f"backward stages without a per-stage replay case: {sorted(missing)}"
  assert not extra, f"COVERAGE rows for classes that are not stages under models/: {sorted(extra)}"


def test_every_named_case_holds_its_stage():
  """Each case named in COVERAGE exists and its model (built on the host) contains that stage class."""
  import test_stage_replay_gpu as R
  from big_vision_b200.models import vit
  for cls, cases in COVERAGE.items():
    assert cases, cls
    for case in cases:
      assert case in R.CASES, f"{cls}: no replay case {case}"
      stages = R.build_model(case)._stages     # pylint: disable=protected-access
      stages = stages + [b for s in stages if isinstance(s, vit.ScanEncoder) for b in s.blocks]
      names = {f"{type(s).__module__}.{type(s).__qualname__}" for s in stages}
      assert cls in names, f"{case} has no {cls}"
