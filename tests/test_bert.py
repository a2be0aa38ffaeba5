"""CPU: the BERT text tower's oracle pinned against `transformers.BertModel`, and the tower's parameters.

`tests/bert_oracle.py` restates post-LN BERT in float64 with an explicit key mask.  `transformers`' BertModel
(built from a BertConfig with random weights; nothing is downloaded) is an implementation of the original
BERT that shares no code with it.  One random parameter tree mapped into both gives the same [CLS] output
and the same gradient for every parameter, with padding present.  The oracle's key-only mask gives the
[CLS] output and gradients of a mask that also covers the padded queries (flaxformer's).  Test
infrastructure only."""
import numpy as np
import pytest
import torch

import bert_oracle as BO

transformers = pytest.importorskip("transformers")

TINY = dict(width=128, depth=2, num_heads=2, mlp_dim=256, vocab_size=97)
N_TOK, BATCH, CLASSES = 16, 6, 24


def _model(cfg=TINY, num_classes=CLASSES, head_zeroinit=False):
  from big_vision_b200.models.proj.flaxformer import bert
  return bert.Model(cfg, num_classes=num_classes, head_zeroinit=head_zeroinit)


def random_tree(model, text_len, seed):
  """The model's initial tree with every leaf perturbed (zero biases and unit scales would hide a wrong
  mapping) -> {name: np.float32 array}."""
  from big_vision_b200 import engine as E
  specs, aliases = model.specs(text_len)
  P = E.FlatParams(specs, aliases, "cpu").init(seed)
  rng = np.random.default_rng(seed + 1)
  return {k: (v + 0.05 * rng.standard_normal(v.shape)).astype(np.float32) for k, v in P.numpy_tree("f").items()}


def _hf_model(tree, cfg, vocab):
  from transformers import BertConfig, BertModel
  d, depth = cfg["width"], cfg["depth"]
  conf = BertConfig(vocab_size=vocab, hidden_size=d, num_hidden_layers=depth, num_attention_heads=cfg["num_heads"],
                    intermediate_size=cfg["mlp_dim"], hidden_act="gelu_new", layer_norm_eps=1e-12,
                    max_position_embeddings=512, type_vocab_size=2, hidden_dropout_prob=0.0,
                    attention_probs_dropout_prob=0.0, attn_implementation="eager")
  model = BertModel(conf, add_pooling_layer=False).double().eval()
  t = {k: torch.from_numpy(np.asarray(v, dtype=np.float64)) for k, v in tree.items()}
  e = "BertEncoder_0/embedder/"
  sd = {"embeddings.word_embeddings.weight": t[e + "embedders_token_ids/embedding"],
        "embeddings.position_embeddings.weight": t[e + "embedders_position_ids/embedding"],
        "embeddings.token_type_embeddings.weight": t[e + "embedders_segment_ids/embedding"],
        "embeddings.LayerNorm.weight": t[e + "layer_norm/scale"],
        "embeddings.LayerNorm.bias": t[e + "layer_norm/bias"]}
  for i in range(depth):
    p, h = f"BertEncoder_0/encoder_layer_{i}/", f"encoder.layer.{i}."
    for ours, theirs in (("query", "attention.self.query"), ("key", "attention.self.key"),
                         ("value", "attention.self.value")):
      sd[h + theirs + ".weight"] = t[p + f"self_attention/{ours}/kernel"].reshape(d, d).T
      sd[h + theirs + ".bias"] = t[p + f"self_attention/{ours}/bias"].reshape(d)
    sd[h + "attention.output.dense.weight"] = t[p + "self_attention/out/kernel"].reshape(d, d).T
    sd[h + "attention.output.dense.bias"] = t[p + "self_attention/out/bias"]
    sd[h + "attention.output.LayerNorm.weight"] = t[p + "attention_layer_norm/scale"]
    sd[h + "attention.output.LayerNorm.bias"] = t[p + "attention_layer_norm/bias"]
    sd[h + "intermediate.dense.weight"] = t[p + "mlp/Dense_0/kernel"].T
    sd[h + "intermediate.dense.bias"] = t[p + "mlp/Dense_0/bias"]
    sd[h + "output.dense.weight"] = t[p + "mlp/Dense_1/kernel"].T
    sd[h + "output.dense.bias"] = t[p + "mlp/Dense_1/bias"]
    sd[h + "output.LayerNorm.weight"] = t[p + "output_layer_norm/scale"]
    sd[h + "output.LayerNorm.bias"] = t[p + "output_layer_norm/bias"]
  missing, unexpected = model.load_state_dict(sd, strict=False)
  assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
  return model, sd


def _leaves(tree):
  return {k: torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True) for k, v in tree.items()}


@pytest.fixture(scope="module")
def pinned():
  model = _model()
  tree = random_tree(model, N_TOK, seed=3)
  text = torch.from_numpy(BO.padded_text(BATCH, N_TOK, TINY["vocab_size"], seed=4)).long()
  assert (text == 0).any() and (text[:, 0] != 0).all()
  cot = torch.from_numpy(np.random.default_rng(5).standard_normal((BATCH, CLASSES)))
  cfg = dict(depth=TINY["depth"], num_heads=TINY["num_heads"], num_classes=CLASSES)
  return tree, text, cot, cfg


def test_oracle_matches_transformers_bert(pinned):
  """[CLS] output within 1e-9 and every parameter gradient within 1e-8 (relative to the tensor's max),
  float64, with padded captions."""
  tree, text, cot, cfg = pinned
  leaves = _leaves(tree)
  ours = BO.bert_forward(leaves, text, cfg)
  (ours * cot).sum().backward()

  hf, sd = _hf_model(tree, TINY, TINY["vocab_size"])
  hf_params = dict(hf.named_parameters())
  kernel, bias = (torch.tensor(np.asarray(tree[k], dtype=np.float64), requires_grad=True)
                  for k in ("head/kernel", "head/bias"))
  out = hf(input_ids=text, attention_mask=(text != 0).long(), token_type_ids=torch.zeros_like(text))
  theirs = out.last_hidden_state[:, 0] @ kernel + bias
  (theirs * cot).sum().backward()

  scale = theirs.abs().max().item()
  assert (ours - theirs).abs().max().item() <= 1e-9 * scale
  theirs_g = {"head/kernel": kernel.grad, "head/bias": bias.grad}
  for name in sd:
    ref = name_map(name)
    theirs_g[ref] = _to_ours(ref, hf_params[name].grad, leaves[ref].shape)
  assert set(theirs_g) == set(tree), sorted(set(tree) ^ set(theirs_g))
  for ref, g in theirs_g.items():
    # the key bias shifts every score of a query equally: its gradient is 0 up to rounding, on both sides,
    # and is held to the value bias's gradient scale
    scale_of = ref.replace("key/bias", "value/bias")
    tol = 1e-8 * theirs_g[scale_of].abs().max().item()
    assert (leaves[ref].grad - g).abs().max().item() <= tol, ref


def name_map(hf_name):
  """Our tree name of a transformers parameter."""
  e = "BertEncoder_0/embedder/"
  fixed = {"embeddings.word_embeddings.weight": e + "embedders_token_ids/embedding",
           "embeddings.position_embeddings.weight": e + "embedders_position_ids/embedding",
           "embeddings.token_type_embeddings.weight": e + "embedders_segment_ids/embedding",
           "embeddings.LayerNorm.weight": e + "layer_norm/scale", "embeddings.LayerNorm.bias": e + "layer_norm/bias"}
  if hf_name in fixed:
    return fixed[hf_name]
  _, _, i, rest = hf_name.split(".", 3)
  p = f"BertEncoder_0/encoder_layer_{i}/"
  table = {"attention.self.query": "self_attention/query", "attention.self.key": "self_attention/key",
           "attention.self.value": "self_attention/value", "attention.output.dense": "self_attention/out",
           "intermediate.dense": "mlp/Dense_0", "output.dense": "mlp/Dense_1"}
  module, kind = rest.rsplit(".", 1)
  if module in table:
    return p + table[module] + ("/kernel" if kind == "weight" else "/bias")
  ln = {"attention.output.LayerNorm": "attention_layer_norm", "output.LayerNorm": "output_layer_norm"}[module]
  return p + ln + ("/scale" if kind == "weight" else "/bias")


def _to_ours(name, g, shape):
  """A transformers gradient in our layout: Linear weights [out, in] -> kernels [in, out], reshaped."""
  if name.endswith("/kernel"):
    return g.T.reshape(shape)
  return g.reshape(shape)


def test_key_mask_alone_equals_masking_the_padded_queries_too(pinned):
  """Masking only the keys (this port) gives flaxformer's [CLS] output and parameter gradients, which
  also mask the padded queries: their rows never reach [CLS]."""
  tree, text, cot, cfg = pinned
  grads, outs = [], []
  for mask_queries in (False, True):
    leaves = _leaves(tree)
    y = BO.bert_forward(leaves, text, cfg, mask_queries=mask_queries)
    (y * cot).sum().backward()
    outs.append(y.detach())
    grads.append({k: v.grad for k, v in leaves.items()})
  assert (outs[0] - outs[1]).abs().max().item() <= 1e-12 * outs[1].abs().max().item()
  for k in tree:
    scale = max(grads[1][k].abs().max().item(), 1e-30)
    assert (grads[0][k] - grads[1][k]).abs().max().item() <= 1e-11 * scale, k


def test_parameter_names_and_shapes():
  from big_vision_b200.models.proj.flaxformer import bert
  model = bert.Model("base", num_classes=768)
  specs, aliases = model.specs(16)
  from big_vision_b200 import engine as E
  shapes = {s.name: s.shape for s in specs}
  shapes.update({a.name: None for a in aliases})
  assert shapes["BertEncoder_0/embedder/embedders_position_ids/embedding"] == (512, 768)
  assert shapes["BertEncoder_0/embedder/embedders_token_ids/embedding"] == (30_522, 768)
  assert shapes["BertEncoder_0/embedder/embedders_segment_ids/embedding"] == (2, 768)
  assert shapes["head/kernel"] == (768, 768)
  layers = {k.split("/")[1] for k in shapes if k.startswith("BertEncoder_0/encoder_layer_")}
  assert layers == {f"encoder_layer_{i}" for i in range(12)}
  large = bert.Model("large")
  assert len(large.specs(16)[0]) == len(specs) - 2 + 24 * 12 - 12 * 12 and large.width == 1024
  P = E.FlatParams(*bert.Model(TINY, num_classes=8).specs(16), "cpu").init(0)
  assert not P.f("head/kernel").any()                      # head_zeroinit
  assert {"query/kernel", "out/kernel"} <= {k.split("self_attention/")[1] for k in P.tree() if "self_attention/" in k}


def test_head_dims_without_the_masked_kernel_are_refused():
  from big_vision_b200.models.proj.flaxformer import bert
  with pytest.raises(NotImplementedError, match="head dim 64"):
    bert.Model(dict(width=144, depth=1, num_heads=2, mlp_dim=256))


def test_load_reads_npz_and_refuses_the_tf_checkpoint(tmp_path):
  from big_vision_b200 import utils
  from big_vision_b200.models.proj.flaxformer import bert
  model = _model()
  tree = random_tree(model, N_TOK, seed=7)
  init = utils.recover_tree(*zip(*random_tree(model, N_TOK, seed=8).items()))
  path = str(tmp_path / "bert.npz")
  np.savez(path, **tree)
  loaded = dict(utils.tree_flatten_with_names(bert.load(init, path, None))[0])
  assert set(loaded) == set(tree) and all(np.array_equal(loaded[k], tree[k]) for k in tree)
  kept = dict(utils.tree_flatten_with_names(bert.load(init, path, None, dont_load=("head/.*",)))[0])
  assert np.array_equal(kept["head/kernel"], dict(utils.tree_flatten_with_names(init)[0])["head/kernel"])
  (tmp_path / "ckpt").mkdir()
  (tmp_path / "ckpt" / "bert_model.ckpt.index").write_bytes(b"")
  with pytest.raises(NotImplementedError, match="tensorflow"):
    bert.load(init, str(tmp_path / "ckpt"), None)


def test_two_towers_builds_with_the_bert_text_tower():
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.image_text import two_towers
  model = two_towers.Model(text_model="proj.flaxformer.bert", text=dict(config="base"),
                           image=dict(variant="B/16", pool_type="tok", head_zeroinit=False),
                           out_dim=(None, 768), bias_init=-2.71)
  specs, aliases = model.specs((4, 224, 224, 3), (4, 16))
  names = {s.name for s in specs}
  assert "txt/BertEncoder_0/embedder/embedders_position_ids/embedding" in names
  assert "txt/head/kernel" in names and "b" in names
  assert model.txt.stages()[0] == ("txt/BertEncoder_0/embedder/",)
  assert E.stage_cut(names, model.txt.stages(), {n for n in names if n.startswith("img/")}) == 0
