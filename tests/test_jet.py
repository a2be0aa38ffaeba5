"""CPU: Jet's host side -- the parameter tree of configs/proj/jet/imagenet64.py, the coupling order, the mask
initialisers, the gather tables against the float64 oracle's einsum split and merge, the noise generator
against numpy, properties of the oracle itself (invertibility, the log-determinant against an autograd
Jacobian, bits per dimension against scipy) and the refusals."""
import os

import numpy as np
import pytest
import torch

import jet_oracle as JO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IMAGENET64 = dict(depth=32, block_depth=2, emb_dim=512, num_heads=8,
                  kinds=("channels", "channels", "channels", "channels", "spatial"),
                  channels_coupling_projs=("random",),
                  spatial_coupling_projs=("checkerboard", "checkerboard-inv", "vstripes", "vstripes-inv",
                                          "hstripes", "hstripes-inv"))
TINY = dict(depth=3, block_depth=1, emb_dim=64, num_heads=1, kinds=("channels", "spatial"),
            spatial_coupling_projs=("checkerboard", "vstripes-inv"))


def _jet():
  from big_vision_b200.models.proj.jet import jet
  return jet


def _meta_tree(model, image_hw=(64, 64)):
  from big_vision_b200 import engine as E
  return E.FlatParams(*model.specs(image_hw, 3), "meta").tree("f")


# ---- parameter tree, coupling order, mask inits --------------------------------------------------------
def test_imagenet64_parameter_tree_has_the_reference_names_and_shapes():
  jet = _jet()
  tree = _meta_tree(jet.Model(**IMAGENET64))
  shapes = {k: tuple(v.shape) for k, v in tree.items()}
  assert shapes["channel_coupling_masks-FREEZE_ME"] == (32, 48, 48)
  assert shapes["spatial_coupling_masks-FREEZE_ME"] == (32, 256, 256)
  dnn = "couplings/dnn/"
  assert shapes[dnn + "init_proj/kernel"] == (32, 24, 512) and shapes[dnn + "init_proj/bias"] == (32, 512)
  assert shapes[dnn + "posemb"] == (32, 1, 256, 512)
  assert shapes[dnn + "final_proj/kernel"] == (32, 512, 48) and shapes[dnn + "final_proj/bias"] == (32, 48)
  assert shapes[dnn + "vit/encoder_norm/scale"] == (32, 512)
  att = dnn + "vit/encoderblock_1/MultiHeadDotProductAttention_0/"
  assert shapes[att + "query/kernel"] == (32, 512, 8, 64) and shapes[att + "out/kernel"] == (32, 8, 64, 512)
  assert shapes[dnn + "vit/encoderblock_0/MlpBlock_0/Dense_0/kernel"] == (32, 512, 2048)
  assert {k.split("/")[3] for k in tree if k.startswith(dnn + "vit/")} == {"encoderblock_0", "encoderblock_1",
                                                                             "encoder_norm"}
  assert all(k.startswith("couplings/") or k.endswith("-FREEZE_ME") for k in tree)
  masks = sum(int(np.prod(s)) for k, s in shapes.items() if k.endswith("FREEZE_ME"))
  trained = sum(int(np.prod(s)) for k, s in shapes.items() if not k.endswith("FREEZE_ME"))
  assert (trained, masks) == (207_177_216, 2_170_880)


def test_runlocal_model_builds_and_initialises():
  jet = _jet()
  model = jet.Model(**{**IMAGENET64, "depth": 1, "block_depth": 1})
  P = model.init(0, (32, 64, 64, 3), device="cpu")
  tree = P.numpy_tree("f")
  assert tree["couplings/dnn/posemb"].shape == (1, 1, 256, 512)
  assert not np.any(tree["couplings/dnn/final_proj/kernel"]) and not np.any(tree["couplings/dnn/final_proj/bias"])
  assert np.std(tree["couplings/dnn/posemb"]) == pytest.approx(1 / np.sqrt(512), rel=0.05)
  assert P.jet_tables.shape == (1, 12288) and P.jet_tables.dtype == torch.int32


def test_coupling_order_is_the_reference_interleave():
  jet = _jet()
  order = jet.Model(**IMAGENET64).couplings
  spatial = [i for i, (k, _, _) in enumerate(order) if k == 0]
  assert spatial == list(range(4, 32, 5))
  assert [order[i][2] for i in spatial] == list(IMAGENET64["spatial_coupling_projs"])
  assert all(order[i] == (1, "random", "zero") for i in range(32) if i not in spatial)
  assert all(order[i][1] == "zero" for i in spatial)


# 4 x 4 tokens, row-major: (first half, second half) of each spatial kind, derived by hand
_KNOWN = {
    "checkerboard": ([0, 2, 5, 7, 8, 10, 13, 15], [1, 3, 4, 6, 9, 11, 12, 14]),
    "vstripes": ([0, 2, 4, 6, 8, 10, 12, 14], [1, 3, 5, 7, 9, 11, 13, 15]),
    "hstripes": ([0, 1, 2, 3, 8, 9, 10, 11], [4, 5, 6, 7, 12, 13, 14, 15]),
}


@pytest.mark.parametrize("kind", sorted(_KNOWN) + [k + "-inv" for k in sorted(_KNOWN)])
def test_spatial_mask_inits_match_known_answers(kind):
  jet = _jet()
  w = jet.spatial_masks(3, 4, 4, ["zero", kind, "zero"])
  assert not np.any(w[0]) and not np.any(w[2])
  first, second = _KNOWN[kind.replace("-inv", "")]
  if kind.endswith("-inv"):
    first, second = second, first
  want = np.zeros((16, 16), np.float32)
  want[first, np.arange(8)] = 1
  want[second, np.arange(8, 16)] = 1
  np.testing.assert_array_equal(w[1], want)


def test_channel_masks_are_permutations_and_placeholders_zero():
  jet = _jet()
  model = jet.Model(**TINY)
  P = model.init(3, (2, 16, 16, 3), device="cpu")
  cm = P.numpy_tree("f")["channel_coupling_masks-FREEZE_ME"]
  sm = P.numpy_tree("f")["spatial_coupling_masks-FREEZE_ME"]
  for i, (k, _, _) in enumerate(model.couplings):
    if k == 1:
      assert set(np.unique(cm[i])) == {0.0, 1.0}
      np.testing.assert_array_equal(cm[i].sum(0), 1)
      np.testing.assert_array_equal(cm[i].sum(1), 1)
      assert not np.any(sm[i])
    else:
      assert not np.any(cm[i])
  assert not np.array_equal(cm[0], cm[2])


# ---- index tables against the oracle's einsum -------------------------------------------------------------
@pytest.mark.parametrize("hw,ps", [((16, 16), 4), ((8, 16), 4)])
def test_index_tables_reproduce_the_oracle_split_and_merge(hw, ps):
  jet = _jet()
  model = jet.Model(depth=5, block_depth=1, emb_dim=64, num_heads=1, ps=ps, kinds=("channels", "spatial"),
                    spatial_coupling_projs=("checkerboard", "hstripes-inv", "vstripes"))
  P = model.init(1, (2,) + hw + (3,), device="cpu")
  tree = {k: torch.from_numpy(v).double() for k, v in P.numpy_tree("f").items()}
  T, dt = model.T, model.dt
  D = T * dt
  x = torch.randn(2, T, dt, dtype=torch.float64)
  for i, (k, _, _) in enumerate(model.couplings):
    idx = P.jet_tables[i].long()
    cm, sm = tree[JO.CH][i], tree[JO.SP][i]
    x1, x2 = JO.split(x, k, cm, sm)
    flat = x.reshape(2, D)
    assert torch.equal(flat[:, idx[:D // 2]].reshape(x1.shape), x1)
    assert torch.equal(flat[:, idx[D // 2:]].reshape(x2.shape), x2)
    y = torch.empty_like(flat)
    y[:, idx] = torch.cat([x1.reshape(2, -1), 2 * x2.reshape(2, -1)], 1)
    assert torch.equal(y.reshape(x.shape), JO.merge(x1, 2 * x2, k, cm, sm))


def test_a_mask_that_is_not_a_permutation_is_refused():
  jet = _jet()
  model = jet.Model(**TINY)
  P = model.init(0, (1, 16, 16, 3), device="cpu")
  tree = P.numpy_tree("f")
  bad = dict(tree)
  bad["channel_coupling_masks-FREEZE_ME"] = tree["channel_coupling_masks-FREEZE_ME"].copy()
  bad["channel_coupling_masks-FREEZE_ME"][0, :, 0] = 0        # an empty column
  with pytest.raises(ValueError, match="permutation"):
    P.load_tree(bad)
  bad["channel_coupling_masks-FREEZE_ME"] = tree["channel_coupling_masks-FREEZE_ME"] * 0.5
  with pytest.raises(ValueError, match="permutation"):
    P.load_tree(bad)
  bad = dict(tree)
  bad["spatial_coupling_masks-FREEZE_ME"] = np.zeros_like(tree["spatial_coupling_masks-FREEZE_ME"])
  with pytest.raises(ValueError, match="spatial"):
    P.load_tree(bad)


def test_load_tree_rederives_the_tables():
  jet = _jet()
  model = jet.Model(**TINY)
  P = model.init(0, (1, 16, 16, 3), device="cpu")
  other = model.init(5, (1, 16, 16, 3), device="cpu")
  assert not torch.equal(P.jet_tables, other.jet_tables)
  P.load_tree(other.numpy_tree("f"))
  assert torch.equal(P.jet_tables, other.jet_tables)


# ---- the noise generator ------------------------------------------------------------------------------
_M0, _M1 = 0xD2E7470EE14C6C93, 0xCA5A826395121157
_W0, _W1 = 0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B
_U64 = (1 << 64) - 1


def philox4x64_10(ctr, key):
  """Philox4x64-10 of Salmon et al. (SC'11) on Python integers."""
  c, k0, k1 = list(ctr), key[0], key[1]
  for r in range(10):
    if r:
      k0, k1 = (k0 + _W0) & _U64, (k1 + _W1) & _U64
    p0, p1 = _M0 * c[0], _M1 * c[2]
    c = [(p1 >> 64) ^ c[1] ^ k0, p1 & _U64, (p0 >> 64) ^ c[3] ^ k1, p0 & _U64]
  return c


def uniform_f32(seed, counter, offset, count):
  """The kernel's stream: element e from block e // 8 at counter (e // 8 + 1, counter, 0, 0), word (e % 8) // 2,
  low half first, u = (u32 >> 8) * 2^-24."""
  out = np.empty(count, np.float32)
  for i, e in enumerate(range(offset, offset + count)):
    word = philox4x64_10([e // 8 + 1, counter, 0, 0], (seed, 0))[(e % 8) // 2]
    u32 = (word >> (32 * (e % 2))) & 0xFFFFFFFF
    out[i] = np.float32(u32 >> 8) * np.float32(2.0 ** -24)
  return out


@pytest.mark.parametrize("seed,counter,offset,count", [(0, 0, 0, 37), (0, 5, 0, 16), (12345, 77, 13, 29),
                                                       (2 ** 40 + 3, 2 ** 33, 1000, 24)])
def test_philox_restatement_is_numpy_stream(seed, counter, offset, count):
  ref = np.random.Generator(np.random.Philox(key=seed, counter=[0, counter, 0, 0])).random(offset + count,
                                                                                            dtype=np.float32)
  np.testing.assert_array_equal(uniform_f32(seed, counter, offset, count), ref[offset:])


def test_numpy_increments_the_first_counter_word_before_its_first_block():
  ref = np.random.Generator(np.random.Philox(key=7, counter=[0, 3, 0, 0])).random(8, dtype=np.float32)
  at0 = philox4x64_10([0, 3, 0, 0], (7, 0))
  at1 = philox4x64_10([1, 3, 0, 0], (7, 0))
  first = lambda words: np.float32((words[0] & 0xFFFFFFFF) >> 8) * np.float32(2.0 ** -24)
  assert first(at1) == ref[0] and first(at0) != ref[0]


# ---- oracle properties ----------------------------------------------------------------------------------
def _tiny_oracle(depth=3, ps=2, hw=(4, 4), C=4, kinds=("channels", "spatial"), seed=0):
  """Oracle tree of a flow the library refuses to build (c % 8 != 0 is fine for the oracle): masks from the
  library's own initialisers, DNN weights random."""
  jet = _jet()
  T, dt = (hw[0] // ps) * (hw[1] // ps), ps * ps * C
  order = jet.interleave_couplings(depth, kinds, ("random",), ("checkerboard", "vstripes-inv"))
  rng = np.random.default_rng(seed)
  e, p = 64, {}
  _, ck, sk = zip(*order)
  p[JO.CH] = jet.channel_masks_init(depth, dt, ck)(rng, (depth, dt, dt))
  p[JO.SP] = jet.spatial_masks(depth, hw[0] // ps, hw[1] // ps, sk)
  pre = "couplings/dnn/"
  g = lambda *s: rng.normal(0, 0.2, s)
  p.update({pre + "init_proj/kernel": g(depth, dt // 2, e), pre + "init_proj/bias": g(depth, e),
            pre + "posemb": g(depth, 1, T, e), pre + "final_proj/kernel": g(depth, e, dt) * 0.3,
            pre + "final_proj/bias": g(depth, dt) * 0.3,
            pre + "vit/encoder_norm/scale": 1 + g(depth, e), pre + "vit/encoder_norm/bias": g(depth, e)})
  b = pre + "vit/encoderblock_0/"
  for ln in ("LayerNorm_0", "LayerNorm_1"):
    p[b + ln + "/scale"], p[b + ln + "/bias"] = 1 + g(depth, e), g(depth, e)
  for nm in ("query", "key", "value"):
    p[b + f"MultiHeadDotProductAttention_0/{nm}/kernel"] = g(depth, e, 1, e) / 4
    p[b + f"MultiHeadDotProductAttention_0/{nm}/bias"] = g(depth, 1, e)
  p[b + "MultiHeadDotProductAttention_0/out/kernel"] = g(depth, 1, e, e) / 4
  p[b + "MultiHeadDotProductAttention_0/out/bias"] = g(depth, e)
  p[b + "MlpBlock_0/Dense_0/kernel"], p[b + "MlpBlock_0/Dense_0/bias"] = g(depth, e, 4 * e) / 4, g(depth, 4 * e)
  p[b + "MlpBlock_0/Dense_1/kernel"], p[b + "MlpBlock_0/Dense_1/bias"] = g(depth, 4 * e, e) / 8, g(depth, e)
  cfg = dict(depth=depth, block_depth=1, num_heads=1, ps=ps, kinds=kinds)
  return {k: torch.as_tensor(np.asarray(v)).double() for k, v in p.items()}, cfg


def test_oracle_inverse_of_forward_is_the_identity():
  p, cfg = _tiny_oracle(depth=5, ps=2, hw=(8, 8), C=3)
  x = torch.rand(3, 8, 8, 3, dtype=torch.float64) * 2 - 1
  z, ld = JO.forward(p, x, cfg)
  y, ld_inv = JO.inverse(p, z, cfg)
  assert (y - x).abs().max() < 1e-12
  assert (ld + ld_inv).abs().max() < 1e-12
  assert ld.abs().min() > 1e-3              # the map is not volume preserving


def test_oracle_logdet_is_log_abs_det_of_the_jacobian():
  p, cfg = _tiny_oracle(depth=3, ps=2, hw=(4, 4), C=4)
  x = torch.rand(1, 4, 4, 4, dtype=torch.float64) * 2 - 1
  J = torch.autograd.functional.jacobian(lambda v: JO.forward(p, v.view(1, 4, 4, 4), cfg)[0].reshape(-1),
                                         x.reshape(-1))
  sign, logabs = torch.linalg.slogdet(J)
  _, ld = JO.forward(p, x, cfg)
  assert sign != 0
  assert abs(float(logabs) - float(ld[0])) < 1e-9


def test_oracle_bits_is_the_normal_logpdf():
  import scipy.stats
  rng = np.random.default_rng(0)
  z = rng.normal(size=(4, 5, 5, 3))
  logdet = rng.normal(size=4) * 10
  bits, nll, ld = JO.bits_per_dim(torch.from_numpy(z), torch.from_numpy(logdet))
  D = 75
  want_nll = -(scipy.stats.norm.logpdf(z) - np.log(127.5)).reshape(4, -1).sum(1)
  np.testing.assert_allclose(nll.numpy(), want_nll / (D * np.log(2)), rtol=1e-13)
  np.testing.assert_allclose(bits.numpy(), (want_nll - logdet) / (D * np.log(2)), rtol=1e-13)
  np.testing.assert_allclose(ld.numpy(), logdet / (D * np.log(2)), rtol=1e-13)


# ---- refusals ------------------------------------------------------------------------------------------
def _config(**kw):
  cfg = dict(seed=0, optax_name="scale_by_adam", optax=dict(mu_dtype="bfloat16", b2=0.95), grad_clip_norm=1.0,
             lr=3e-4, wd=1e-5, wd_mults=((".*", 1.0),),
             schedule=[(".*FREEZE_ME.*", None), (".*", dict(decay_type="cosine", warmup_percent=0.1))])
  cfg.update(kw)
  return cfg


def _tx(P, config):
  from big_vision_b200 import optax as bv_optax
  return bv_optax.make(config, P, sched_kw=dict(total_steps=10, batch_size=2, data_size=20))[0]


def test_update_fn_refuses_unfrozen_masks_and_labels():
  jet = _jet()
  from big_vision_b200.trainers.proj.jet import train as jt
  model = jet.Model(**TINY)
  P = model.init(0, (2, 16, 16, 3), device="cpu")
  unfrozen = _config(schedule=[(".*", dict(decay_type="cosine", warmup_percent=0.1))])
  with pytest.raises(NotImplementedError, match="frozen"):
    jt.make_update_fn(model, _tx(P, unfrozen), unfrozen)
  config = _config()
  tx = _tx(P, config)
  update_fn = jt.make_update_fn(model, tx, config)
  state = {"params": P, "opt": {"count": 0}}
  for key in ("label", "context"):
    with pytest.raises(NotImplementedError, match="class-conditional"):
      update_fn(state, None, {"image": torch.zeros(2, 16, 16, 3), key: torch.zeros(2, dtype=torch.int32)})
  with pytest.raises(NotImplementedError, match="class-conditional"):
    jt.make_predict_fns(model, config)["loss"](P, {"image": torch.zeros(2, 16, 16, 3), "label": None}, 0, 0)


@pytest.mark.parametrize("ps,C", [(2, 3), (2, 1), (2, 2)])
def test_half_tokens_that_are_not_a_multiple_of_8_are_refused(ps, C):
  jet = _jet()
  with pytest.raises(NotImplementedError, match="multiple of 8"):
    jet.Model(**{**TINY, "ps": ps}).specs((16, 16), C)


def test_jet_ops_refuse_cpu_tensors():
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  x, idx = torch.zeros(1, 4, 16), torch.arange(64, dtype=torch.int32)
  br, ld = torch.zeros(4, 16), torch.zeros(1)
  calls = [lambda: ops.jet_dequantize_patchify(torch.zeros(1, 8, 8, 1), 4),
           lambda: ops.jet_unpatchify(x, (1, 8, 8, 1), 4),
           lambda: ops.jet_split(x, idx, 4, 8),
           lambda: ops.jet_coupling_fwd(x, idx, br, ld, 4, 8),
           lambda: ops.jet_coupling_bwd(x, x, idx, br, 0.0, 4, 8),
           lambda: ops.jet_merge_grad(x, torch.zeros(4, 8), idx, 4, 8),
           lambda: ops.jet_bits(x, ld, 1.0)]
  for call in calls:
    with pytest.raises(L.BvError):
      call()
  with pytest.raises(L.BvError, match="contiguous"):
    ops.jet_split(x.double(), idx, 4, 8)
