"""CPU: FlexiViT's host side -- the resize matrices against torch's F.interpolate, the pseudo-inverse identity,
the float64 oracle against the ViT oracle, the per-step draws against the reference's own helpers (committed
golden values), the parameter tree, the refusals and checkpoint loading."""
import json
import os

import numpy as np
import pytest
import torch

import flexi_oracle as FO
from oracle import bv_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "flexi_choices.json")
SEQHW = (5, 6, 8, 10, 12, 15, 16, 20, 24, 30)            # configs/proj/flexivit/i21k_sup.py
PATCHES = tuple(240 // s for s in SEQHW)                  # 48 ... 8
I21K_SUP = dict(variant="B", pool_type="tok", posemb="learn", patch_size=(8, 8), posemb_size=(7, 7), seqhw=None)


def _fv():
  from big_vision_b200.models.proj.flexi import vit as fv
  return fv


# ---- resize matrices -----------------------------------------------------------------------------
@pytest.mark.parametrize("n_in,outs", [(7, SEQHW + (3, 4, 7)), (8, PATCHES + (4, 8)), (32, (8, 16, 24, 48))])
@pytest.mark.parametrize("antialias", [True, False])
def test_resize_weights_equal_torch_bilinear(n_in, outs, antialias):
  fv = _fv()
  for n_out in outs:
    w = fv.resize_weights(n_in, n_out, antialias)
    got = np.kron(w, w)
    ref = FO.resize_matrix(n_in, n_out, antialias).numpy()
    assert got.shape == (n_out * n_out, n_in * n_in)
    assert np.abs(got - ref).max() <= 1e-12, (n_in, n_out, antialias)


def test_model_matrices_are_the_two_resizes():
  fv = _fv()
  for s in SEQHW:
    ref = FO.resize_matrix(7, s, antialias=True).numpy()
    assert np.abs(fv.posemb_resize_matrix((7, 7), s) - ref).max() <= 1e-12
  for p in PATCHES + (4,):
    ref = FO.patch_matrix(8, p).numpy()
    assert np.abs(fv.pi_resize_matrix(8, p) - ref).max() <= 1e-10, p


@pytest.mark.parametrize("p0,p", [(8, 8), (8, 10), (8, 15), (8, 24), (8, 48), (32, 48), (16, 30)])
def test_pseudo_inverse_keeps_the_embedding_of_a_resized_patch(p0, p):
  """For p >= p0, R^T pinv(R^T) = I: <resize(x), W'> = <x, W> for every patch x and kernel column W."""
  fv = _fv()
  w = fv.resize_weights(p0, p, antialias=False)
  R = np.kron(w, w)
  M = fv.pi_resize_matrix(p0, p)
  assert np.abs(R.T @ M - np.eye(p0 * p0)).max() <= 1e-12
  rng = np.random.default_rng(p)
  x, W = rng.standard_normal((5, p0 * p0)), rng.standard_normal((p0 * p0, 3))
  np.testing.assert_allclose((x @ R.T) @ (M @ W), x @ W, rtol=0, atol=1e-11)


def test_resample_patchemb_matches_the_oracle():
  fv = _fv()
  old = np.random.default_rng(0).standard_normal((8, 8, 3, 16))
  assert fv.resample_patchemb(old, (8, 8)) is old
  for p in (4, 16, 30):
    ref = FO.resample_kernel(torch.from_numpy(old), p).numpy()
    np.testing.assert_allclose(fv.resample_patchemb(old, (p, p)), ref, rtol=0, atol=1e-11)
  with pytest.raises(NotImplementedError, match="square"):
    fv.resample_patchemb(old, (8, 16))


# ---- the oracle ------------------------------------------------------------------------------------
def _tree(model, in_ch=3, seed=0):
  """A reference-named float64 tree of `model` with every zero-initialised leaf randomised."""
  from big_vision_b200 import engine as E
  P = E.FlatParams(*model.specs(None, in_ch), "cpu").init(seed)
  rng = np.random.default_rng(seed + 1)
  return {k: (v.astype(np.float64) if np.any(v) else rng.standard_normal(v.shape) * 0.05)
          for k, v in P.numpy_tree("f").items()}


@pytest.mark.parametrize("pool,posemb", [("tok", "learn"), ("gap", "sincos2d"), ("map", "learn")])
def test_oracle_at_base_patch_and_grid_is_the_vit_oracle(pool, posemb):
  fv = _fv()
  model = fv.Model(10, width=64, depth=1, mlp_dim=64, num_heads=1, patch_size=(8, 8), pool_type=pool, posemb=posemb)
  tree = O.to_f64_tree(_tree(model))
  image = torch.from_numpy(np.random.default_rng(3).uniform(-1, 1, (2, 56, 56, 3)))
  cfg = dict(depth=1, num_heads=1, pool_type=pool, posemb=posemb, posemb_size=(7, 7), num_classes=10)
  got = FO.flexi_forward(tree, image, cfg, 7)
  ref = O.vit_forward(tree, image, {**cfg, "rep_size": False})
  assert torch.equal(got, ref)


def test_oracle_resamples_kernel_and_posemb():
  """At seqhw 5 on 240 px (p = 48) the flexi oracle is the ViT oracle on the resampled kernel and table."""
  fv = _fv()
  model = fv.Model(4, width=64, depth=1, mlp_dim=64, num_heads=1, patch_size=(8, 8), pool_type="gap")
  tree = O.to_f64_tree(_tree(model))
  image = torch.from_numpy(np.random.default_rng(4).uniform(-1, 1, (1, 240, 240, 3)))
  cfg = dict(depth=1, num_heads=1, pool_type="gap", posemb="learn", posemb_size=(7, 7), num_classes=4)
  q = dict(tree)
  q["embedding/kernel"] = torch.from_numpy(fv.resample_patchemb(tree["embedding/kernel"].numpy(), (48, 48)))
  q["pos_embedding"] = torch.from_numpy(fv.posemb_resize_matrix((7, 7), 5) @ tree["pos_embedding"].numpy()[0])[None]
  torch.testing.assert_close(FO.flexi_forward(tree, image, cfg, 5), O.vit_forward(q, image, {**cfg, "rep_size": False}),
                             rtol=1e-10, atol=1e-12)


# ---- the trainer's draws -----------------------------------------------------------------------------
def test_flexi_args_reproduce_the_reference_draws():
  from big_vision_b200.trainers.proj.flexi import train as ft
  golden = json.load(open(GOLDEN))
  assert len(golden["draws"]) == 18
  for key, rows in golden["draws"].items():
    name, xid, wid = key.split("/")
    config = {"flexi": golden["flexi"][name]}
    names = sorted(config["flexi"])
    got = [[ft.flexi_args(config, step, int(xid), int(wid))[n] for n in names] for step in range(1, 201)]
    assert got == rows, key
  draws = {r[0] for r in golden["draws"]["uniform/-1/-1"]}
  assert draws == set(SEQHW)


def test_predict_fn_names_are_the_reference_names():
  from big_vision_b200.trainers.proj.flexi import common as fc
  from big_vision_b200.trainers.proj.flexi import train as ft
  golden = json.load(open(GOLDEN))
  fns = fc.mkpredictfns(lambda **kw: kw, {"seqhw": {"v": [5, 30]}, "alpha": {"v": [0.5, 2.0]}})
  assert list(fns) == golden["predict_names"]
  assert [fns[k]() for k in fns] == golden["predict_kw"]

  class Fake:
    def apply(self, variables, image, *, seqhw=None, train=False):
      return (variables["params"], image, seqhw), {}

  fns = ft.make_predict_fns(Fake(), {"flexi": {"seqhw": {"v": SEQHW, "p": [1] * 10}}})
  assert list(fns) == [f"predict_seqhw={s}" for s in SEQHW]
  assert fns["predict_seqhw=12"]("P", "img") == (("P", "img", 12), {})


def test_update_fn_demands_every_flexible_argument():
  from big_vision_b200.trainers.proj.flexi import train as ft

  class Tx:
    def frozen(self):
      return frozenset()

  fn = ft.make_update_fn(object(), Tx(), {"flexi": {"seqhw": {"v": (5,), "p": (1,)}}})
  with pytest.raises(TypeError, match="seqhw"):
    fn({}, None, {})
  with pytest.raises(TypeError, match="seqhw"):
    fn({}, None, {}, seqhw=5, other=1)


# ---- parameter tree and refusals ----------------------------------------------------------------------
def test_parameter_tree_has_the_reference_names_shapes_and_init():
  from big_vision_b200 import engine as E
  fv = _fv()
  d = 64
  model = fv.Model(21, width=d, depth=2, mlp_dim=128, num_heads=1, patch_size=(8, 8), pool_type="tok")
  P = E.FlatParams(*model.specs(None, 3), "cpu").init(0)
  tree = P.numpy_tree("f")
  shapes = {k: v.shape for k, v in tree.items() if not k.startswith("Transformer/")}
  assert shapes == {"embedding/kernel": (8, 8, 3, d), "embedding/bias": (d,), "pos_embedding": (1, 49, d),
                    "cls": (1, 1, d), "head/kernel": (d, 21), "head/bias": (21,)}
  blocks = {k.split("/")[1] for k in tree if k.startswith("Transformer/")}
  assert blocks == {"encoderblock_0", "encoderblock_1", "encoder_norm"}
  assert tree["Transformer/encoderblock_0/MultiHeadDotProductAttention_0/query/kernel"].shape == (d, 1, d)
  for k in ("embedding/kernel", "pos_embedding"):
    assert np.std(tree[k]) == pytest.approx(1 / np.sqrt(d), rel=0.1), k
    assert np.abs(tree[k]).max() > 2.5 / np.sqrt(d), k       # normal, not truncated like lecun_normal
  for k in ("embedding/bias", "cls", "head/kernel", "head/bias"):
    assert not np.any(tree[k]), k
  gap = fv.Model(21, width=d, depth=1, mlp_dim=128, num_heads=1, patch_size=(8, 8), pool_type="map",
                 posemb="sincos2d", head_zeroinit=False)
  names = set(E.FlatParams(*gap.specs(None, 3), "cpu").numpy_tree("f"))
  assert "pos_embedding" not in names and "cls" not in names and "MAPHead_0/probe" in names
  assert not any(n.startswith("pre_logits") for n in names)


def test_i21k_sup_model_builds():
  fv = _fv()
  model = fv.Model(21843, **I21K_SUP)
  specs, _ = model.specs(None, 3)
  shapes = {s.name: s.shape for s in specs}
  assert shapes["embedding/kernel_flat"] == (192, 768) and shapes["pos_embedding"] == (1, 49, 768)
  assert shapes["head/kernel_pad"] == (768, 21848) and shapes["cls"] == (1, 1, 768)
  assert (model.width, model.depth, model.mlp, model.num_heads) == (768, 12, 3072, 12)
  assert [model.geom(torch.empty(1, 240, 240, 3), s).N for s in SEQHW] == [s * s + 1 for s in SEQHW]
  scanned = fv.Model(21843, **I21K_SUP, scan=True)
  assert "Transformer/encoderblock/LayerNorm_0/scale" in {s.name for s in scanned.specs(None, 3)[0]}


def test_refusals():
  from big_vision_b200 import engine as E
  fv = _fv()
  model = fv.Model(10, width=64, depth=1, mlp_dim=64, num_heads=1, patch_size=(8, 8))
  P = E.FlatParams(*model.specs(None, 3), "cpu").init(0)
  with pytest.raises(NotImplementedError, match="non-square"):
    model.fwd(P, torch.zeros(1, 48, 40, 3), seqhw=8)
  with pytest.raises(NotImplementedError, match="not a multiple"):
    model.fwd(P, torch.zeros(1, 50, 50, 3), seqhw=8)
  with pytest.raises(ValueError, match="seqhw"):
    model.fwd(P, torch.zeros(1, 56, 56, 3))
  with pytest.raises(ValueError, match="pool type"):
    fv.Model(10, pool_type="0")
  with pytest.raises(NotImplementedError, match="square patches"):
    fv.Model(10, patch_size=(8, 16))


# ---- checkpoint loading --------------------------------------------------------------------------------
def test_load_resamples_a_patch16_checkpoint_into_a_patch8_model(tmp_path):
  """A ViT-style B/16 tree at 224 px (14 x 14 posemb) loads into a patch-8, 7 x 7 model: the kernel by the
  pseudo-inverse resample, the table by vit.resample_posemb, everything else as stored."""
  import scipy.ndimage
  from big_vision_b200 import engine as E
  from big_vision_b200 import utils as u
  fv = _fv()
  d = 64
  kw = dict(width=d, depth=2, mlp_dim=128, num_heads=1, pool_type="tok")
  init = u.recover_tree(*zip(*E.FlatParams(*fv.Model(5, patch_size=(8, 8), **kw).specs(None, 3), "cpu")
                             .init(1).numpy_tree("f").items()))
  ckpt = u.recover_tree(*zip(*_tree(fv.Model(5, patch_size=(16, 16), **kw)).items()))
  ckpt["pos_embedding"] = np.random.default_rng(2).standard_normal((1, 196, d))
  path = os.path.join(tmp_path, "b16.npz")
  u.save_checkpoint_np(ckpt, path)
  got = fv.load(init, path, dict(patch_size=(8, 8), **kw))
  ref_k = FO.resample_kernel(torch.from_numpy(ckpt["embedding"]["kernel"]), 8).numpy()
  np.testing.assert_allclose(got["embedding"]["kernel"], ref_k, rtol=0, atol=1e-11)
  ref_pe = scipy.ndimage.zoom(ckpt["pos_embedding"].reshape(14, 14, d), (0.5, 0.5, 1), order=1).reshape(1, 49, d)
  np.testing.assert_allclose(got["pos_embedding"], ref_pe, rtol=0, atol=1e-12)
  np.testing.assert_array_equal(got["Transformer"]["encoderblock_1"]["MlpBlock_0"]["Dense_0"]["kernel"],
                                ckpt["Transformer"]["encoderblock_1"]["MlpBlock_0"]["Dense_0"]["kernel"])
  kept = fv.load(init, path, dict(patch_size=(8, 8), **kw), dont_load=("head/.*",))
  np.testing.assert_array_equal(kept["head"]["kernel"], init["head"]["kernel"])
  # into a scanned model: the blocks are stacked
  scanned = fv.load(None, path, dict(patch_size=(8, 8), scan=True, **kw))
  assert scanned["Transformer"]["encoderblock"]["LayerNorm_0"]["scale"].shape == (2, d)


def test_flexi_ops_refuse_cpu_tensors():
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  M, x = torch.zeros(4, 2), torch.zeros(2, 8)
  with pytest.raises(L.BvError):
    ops.resample_fwd(M, x)
  with pytest.raises(L.BvError):
    ops.resample_bwd(M, torch.zeros(4, 8), x)
  with pytest.raises(L.BvError, match="fp32"):
    ops.resample_fwd(M.double(), x)
