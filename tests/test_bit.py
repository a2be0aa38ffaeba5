"""CPU: the BiT ResNet-v2 model (models/bit_paper.py): its parameter tree against the reference's layout, its
parameter count, the float64 oracle's own checks, checkpoint conversion of TF-dumped BiT files and the refusal
of the paper's gs:// short names, and the trainer plumbing shared with the FlexiViT distillation trainer."""
import numpy as np
import pytest
import torch

import bit_oracle as O
from big_vision_b200.models import bit_paper


def _reference_layout(depth, width, classes):
  """{name: shape} that bit_paper.Model(num_classes, width, depth) creates (bit_paper.py:61-156)."""
  w = int(64 * width)
  out = {"root_block/conv_root/kernel": (7, 7, 3, w)}
  cin = w
  for b, size in enumerate(O.block_desc(depth)):
    nmid = w * 2 ** b
    for u in range(size):
      pre = f"block{b + 1}/unit{u + 1:02d}/"
      out[pre + "gn1/scale"] = out[pre + "gn1/bias"] = (1, 1, 1, cin)
      if cin != 4 * nmid or (b > 0 and u == 0):
        out[pre + "conv_proj/kernel"] = (1, 1, cin, 4 * nmid)
      out[pre + "conv1/kernel"] = (1, 1, cin, nmid)
      out[pre + "gn2/scale"] = out[pre + "gn2/bias"] = (1, 1, 1, nmid)
      out[pre + "conv2/kernel"] = (3, 3, nmid, nmid)
      out[pre + "gn3/scale"] = out[pre + "gn3/bias"] = (1, 1, 1, nmid)
      out[pre + "conv3/kernel"] = (1, 1, nmid, 4 * nmid)
      cin = 4 * nmid
  out["norm-pre-head/scale"] = out["norm-pre-head/bias"] = (1, 1, 1, cin)
  out["head/kernel"], out["head/bias"] = (cin, classes), (classes,)
  return out


@pytest.mark.parametrize("depth,width,count", [(50, 1, 25_549_352), (152, 2, 236_335_208)])
def test_parameter_tree_matches_the_reference_layout(depth, width, count):
  specs, aliases = bit_paper.Model(num_classes=1000, depth=depth, width=width).specs((224, 224))
  got = {s.name: tuple(s.shape) for s in specs}
  assert not aliases
  assert got == _reference_layout(depth, width, 1000)
  assert sum(int(np.prod(s)) for s in got.values()) == count


def test_block_descriptions():
  assert [bit_paper.get_block_desc(d) for d in (26, 50, 101, 152, 200)] == [
      [2, 2, 2, 2], [3, 4, 6, 3], [3, 4, 23, 3], [3, 8, 36, 3], [3, 24, 36, 3]]
  assert bit_paper.get_block_desc([1, 2, 1, 1]) == (1, 2, 1, 1)


def test_init_follows_flax_defaults():
  specs, _ = bit_paper.Model(num_classes=16, depth=[1, 1, 1, 1]).specs((32, 32))
  rng = np.random.default_rng(0)
  by = {s.name: np.asarray(s.init(rng, s.shape)) for s in specs}
  assert (by["head/kernel"] == 0).all() and (by["head/bias"] == 0).all()
  assert (by["block1/unit01/gn1/scale"] == 1).all() and (by["block1/unit01/gn1/bias"] == 0).all()
  k = by["block3/unit01/conv2/kernel"]
  assert abs(k.std() - (9 * 256) ** -0.5) < 0.05 * (9 * 256) ** -0.5 and np.abs(k).max() <= 2 * (9 * 256) ** -0.5 / 0.8796 + 1e-6


def test_oracle_standardises_and_pads_with_minus_inf():
  k = torch.randn(3, 3, 4, 5, dtype=torch.float64) * 3 + 1
  s = O.standardize(k, axis=(0, 1, 2), eps=1e-10)
  assert torch.allclose(s.mean(dim=(0, 1, 2)), torch.zeros(5, dtype=torch.float64), atol=1e-12)
  assert torch.allclose((s * s).mean(dim=(0, 1, 2)), torch.ones(5, dtype=torch.float64), atol=1e-9)
  x = -torch.ones(1, 3, 3, 1, dtype=torch.float64)
  assert O.max_pool(x)[0, 0, 0, 0] == -1.0          # a zero pad would give 0


def _tf_tree(depth, width, classes, rng):
  """A synthetic TF-dumped BiT checkpoint for bit_paper.Model(classes, width, depth), flat."""
  ref = _reference_layout(depth, width, classes)
  tf = {}
  for name, shape in ref.items():
    v = rng.standard_normal(shape).astype(np.float32)
    parts = name.split("/")
    if name == "root_block/conv_root/kernel":
      tf["resnet/root_block/standardized_conv2d/kernel"] = v
    elif name.startswith("norm-pre-head/"):
      tf["resnet/group_norm/" + {"scale": "gamma", "bias": "beta"}[parts[1]]] = v[0, 0, 0]
    elif name == "head/kernel":
      tf["resnet/head/conv2d/kernel"] = v[None, None]
    elif name == "head/bias":
      tf["resnet/head/conv2d/bias"] = v
    elif parts[2] == "conv_proj":
      tf[f"resnet/{parts[0]}/{parts[1]}/a/proj/standardized_conv2d/kernel"] = v
    elif parts[2].startswith("conv"):
      g = "abc"[int(parts[2][-1]) - 1]
      # some files number the convolutions: standardized_conv2d_3
      suffix = "_3" if parts[1] == "unit01" and g == "b" else ""
      tf[f"resnet/{parts[0]}/{parts[1]}/{g}/standardized_conv2d{suffix}/kernel"] = v
    else:
      g = "abc"[int(parts[2][-1]) - 1]
      tf[f"resnet/{parts[0]}/{parts[1]}/{g}/group_norm/" + {"scale": "gamma", "bias": "beta"}[parts[3]]] = v[0, 0, 0]
  return ref, tf


def test_load_converts_a_tf_dumped_checkpoint(tmp_path):
  from big_vision_b200 import utils as u
  depth, classes = [2, 1, 1, 1], 8
  ref, tf = _tf_tree(depth, 1, classes, np.random.default_rng(1))
  assert any("/a/proj/" in k for k in tf) and any(k.startswith("resnet/block1/unit02/") for k in tf)
  assert not any(k.startswith("resnet/block1/unit02/a/proj") for k in tf)    # a unit without a projection
  path = str(tmp_path / "bit.npz")
  np.savez(path, **tf)
  specs, _ = bit_paper.Model(num_classes=classes, depth=depth).specs((32, 32))
  init = u.recover_tree([s.name for s in specs], [np.zeros(s.shape, np.float32) for s in specs])
  tree = dict(u.tree_flatten_with_names(bit_paper.load(init, path, {"depth": depth, "width": 1}))[0])
  assert set(tree) == set(ref)
  assert np.array_equal(tree["block1/unit01/conv2/kernel"], tf["resnet/block1/unit01/b/standardized_conv2d_3/kernel"])
  assert np.array_equal(tree["block2/unit01/conv_proj/kernel"], tf["resnet/block2/unit01/a/proj/standardized_conv2d/kernel"])
  assert np.array_equal(tree["block3/unit01/gn2/scale"][0, 0, 0], tf["resnet/block3/unit01/b/group_norm/gamma"])
  assert np.array_equal(tree["head/kernel"], tf["resnet/head/conv2d/kernel"][0, 0])
  # dont_load keeps the fresh head
  tree = dict(u.tree_flatten_with_names(bit_paper.load(init, path, {}, dont_load=["head/.*"]))[0])
  assert (tree["head/kernel"] == 0).all()


@pytest.mark.parametrize("name", ["M", "S", "L-imagenet2012", "M-run0-caltech101", "FunMatch-224px-i1k82.8"])
def test_short_names_ask_for_a_local_file(name):
  with pytest.raises(ValueError, match="local"):
    bit_paper.load(None, name, {"depth": 50, "width": 1})


def test_distillation_init_is_shared_with_the_flexi_trainer():
  from big_vision_b200.trainers.proj.distill import distill
  from big_vision_b200.trainers.proj.flexi import distill as fd
  assert fd.init_params is distill.init_params
  cfg = {"student_name": "bit_paper", "prof_m_name": "bit_paper"}
  assert distill._model_module(cfg, "prof_m") is bit_paper
