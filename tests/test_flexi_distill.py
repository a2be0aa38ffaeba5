"""CPU: the FlexiViT distillation trainer's host side (trainers/proj/flexi/distill.py) -- the predict functions
named as the reference names them for configs/proj/flexivit/i1k_deit3_distill.py, the teachers' own inputs,
the refusal of a call without exactly the flexible arguments, the per-step draws against the reference's own
helpers (committed golden values), mixup over the teacher-named input, and initialisation from plain-ViT
checkpoints whose grid and patch size differ from the student's."""
import json
import os

import numpy as np
import pytest
import torch

import flexi_oracle as FO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "flexi_choices.json")
SEQHW = (5, 6, 8, 10, 12, 15, 16, 20, 24, 30)
# the flexi, teacher and distance sections of configs/proj/flexivit/i1k_deit3_distill.py
I1K_DEIT3_DISTILL = dict(teachers=["prof"], distance="kl", distance_kw=dict(t=1.0), mixup=dict(p=1.0, n=2),
                         flexi=dict(seqhw=dict(v=SEQHW, p=(1,) * len(SEQHW))))


def _fd():
  from big_vision_b200.trainers.proj.flexi import distill as fd
  return fd


class _Fake:
  """A model whose apply returns what it was called with."""

  def __init__(self, name):
    self.name = name

  def apply(self, variables, image, **kw):
    return (self.name, variables["params"], image, kw), {}


class _Tx:
  def frozen(self):
    return frozenset()

  def update(self, P, opt, grad_mult=1.0):
    return torch.tensor([4.0, 9.0, 16.0, 0.0])


def _models():
  return {"student": _Fake("student"), "prof": _Fake("prof")}


def test_predict_fn_names_are_the_reference_names():
  """10 student variants, the teacher, and the 10 (student variant, teacher) pairs, in the reference's
  order: the names its configs' evaluators ask for (`pred="student_seqhw=5"`, `"prof"`,
  `"student_seqhw=5_prof"`)."""
  fns = _fd().make_predict_fns(_models(), I1K_DEIT3_DISTILL)
  student = [f"student_seqhw={s}" for s in SEQHW]
  assert list(fns) == student + ["prof"] + [f"{n}_prof" for n in student]


def test_teacher_reads_its_own_input_and_the_pairs_pass_seqhw_to_the_student_only():
  fns = _fd().make_predict_fns(_models(), I1K_DEIT3_DISTILL)
  state = {"params": {"student": "Ps", "prof": "Pt"}}
  batch = {"image": "img240", "prof": "img384", "labels": "y"}
  assert fns["prof"](state, batch) == (("prof", "Pt", "img384", {}), {})
  assert fns["prof"](state, {"image": "img240"}) == (("prof", "Pt", "img240", {}), {})
  assert fns["student_seqhw=12"](state, batch) == (("student", "Ps", "img240", {"seqhw": 12}), {})
  s, t = fns["student_seqhw=30_prof"](state, batch)
  assert s == (("student", "Ps", "img240", {"seqhw": 30}), {}) and t == (("prof", "Pt", "img384", {}), {})


def test_update_fn_demands_every_flexible_argument():
  fn = _fd().make_update_fn(_models(), _Tx(), I1K_DEIT3_DISTILL)
  with pytest.raises(TypeError, match="seqhw"):
    fn({}, None, {})
  with pytest.raises(TypeError, match="seqhw"):
    fn({}, None, {}, seqhw=5, other=1)
  with pytest.raises(TypeError, match="seqhw"):
    fn({}, None, {}, patch=8)


def test_untrained_distances_stay_refused():
  for kind in ("euclidean", "l2", "logsoftmax_euclidean", "agree"):
    with pytest.raises(NotImplementedError, match=kind):
      _fd().make_update_fn(_models(), _Tx(), dict(I1K_DEIT3_DISTILL, distance=kind))


def test_flexi_args_reproduce_the_reference_draws():
  """The seqhw of steps 1..200 for every (xid, wid) equal the reference helpers' draws for the config's
  uniform weights: every rank, calling with the same step, draws the same."""
  fd = _fd()
  golden = json.load(open(GOLDEN))
  assert golden["flexi"]["uniform"]["seqhw"]["v"] == list(SEQHW)
  assert golden["flexi"]["uniform"]["seqhw"]["p"] == list(I1K_DEIT3_DISTILL["flexi"]["seqhw"]["p"])
  keys = [k for k in golden["draws"] if k.startswith("uniform/")]
  assert len(keys) == 9
  for key in keys:
    _, xid, wid = key.split("/")
    got = [[fd.flexi_args(I1K_DEIT3_DISTILL, step, int(xid), int(wid))["seqhw"]] for step in range(1, 201)]
    assert got == golden["draws"][key], key


def test_mixup_covers_the_teacher_input_and_seqhw_reaches_the_student_only(monkeypatch):
  """One coefficient over image, labels and `prof` (distill.py:256-261); the drawn seqhw goes to the
  student's forward, the teachers get none."""
  from big_vision_b200 import ops
  from big_vision_b200 import utils as u
  from big_vision_b200.trainers.proj.distill import distill
  seen = {}

  def fake_loss_and_grads(models, params, data, teachers, kind, distance_kw, dist_view=None, frozen=None, **kw):
    seen.update(data=data, teachers=teachers, kw=kw)
    return {"distill_loss": torch.tensor(2.0), "distill_loss_prof": torch.tensor(2.0)}

  monkeypatch.setattr(ops, "mixup", lambda x, a: a * x + (1 - a) * torch.roll(x, 1, 0))
  monkeypatch.setattr(distill, "loss_and_grads", fake_loss_and_grads)
  g = torch.Generator().manual_seed(0)
  batch = {"image": torch.randn(4, 6, 6, 3, generator=g), "prof": torch.randn(4, 8, 8, 3, generator=g),
           "labels": torch.randn(4, 5, generator=g), "other": torch.randn(4, 2, generator=g)}
  fn = _fd().make_update_fn(_models(), _Tx(), I1K_DEIT3_DISTILL)
  _, m = fn({"params": {"student": None, "prof": None}, "opt": None}, np.random.default_rng(7), batch, seqhw=12)
  a = u.get_mixup(np.random.default_rng(7), 1.0).a
  assert 0.5 <= a < 1.0
  for k in ("image", "prof", "labels"):
    torch.testing.assert_close(seen["data"][k], a * batch[k] + (1 - a) * torch.roll(batch[k], 1, 0), rtol=0, atol=0)
  assert seen["data"]["other"] is batch["other"]
  assert seen["teachers"] == ("prof",) and seen["kw"] == {"seqhw": 12}
  assert float(m["training_loss"]) == 2.0 and float(m["l2_grads"]) == 2.0


# ---- initialisation from checkpoints -----------------------------------------------------------------
D = 64


def _vit(patch, **kw):
  from big_vision_b200.models import vit
  return vit.Model(7, width=D, depth=2, mlp_dim=128, num_heads=1, patch_size=(patch, patch), pool_type="tok",
                   rep_size=False, **kw)


def _save(model, image_hw, seed, path):
  """A plain-ViT checkpoint of `model` at `image_hw` with every leaf random."""
  from big_vision_b200 import engine as E
  from big_vision_b200 import utils as u
  P = E.FlatParams(*model.specs((image_hw, image_hw), 3), "cpu").init(seed)
  rng = np.random.default_rng(seed)
  flat = {k: rng.standard_normal(v.shape).astype(np.float32) * 0.1 for k, v in P.numpy_tree("f").items()}
  u.save_checkpoint_np(u.recover_tree(*zip(*flat.items())), path)
  return flat


def _config(tmp_path, **kw):
  """A student FlexiViT (base patch 8, 7 x 7 grid) under a ViT teacher at 96 px, as the two configs lay
  them out; the student's checkpoint is a plain ViT B/16-style tree at 384 px (24 x 24 grid)."""
  s_cfg = dict(width=D, depth=2, mlp_dim=128, num_heads=1, patch_size=(8, 8), pool_type="tok")
  t_cfg = dict(width=D, depth=2, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type="tok", rep_size=False)
  return dict(I1K_DEIT3_DISTILL, student_name="proj.flexi.vit", student=s_cfg, student_init=str(tmp_path / "s.npz"),
              prof_name="vit", prof=t_cfg, prof_init=str(tmp_path / "t.npz"), **kw)


def _params(config):
  from big_vision_b200 import engine as E
  from big_vision_b200.models import vit
  from big_vision_b200.models.proj.flexi import vit as fv
  student = fv.Model(7, **config["student"])
  teacher = vit.Model(7, **config["prof"])
  return {"student": E.FlatParams(*student.specs(None, 3), "cpu").init(0),
          "prof": E.FlatParams(*teacher.specs((96, 96), 3), "cpu").init(1)}


def test_init_loads_plain_vit_checkpoints_into_the_flexi_student_and_the_teacher(tmp_path):
  from big_vision_b200.models import vit
  fd = _fd()
  ckpt_s = _save(_vit(16), 384, 2, str(tmp_path / "s.npz"))
  ckpt_t = _save(_vit(16), 96, 3, str(tmp_path / "t.npz"))
  assert ckpt_s["embedding/kernel"].shape == (16, 16, 3, D) and ckpt_s["pos_embedding"].shape == (1, 576, D)
  config = _config(tmp_path, init_head_bias=-10.0)
  params = fd.init_params(_params(config), config)
  got, teacher = params["student"].numpy_tree("f"), params["prof"].numpy_tree("f")
  assert got["embedding/kernel"].shape == (8, 8, 3, D) and got["pos_embedding"].shape == (1, 49, D)
  ref_k = FO.resample_kernel(torch.from_numpy(ckpt_s["embedding/kernel"]).double(), 8).numpy()
  np.testing.assert_allclose(got["embedding/kernel"], ref_k, rtol=0, atol=1e-5 * np.abs(ref_k).max())
  ref_pe = vit.resample_posemb(old=ckpt_s["pos_embedding"], new=np.zeros((1, 49, D)))
  np.testing.assert_allclose(got["pos_embedding"], ref_pe, rtol=0, atol=1e-6)
  for k in got:
    if k not in ("embedding/kernel", "pos_embedding"):
      np.testing.assert_array_equal(got[k], ckpt_s[k], err_msg=k)      # head included: the checkpoint's
  assert set(teacher) == set(ckpt_t)
  for k in teacher:
    np.testing.assert_array_equal(teacher[k], ckpt_t[k], err_msg=k)
  assert torch.equal(params["student"].half, params["student"].flat.to(torch.bfloat16))


def test_init_head_bias_applies_where_the_head_is_not_loaded(tmp_path):
  """The i21k config's init_head_bias = -10 fills the head bias before loading: a student that keeps its
  fresh head (dont_load) or loads nothing starts at -10, its kernel at the zero init."""
  fd = _fd()
  _save(_vit(16), 384, 2, str(tmp_path / "s.npz"))
  ckpt_t = _save(_vit(16), 96, 3, str(tmp_path / "t.npz"))
  config = _config(tmp_path, init_head_bias=-10.0, student_load=dict(dont_load=("head/.*",)))
  params = fd.init_params(_params(config), config)
  s = params["student"].numpy_tree("f")
  assert np.all(s["head/bias"] == -10.0) and not np.any(s["head/kernel"])
  np.testing.assert_array_equal(params["prof"].numpy_tree("f")["head/bias"], ckpt_t["head/bias"])
  config = dict(_config(tmp_path, init_head_bias=-10.0), student_init=None)
  params = fd.init_params(_params(config), config)
  s = params["student"].numpy_tree("f")
  assert np.all(s["head/bias"] == -10.0)
  assert s["embedding/kernel"].shape == (8, 8, 3, D) and np.std(s["embedding/kernel"]) > 0   # the fresh init
  with pytest.raises(ValueError, match="prof_init"):
    fd.init_params(_params(config), dict(config, prof_init=None))
