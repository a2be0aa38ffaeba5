"""CPU: distillation (trainers/proj/distill, evaluators/proj/distill) -- its float64 oracle against closed
forms, config parsing and the refused distances, the choice of each model's input, the evaluator's summary,
and the refusal of CPU tensors by the distillation ops."""
import math
import os

import numpy as np
import pytest
import torch

import distill_oracle as DO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _logits(n, C, seed, scale=3.0):
  g = torch.Generator().manual_seed(seed)
  return torch.randn(n, C, generator=g, dtype=torch.float64) * scale


# ---- the oracle against closed forms -------------------------------------------------------------
def test_kl_of_equal_logits_is_zero_and_kl_is_positive():
  s = _logits(5, 11, 0)
  assert float(DO.dist(s, s, "kl", t=3).abs().max()) < 1e-12
  assert float(DO.dist(s, s + 1.7, "kl").abs().max()) < 1e-12          # softmax ignores a shift
  assert float(DO.dist(s, _logits(5, 11, 1), "kl").min()) > 0


def test_kl_is_the_textbook_divergence_times_t_squared():
  s, u = _logits(4, 9, 2), _logits(4, 9, 3)
  for t in (1, 2, 8):
    p, q = torch.softmax(u / t, -1), torch.softmax(s / t, -1)
    ref = t ** 2 * (p * (p.log() - q.log())).sum(-1)
    torch.testing.assert_close(DO.dist(s, u, "kl", t=t), ref, rtol=1e-12, atol=1e-14)
  # temperature -> infinity: t^2 KL -> half the squared distance of the centred logits, over C
  t = 1e4
  c = lambda x: x - x.mean(-1, keepdim=True)
  ref = ((c(s) - c(u)) ** 2).sum(-1) / (2 * 9)
  torch.testing.assert_close(DO.dist(s, u, "kl", t=t), ref, rtol=5e-3, atol=0)


def test_kl_clips_tiny_teacher_probabilities():
  """utils.py:280: p log(clip(p, 1e-8)), not p log p -- a class at p = 1e-12 contributes p log 1e-8."""
  u = torch.tensor([[0.0, math.log(1e-12)]], dtype=torch.float64)
  s = torch.zeros(1, 2, dtype=torch.float64)
  p = torch.softmax(u, -1)[0]
  ref = -(p * math.log(0.5)).sum() + p[0] * p[0].log() + p[1] * math.log(1e-8)
  assert float(DO.dist(s, u, "kl")) == pytest.approx(float(ref), rel=1e-13)
  assert float(DO.dist(s, u, "kl")) != pytest.approx(float((p * (p.log() - math.log(0.5))).sum()), rel=1e-12)


def test_hard_without_smoothing_is_softmax_xent_on_the_argmax():
  s, u = _logits(6, 7, 4), _logits(6, 7, 5)
  onehot = torch.nn.functional.one_hot(u.argmax(-1), 7).double()
  torch.testing.assert_close(DO.dist(s, u, "hard"), DO.softmax_xent(s, onehot), rtol=1e-13, atol=0)
  # smoothing: (1 - ls) on the pseudo-label, ls / (C - 1) elsewhere, plus the label entropy term
  ls = 0.1
  pl = (1 - ls) * onehot + ls / 6 * (1 - onehot)
  ref = DO.softmax_xent(s, pl) + (1 - ls) * math.log(1 - ls) + ls * math.log(ls / 6)
  torch.testing.assert_close(DO.dist(s, u, "hard", ls=ls), ref, rtol=1e-12, atol=0)
  # ties: the first maximal index is the pseudo-label
  u = torch.tensor([[1.0, 3.0, 3.0, 0.0]], dtype=torch.float64)
  s = _logits(1, 4, 6)
  assert float(DO.dist(s, u, "hard")) == pytest.approx(float(-torch.log_softmax(s, -1)[0, 1]), rel=1e-13)


def test_euclidean_kinds():
  s, u = _logits(3, 5, 7), _logits(3, 5, 8)
  torch.testing.assert_close(DO.dist(s, u, "l2"), ((s - u) ** 2).sum(-1))
  torch.testing.assert_close(DO.dist(s, u, "euclidean", epsilon=0.5), (((s - u) ** 2).sum(-1) + 0.5).sqrt())
  assert float(DO.dist(s, s + 2.0, "logsoftmax_euclidean", epsilon=1e-12).max()) == pytest.approx(1e-6, rel=1e-3)


def test_agree_tie_cases():
  # teacher's top-1 is class 2; the student ties classes 0, 2, 3 at the top: order 0, 2, 3 (lower index first)
  u = torch.tensor([[0.0, 1.0, 5.0, 2.0]])
  s = torch.tensor([[4.0, 1.0, 4.0, 4.0]])
  assert [int(DO.dist(s, u, "agree", k=k)) for k in (1, 2, 3)] == [0, 1, 1]
  # the teacher ties too: its first maximum (class 1) is its top-1
  u = torch.tensor([[0.0, 5.0, 5.0, 2.0]])
  s = torch.tensor([[0.0, 3.0, 9.0, 1.0]])
  assert [int(DO.dist(s, u, "agree", k=k)) for k in (1, 2)] == [0, 1]
  with pytest.raises(AssertionError, match="Unknown kind"):
    DO.dist(s, u, "cosine")


@pytest.mark.parametrize("t", [1, 2, 8])
def test_autograd_gradient_of_kl_is_the_closed_form(t):
  n, C = 5, 13
  s, u = _logits(n, C, 9).requires_grad_(), _logits(n, C, 10)
  DO.dist(s, u, "kl", t=t).mean().backward()
  ref = (t / n) * (torch.softmax(s.detach() / t, -1) - torch.softmax(u / t, -1))
  torch.testing.assert_close(s.grad, ref, rtol=1e-10, atol=1e-14)


def test_loss_fn_sums_teachers_and_reports_means():
  s, a, b = _logits(4, 6, 11), _logits(4, 6, 12), _logits(4, 6, 13)
  labels = torch.nn.functional.one_hot(torch.tensor([0, 5, 2, 2]), 6).double()
  loss, m = DO.loss_fn({"student": s, "a": a, "b": b}, ("a", "b"), labels, "kl", dict(t=2))
  assert float(loss) == pytest.approx(float(m["distill_loss_a"] + m["distill_loss_b"]), rel=1e-14)
  assert float(m["distill_loss_a"]) == pytest.approx(float(DO.dist(s, a, "kl", t=2).mean()), rel=1e-14)
  # the entropies are at temperature 1 whatever t is
  q = torch.softmax(s, -1)
  assert float(m["entropy_student"]) == pytest.approx(float(-(q * q.log()).sum(-1).mean()), rel=1e-13)
  assert float(m["task_loss_b"]) == pytest.approx(float(DO.softmax_xent(b, labels).mean()), rel=1e-14)
  assert "task_loss_student" not in DO.loss_fn({"student": s, "a": a}, ("a",))[1]


# ---- host side -----------------------------------------------------------------------------------
def test_getfirst_selects_a_models_own_input():
  from big_vision_b200.trainers.proj.distill import distill as D
  data = {"image": "i", "prof": "p"}
  assert D.getfirst(data, "prof", "image") == "p"
  assert D.getfirst(data, "student", "image") == "i"
  with pytest.raises(KeyError):
    D.getfirst({"labels": 0}, "student", "image")


def test_config_is_parsed_and_untrained_distances_are_refused():
  from big_vision_b200.trainers.proj.distill import distill as D
  models = {"student": object(), "prof": object()}
  assert D.parse_config(dict(teachers=["prof"]), models) == (("prof",), "kl", {})
  assert D.parse_config(dict(teachers=["prof"], distance="hard", distance_kw=dict(ls=0.1)), models) \
      == (("prof",), "hard", dict(ls=0.1))
  for kind in ("euclidean", "l2", "logsoftmax_euclidean", "agree"):
    with pytest.raises(NotImplementedError, match="kl and hard"):
      D.parse_config(dict(teachers=["prof"], distance=kind), models)
  with pytest.raises(ValueError, match="Unknown kind"):
    D.parse_config(dict(teachers=["prof"], distance="cosine"), models)
  with pytest.raises(ValueError, match="missing"):
    D.parse_config(dict(teachers=["prof", "prof2"]), models)
  with pytest.raises(TypeError, match="unknown"):
    D.parse_config(dict(teachers=["prof"], distance_kw=dict(temperature=2)), models)
  with pytest.raises(NotImplementedError):
    D.make_update_fn(models, object(), dict(teachers=["prof"], distance="l2"))


def test_a_teacher_needs_no_gradient_buffer():
  from big_vision_b200 import engine as E
  from big_vision_b200.models import vit
  model = vit.Model(10, width=64, depth=2, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type="gap")
  P = E.FlatParams(*model.specs((32, 32), 3), "cpu")
  name = next(iter(P.offsets))
  P.g(name)
  total = P.total
  assert P.drop_grad() is P and P.grad is None and P.total == total
  assert P.f(name).shape == P.offsets[name][1] and not any(k[0] == "g" for k in P._views)
  with pytest.raises(TypeError):
    P.g(name)


def test_summary_of_the_distance_evaluator():
  from big_vision_b200.evaluators.proj.distill import distance as dd
  out = dd.summarize("kind=kl_t=2", [torch.tensor([1.0, 9.0, 3.0]), torch.tensor([5.0, 7.0])],
                     [torch.tensor([1, 0, 1]), torch.tensor([1, 1])])
  assert out["kind=kl_t=2/all"].tolist() == [1.0, 3.0, 5.0, 7.0]
  assert (out["kind=kl_t=2/avg"], out["kind=kl_t=2/min"], out["kind=kl_t=2/max"]) == (4.0, 1.0, 7.0)
  assert dd.dist_name(dict(kind="kl", t=2)) == "kind=kl_t=2"
  assert dd.flatten(torch.zeros(3, 4, 5, 6)).shape == (3, 120)


def test_predict_fns_are_the_reference_set():
  from big_vision_b200.trainers.proj.distill import distill as D

  class Fake:
    def __init__(self, row):
      self.row = row

    def apply(self, variables, image):
      x = torch.tensor([self.row], dtype=torch.float32) + variables["params"]
      return x, {"logits": x}

  models = {"student": Fake([0.0, 0.0]), "a": Fake([0.0, math.log(3.0)]), "b": Fake([math.log(3.0), 0.0])}
  fns = D.make_predict_fns(models, dict(teachers=["a", "b"]))
  assert set(fns) == {"student_fwd", "a_fwd", "b_fwd", "teacher_ensemble_fwd", "student_a_fwd", "student_b_fwd",
                      "student_teacher_ensemble_fwd"}
  state = {"params": {"student": 1.0, "a": 0.0, "b": 0.0}}
  probs, out = fns["teacher_ensemble_fwd"](state, {"image": None})
  assert out == {} and probs.tolist() == [pytest.approx([0.5, 0.5])]      # mean of (1/4, 3/4) and (3/4, 1/4)
  (s, _), (t, _) = fns["student_a_fwd"](state, {"image": None})
  assert s.tolist() == [[1.0, 1.0]] and t.tolist() == [pytest.approx([0.0, math.log(3.0)])]


def test_distill_ops_refuse_cpu_tensors():
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  from big_vision_b200.evaluators.proj.distill import distance as dd
  x = torch.zeros(4, 8)
  with pytest.raises(L.BvError):
    ops.distill_loss(x, x)
  with pytest.raises(L.BvError):
    ops.distance(x, x, "agree", k=5)
  with pytest.raises(L.BvError):
    dd.dist(x, x, "kl")
  with pytest.raises(ValueError, match="Unknown kind"):
    ops.distance(x, x, "cosine")
