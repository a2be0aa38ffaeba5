"""GPU: the BiT ResNet-v2 (models/bit_paper.py) against the oracles of tests/bit_oracle.py: a small model
forward and backward, the frozen path, one distillation step of a BiT student under a BiT teacher, and R50x1 at
224 px.  Each tensor is compared in the relative Frobenius norm ||got - want|| / ||want||.

The gradients are pinned to the bf16-emulating oracle.  The activations are bf16, so against plain float64 a
ReLU or a max-pool argmax whose input lies within a bf16 rounding of its threshold decides differently and
moves a whole gradient term: with 8 terms per channel in a small model's GroupNorm bias that is tens of
percent, and says nothing about the kernels.  Even against the bf16-emulating oracle the two accumulation
orders round a few stored activations one ulp apart, and across a whole model the decisions those flip add
up to 15-20 % in a small model's gradients: so the whole model's gradients are held to a bound that catches a
wrong sign, scale or routing only, and every residual unit is pinned on its own inputs, where the gradients
agree within 2 %.  The logits are checked against both oracles."""
import numpy as np
import pytest
import torch

import bit_oracle as O
from big_vision_b200 import utils as u
from big_vision_b200.models import bit_paper

pytestmark = pytest.mark.gpu


def _model(depth, width, classes, hw, seed):
  m = bit_paper.Model(num_classes=classes, depth=depth, width=width, head_zeroinit=False)
  P = m.init(seed, (1, hw, hw, 3))
  return m, P


def _tree(P):
  return {k: v.detach().cpu().numpy().astype(np.float64) for k, v in P.tree("f").items()}


def _rel(got, want):
  return float(np.linalg.norm(np.asarray(got, np.float64) - want) / (np.linalg.norm(want) + 1e-30))


def _fwd_bwd(m, P, image, dlogits):
  P.zero_grad()
  logits, saved = m.fwd(P, image)
  m.bwd(P, dlogits, saved)
  torch.cuda.synchronize()
  return logits.cpu().numpy(), {k: v.cpu().numpy() for k, v in P.tree("g").items()}


@pytest.mark.parametrize("depth,width,hw", [([1, 1, 1, 1], 1, 64), ([2, 2, 1, 1], 1, 48), ([1, 1, 1, 1], 2, 40)])
def test_small_model_forward_and_backward_match_fp64(depth, width, hw):
  classes = 16
  m, P = _model(depth, width, classes, hw, seed=1)
  gen = np.random.default_rng(2)
  image = gen.standard_normal((2, hw, hw, 3)).astype(np.float32)
  dlogits = gen.standard_normal((2, classes)).astype(np.float32)
  logits, grads = _fwd_bwd(m, P, torch.from_numpy(image).cuda(), torch.from_numpy(dlogits).cuda())
  want, _ = O.value_and_grads(_tree(P), image, depth, dlogits)
  assert _rel(logits, want) < 5e-2
  want, want_g = O.value_and_grads(_tree(P), image, depth, dlogits, bf16=True)
  assert _rel(logits, want) < 2e-2
  assert set(grads) == set(want_g)
  assert all(np.isfinite(g).all() for g in grads.values())
  bad = {k: _rel(g, want_g[k]) for k, g in grads.items()}
  bad = {k: v for k, v in bad.items() if v >= 0.3}
  assert not bad, bad


def test_frozen_apply_gives_the_bits_of_fwd():
  m, P = _model([1, 2, 1, 1], 1, 16, 48, seed=3)
  image = torch.randn(3, 48, 48, 3, device="cuda")
  a, _ = m.apply({"params": P}, image)
  b, _ = m.fwd(P, image)
  assert torch.equal(a, b)
  # a linear probe: only the head is trained, so only the head gets a gradient
  frozen = {s.name for s in P.specs if not s.name.startswith("head/")}
  P.zero_grad()
  logits, saved = m.fwd(P, image, frozen=frozen)
  assert all(s is None for s in saved["stages"][:-1])
  m.bwd(P, torch.ones(3, 16, device="cuda"), saved)
  g = P.tree("g")
  assert (g["block1/unit01/conv1/kernel"] == 0).all() and (g["head/kernel"] != 0).any()


def test_distillation_step_with_a_bit_teacher():
  from big_vision_b200.trainers.proj.distill import distill
  models, params = {}, {}
  models["student"], params["student"] = _model([1, 1, 1, 1], 1, 16, 64, seed=4)
  models["prof_m"], params["prof_m"] = _model([1, 2, 1, 1], 2, 16, 64, seed=5)
  params["prof_m"].drop_grad()
  teacher_before = params["prof_m"].flat.clone()
  gen = torch.Generator().manual_seed(6)
  data = {"image": torch.randn(4, 64, 64, 3, generator=gen).cuda()}
  runs = []
  for _ in range(2):
    m = distill.loss_and_grads(models, params, data, ("prof_m",), "kl")
    runs.append((m["distill_loss"].item(), params["student"].grad.clone()))
  assert params["prof_m"].grad is None
  assert torch.equal(params["prof_m"].flat, teacher_before)
  assert runs[0][0] == runs[1][0]
  # against the oracle: kl(teacher || student) with t = 1, mean over the batch
  img = data["image"].cpu().numpy()
  t = torch.tensor(O.forward({k: torch.tensor(v) for k, v in _tree(params["prof_m"]).items()},
                             torch.tensor(img, dtype=torch.float64), [1, 2, 1, 1]))
  s = torch.tensor(O.forward({k: torch.tensor(v) for k, v in _tree(params["student"]).items()},
                             torch.tensor(img, dtype=torch.float64), [1, 1, 1, 1]))
  kl = (torch.softmax(t, -1) * (torch.log_softmax(t, -1) - torch.log_softmax(s, -1))).sum(-1).mean().item()
  assert abs(runs[0][0] - kl) <= 3e-2 * abs(kl) + 1e-3


def test_r50x1_at_224_matches_fp64():
  m, P = _model(50, 1, 1000, 224, seed=7)
  gen = np.random.default_rng(8)
  image = gen.standard_normal((2, 224, 224, 3)).astype(np.float32)
  dlogits = gen.standard_normal((2, 1000)).astype(np.float32)
  logits, grads = _fwd_bwd(m, P, torch.from_numpy(image).cuda(), torch.from_numpy(dlogits).cuda())
  want, _ = O.value_and_grads(_tree(P), image, 50, dlogits)
  assert _rel(logits, want) < 8e-2
  want, want_g = O.value_and_grads(_tree(P), image, 50, dlogits, bf16=True)
  assert _rel(logits, want) < 3e-2
  # the top of the backward only: every deeper gradient also depends on activations that 16 units of flipped
  # decisions have moved (the units and the root block are pinned on their own inputs below)
  for k in ("norm-pre-head/scale", "norm-pre-head/bias", "head/kernel", "head/bias"):
    assert _rel(grads[k], want_g[k]) < 0.3, (k, _rel(grads[k], want_g[k]))


@pytest.mark.parametrize("cin,nmid,stride,hw", [(64, 64, 1, 16), (256, 64, 1, 12), (256, 128, 2, 12), (512, 128, 1, 7),
                                                (1024, 512, 2, 8)])
def test_each_residual_unit_backward_on_its_own_inputs(cin, nmid, stride, hw):
  """One residual unit's forward and backward against the bf16-emulating oracle on the same bf16 input and
  output gradient: within one unit a ReLU decision rarely differs, so this pins every gradient it writes."""
  unit = bit_paper.ResidualUnit("u/", cin, nmid, stride)
  specs, _ = unit.specs()
  from big_vision_b200 import engine as E
  P = E.FlatParams(specs, [], "cuda").init(9)
  gen = torch.Generator().manual_seed(cin + nmid + hw)
  with torch.no_grad():
    for s in specs:
      if "/gn" in s.name:     # GroupNorm parameters away from their init, so every term of the backward counts
        P.f(s.name).add_(0.3 * torch.randn(P.f(s.name).shape, generator=gen).cuda())
  P.sync_half()
  x = torch.randn(2, hw, hw, cin, generator=gen).to(torch.bfloat16)
  ho = (hw - 1) // stride + 1
  dy = torch.randn(2, ho, ho, 4 * nmid, generator=gen).to(torch.bfloat16)
  P.zero_grad()
  out, saved = unit.fwd(P, x.cuda(), E.Geom(2, 0))
  dx = unit.bwd(P, dy.cuda(), saved, E.Geom(2, 0), None)
  torch.cuda.synchronize()
  tree = {k: torch.tensor(v, requires_grad=True) for k, v in _tree(P).items()}
  x64 = x.double().requires_grad_()
  O.BF16[0] = True
  try:
    want = O.unit(tree, x64, "u/", stride)
  finally:
    O.BF16[0] = False
  grads = torch.autograd.grad(want, [x64] + list(tree.values()), dy.double())
  assert _rel(out.float().cpu().numpy(), want.detach().numpy()) < 1e-2
  assert _rel(dx.float().cpu().numpy(), grads[0].numpy()) < 2e-2
  g = P.tree("g")
  for (k, _), gw in zip(tree.items(), grads[1:]):
    assert _rel(g[k].cpu().numpy(), gw.numpy()) < 2e-2, (k, _rel(g[k].cpu().numpy(), gw.numpy()))


def test_root_block_backward_on_its_own_inputs():
  """The root block's kernel gradient against the bf16-emulating oracle on the same image and output
  gradient (its max pool routes as the kernels' does: the oracle's convolution output is the same bf16)."""
  from big_vision_b200 import engine as E
  root = bit_paper.RootBlock(64)
  specs, _ = root.specs()
  P = E.FlatParams(specs, [], "cuda").init(10)
  gen = torch.Generator().manual_seed(11)
  image = torch.randn(2, 36, 36, 3, generator=gen)
  P.zero_grad()
  out, saved = root.fwd(P, image.cuda(), E.Geom(2, 0))
  dy = torch.randn(out.shape, generator=gen).to(torch.bfloat16)
  root.bwd(P, dy.cuda(), saved, E.Geom(2, 0), None)
  torch.cuda.synchronize()
  k = torch.tensor(_tree(P)["root_block/conv_root/kernel"], requires_grad=True)
  O.BF16[0] = True
  try:
    want = O.max_pool(O.std_conv(O.rnd(image.double()), k, 2, 3))
  finally:
    O.BF16[0] = False
  (gk,) = torch.autograd.grad(want, (k,), dy.double())
  assert torch.equal(out.double().cpu(), want.detach())
  assert _rel(P.tree("g")["root_block/conv_root/kernel"].cpu().numpy(), gk.numpy()) < 2e-2
