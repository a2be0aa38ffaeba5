"""GPU: the BERT text tower (models/proj/flaxformer/bert.py) and SigLiT with it.

The tower's forward against the bf16-emulating float64 oracle (tests/bert_oracle.py, 2^-7 of the output
scale) and every parameter gradient against the float64 oracle (6e-2 of the tensor's max), at a tiny size
and at BERT-Base width, on zero-padded captions.  The pad token's embedding row reaches only the padded
positions: changing it changes no output bit and no other gradient, and its own gradient is exactly 0.
A SigLiT step with the BERT text tower and a frozen ViT image tower against the oracle's loss and
gradients, with the image tower forward-only; and the same step on 2 ranks (skips on one GPU)."""
import os
import sys

import numpy as np
import pytest
import torch

import bert_oracle as BO
import common
from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = dict(width=128, depth=2, num_heads=2, mlp_dim=256, vocab_size=97)
BASE_WIDTH = dict(width=768, depth=2, num_heads=12, mlp_dim=3072, vocab_size=30_522)
EMB = "BertEncoder_0/embedder/embedders_token_ids/embedding"


def _tower(cfg, n, length, classes=64, seed=0):
  from big_vision_b200.models.proj.flaxformer import bert
  model = bert.Model(cfg, num_classes=classes, head_zeroinit=False)
  P = model.init(seed, (n, length), device="cuda")
  # perturb the unit LayerNorm scales and zero biases so that a wrong gradient cannot hide
  rng = np.random.default_rng(seed + 1)
  P.flat.add_(torch.from_numpy(0.02 * rng.standard_normal(P.total).astype(np.float32)).cuda())
  P.sync_half()
  text = torch.from_numpy(BO.padded_text(n, length, cfg["vocab_size"], seed=seed + 2)).cuda()
  return model, P, text


def _fwd_bwd(model, P, text, cot):
  P.zero_grad()
  out, saved = model.fwd(P, text)
  model.bwd(P, cot, saved)
  torch.cuda.synchronize()
  return out.clone(), {k: v.clone() for k, v in P.tree("g").items()}


def _oracle(P, text, cfg, classes, cot, mm):
  leaves = {k: v.detach().double().clone().requires_grad_(True) for k, v in P.tree("f").items()}
  y = BO.bert_forward(leaves, text.long(), dict(depth=cfg["depth"], num_heads=cfg["num_heads"],
                                                num_classes=classes), mm=mm)
  (y * cot.double()).sum().backward()
  return y.detach(), {k: v.grad for k, v in leaves.items()}


@pytest.mark.parametrize("cfg,n", [(TINY, 8), (BASE_WIDTH, 8)], ids=["tiny", "base_width"])
def test_tower_forward_and_backward_match_the_oracle(cfg, n):
  classes = 64
  model, P, text = _tower(cfg, n, 16, classes)
  assert (text == 0).any()
  cot = torch.from_numpy(np.random.default_rng(9).standard_normal((n, classes)).astype(np.float32)).cuda()
  out, grads = _fwd_bwd(model, P, text, cot)
  y16, _ = _oracle(P, text, cfg, classes, cot, "bfloat16")
  y64, g64 = _oracle(P, text, cfg, classes, cot, "float32")
  assert (out.double() - y16).abs().max().item() <= 2.0 ** -7 * y16.abs().max().item()
  assert (out.double() - y64).abs().max().item() <= 3e-2 * y64.abs().max().item()
  for name, g in grads.items():
    ref = g64[name]
    scale = ref.abs().max().item()
    if name.endswith("key/bias"):         # 0 in exact arithmetic: held to the value bias's scale
      scale = g64[name.replace("key/bias", "value/bias")].abs().max().item()
    assert (g.double() - ref).abs().max().item() <= 6e-2 * scale + 1e-30, name


def test_the_pad_row_reaches_only_padded_positions():
  """Row 0 of the token table (the pad token) changes no output bit, and its gradient is exactly 0.  The
  other gradients include sums by cross-CTA atomics (LayerNorm dγ/dβ, bias column sums, the embedding
  scatter, split-K weight gradients), whose last bits depend on the arrival order from run to run; they
  are held to 1e-5 of their scale, the spread of two runs without the change."""
  model, P, text = _tower(TINY, 8, 16)
  cot = torch.from_numpy(np.random.default_rng(3).standard_normal((8, 64)).astype(np.float32)).cuda()
  out1, g1 = _fwd_bwd(model, P, text, cot)
  out2, g2 = _fwd_bwd(model, P, text, cot)
  P.f(EMB)[0].normal_(generator=torch.Generator(device="cuda").manual_seed(0)).mul_(3.0)
  P.sync_half()
  out3, g3 = _fwd_bwd(model, P, text, cot)
  assert torch.equal(out1, out3) and torch.equal(out1, out2)
  assert not g3[EMB][0].any() and not g1[EMB][0].any()
  for name in g1:
    scale = g1[name].abs().max().item()
    assert (g2[name] - g1[name]).abs().max().item() <= 1e-5 * scale, name
    assert (g3[name] - g1[name]).abs().max().item() <= 1e-5 * scale, name


def test_apply_is_the_training_forward_and_train_is_refused():
  model, P, text = _tower(TINY, 4, 16)
  out, _ = model.fwd(P, text)
  x, aux = model.apply({"params": P}, text)
  assert torch.equal(out, x) and torch.equal(aux["logits"], x)
  with pytest.raises(NotImplementedError, match="dropout"):
    model.apply({"params": P}, text, train=True)


# ---- SigLiT with the BERT text tower --------------------------------------------------------------
SIGLIT = dict(image=dict(width=64, depth=2, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type="tok",
                         head_zeroinit=False),
              text=dict(config=TINY), text_model="proj.flaxformer.bert", out_dim=(None, 64),
              temperature_init=10.0, bias_init=-2.71)
LIT = [("img/.*", None), (".*", dict(decay_type="cosine"))]


def _siglit_model(n=8):
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.models.proj.image_text import two_towers
  model = two_towers.Model(**SIGLIT)
  P = model.init(0, (n, 64, 64, 3), (n, 16), device="cuda")
  rng = np.random.default_rng(1)
  P.flat.add_(torch.from_numpy(0.02 * rng.standard_normal(P.total).astype(np.float32)).cuda())
  P.sync_half()
  image, _ = common.synthetic_batch((n, 64, 64, 3), (n, 16), 97)
  text = BO.padded_text(n, 16, TINY["vocab_size"], seed=2)
  tx, _ = bv_optax.make(dict(lr=1e-3, schedule=LIT, optax=dict(b2=0.95)), P, sched_kw=dict(total_steps=100))
  return model, P, torch.from_numpy(image).cuda(), torch.from_numpy(text).cuda(), tx.frozen()


def test_siglit_bert_step_matches_the_oracle():
  from big_vision_b200.trainers.proj.image_text import siglip
  model, P, image, text, frozen = _siglit_model()
  zimg, ztxt, saved = model.fwd(P, image, text, frozen=frozen)
  assert saved["img"] is None and saved["img_norm"] is None      # the image tower kept nothing
  loss, out = siglip.loss_and_grads(model, P, image, text, frozen=frozen)
  assert out["dzimg"] is None
  g = P.grad.cpu().numpy()
  tr = np.zeros(P.total, dtype=bool)
  for lo, hi in P.trained_ranges(frozen):
    tr[lo:hi] = True
  assert not g[~tr].any()

  # the oracle on the host (its loss builds host tensors)
  leaves = {k: v.detach().double().cpu().requires_grad_(True) for k, v in P.tree("f").items()}
  img_cfg = dict(depth=2, num_heads=1, pool_type="tok", num_classes=None)
  zi = O.l2_normalize(O.vit_forward(O.sub(leaves, "img/"), image.double().cpu(), img_cfg))
  zt = O.l2_normalize(BO.bert_forward(O.sub(leaves, "txt/"), text.long().cpu(),
                                      dict(depth=2, num_heads=2, num_classes=64)))
  ref = O.siglip_loss(zi, zt, torch.exp(leaves["t"]), leaves["b"])
  ref.backward()
  assert abs(float(loss) - ref.item()) <= 5e-3 * max(abs(ref.item()), 1.0)
  grads = P.tree("g")
  for name, leaf in leaves.items():
    if name.startswith("img/"):
      continue
    want = leaf.grad
    scale = want.abs().max().item()
    if name.endswith("key/bias"):
      scale = leaves[name.replace("key/bias", "value/bias")].grad.abs().max().item()
    assert (grads[name].double().cpu() - want).abs().max().item() <= 6e-2 * scale + 1e-30, name


def _worker(rank, world, port, ret):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  import test_bert_gpu as T
  from big_vision_b200.trainers.proj.image_text import siglip
  model, P, image, text, frozen = T._siglit_model()
  n = image.shape[0] // world
  loss, _ = siglip.loss_and_grads(model, P, image[rank * n:(rank + 1) * n], text[rank * n:(rank + 1) * n],
                                  frozen=frozen)
  torch.cuda.synchronize()
  if rank == 0:
    ret["loss"] = float(loss)
    ret["grad"] = P.grad.cpu().numpy()
  dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_siglit_bert_step_equals_single_rank_global_batch():
  import torch.multiprocessing as mp
  from big_vision_b200.trainers.proj.image_text import siglip
  ctx = mp.get_context("spawn")
  ret = ctx.Manager().dict()
  port = 29690 + os.getpid() % 40
  procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  model, P, image, text, frozen = _siglit_model()
  loss, _ = siglip.loss_and_grads(model, P, image, text, frozen=frozen)
  g1, g2 = P.grad.cpu().numpy(), ret["grad"]
  assert ret["loss"] == pytest.approx(float(loss), rel=1e-4)
  assert np.abs(g1 - g2).max() <= 2e-2 * np.abs(g1).max()
  assert np.linalg.norm(g1 - g2) <= 1e-2 * np.linalg.norm(g1)
