"""GPU: BERT dropout.  The attention kernels with BV_ATTN_DROPOUT (head_dim 64 | BV_ATTN_KEY_MASK |
BV_ATTN_DROPOUT) against float64 with the numpy restatement of the mask (tests/bert_dropout_oracle.py): O,
lse, dQ, dK, dV and the bias column sums at N = 16, 64, 128 and 512, rates 0.1 and 0.5, suffix and random key
masks and fully masked rows.  The kernel's keep mask read out exactly through one-hot values, rate 0 giving
the bits of the masked call, two runs giving the same bits, and a batch slice called at its global rows giving
that slice of the whole batch.  The BERT tower with both rates at 0.1 against the float64 oracle with the
same masks at a tiny size and at BERT-Base width, different steps and seeds giving different masks, the pad
row's gradient staying exactly 0, and a SigLiT-BERT step with dropout against the oracle (and on 2 ranks,
which skips on one GPU)."""
import os
import sys

import numpy as np
import pytest
import torch

import bert_dropout_oracle as BD
import bert_oracle as BO
import common
import test_attention_mask_gpu as AM
from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, DH = AM.H, AM.DH


def _key(rate, row0=0, seed=3, step=5, site=9):
  from big_vision_b200 import lib as L
  return L.DropoutKey(seed=seed, step=step, site=site, row0=row0, rate=rate)


def run(q, k, v, do, mask, key, colsums=False):
  from big_vision_b200 import ops
  o, lse = ops.attention_fwd(q, k, v, H, key_mask=mask, dropout=key)
  cs = {n: torch.zeros(H * DH, dtype=torch.float32, device="cuda") for n in ("dq_colsum", "dk_colsum", "dv_colsum")}
  dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, H, key_mask=mask, dropout=key, **(cs if colsums else {}))
  torch.cuda.synchronize()
  return (o, lse, dq, dk, dv) + ((cs,) if colsums else ())


def reference(q, k, v, do, mask, key):
  """float64 O, lse and dQ, dK, dV with the numpy keep mask of `key`."""
  B, N, d = q.shape
  split = lambda t: t.double().cpu().reshape(B, -1, H, DH).transpose(1, 2).requires_grad_(True)
  q6, k6, v6 = split(q), split(k), split(v)
  keep = BD.scaled(BD.attn_keep_of(key, B, H, N, N), key.rate)
  o, lse = BD.attention(q6, k6, v6, mask.bool().cpu(), keep)
  o = o.transpose(1, 2).reshape(B, N, d)
  o.backward(do.double().cpu())
  merge = lambda t: t.grad.transpose(1, 2).reshape(B, -1, d)
  return o.detach(), lse.detach(), merge(q6), merge(k6), merge(v6)


@pytest.mark.parametrize("N", [16, 64, 128, 512])
@pytest.mark.parametrize("rate", [0.1, 0.5])
@pytest.mark.parametrize("kind", ["suffix", "random", "empty"])
def test_dropout_attention_matches_fp64(N, rate, kind):
  B = 2 if N == 512 else 4
  q, k, v, do = AM.make_inputs(B, N, seed=N + 100)
  mask = AM.make_mask(B, N, kind, seed=N + 101)
  key = _key(rate, row0=B * H * N)           # the rows of the second rank of a batch of 2 B
  o, lse, dq, dk, dv, cs = run(q, k, v, do, mask, key, colsums=True)
  ro, rlse, rdq, rdk, rdv = reference(q, k, v, do, mask, key)
  cpu = lambda t: t.cpu()
  AM._close(cpu(o), ro, "o", rel=2.0 ** -6)   # pylint: disable=protected-access
  assert (lse.double().cpu() - rlse).abs().max().item() <= 1e-4 * max(rlse.abs().max().item(), 1.0)
  for name, got, ref in (("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
    AM._close(cpu(got), ref, name, rel=2.0 ** -6)   # pylint: disable=protected-access
    colsum = ref.sum((0, 1))
    err = (cs[name + "_colsum"].double().cpu() - colsum).abs().max().item()
    assert err <= 2.0 ** -6 * ref.abs().sum((0, 1)).max().item() + 1e-30, name
  masked = ~mask.bool()
  assert not dk[masked].any() and not dv[masked].any(), "a masked key has a nonzero gradient"
  if kind == "empty":
    assert not o[1].any() and not lse[1].any() and not dq[1].any()


@pytest.mark.parametrize("rate", [0.1, 0.5])
def test_one_hot_values_read_out_the_keep_mask_bit_for_bit(rate):
  """Q = K = 0 and V[k] = e_(k % 64), with the key mask restricted to one 64-key window: each O[b, q, h] is
  the window's row of the keep mask times 1 / (64 (1 - rate)).  Every window of N = 512 equals numpy's mask."""
  B, N = 2, 512
  key = _key(rate, row0=5 * H * N, seed=21, step=8, site=41)
  want = BD.attn_keep_of(key, B, H, N, N)
  eye = torch.eye(DH, dtype=torch.bfloat16, device="cuda")
  q = torch.zeros((B, N, H * DH), dtype=torch.bfloat16, device="cuda")
  v = eye.repeat(N // DH, H).expand(B, N, H * DH).contiguous()
  from big_vision_b200 import ops
  for w in range(N // DH):
    mask = torch.zeros((B, N), dtype=torch.uint8, device="cuda")
    mask[:, DH * w:DH * (w + 1)] = 1
    o, _ = ops.attention_fwd(q, q, v, H, key_mask=mask, dropout=key)
    got = (o.view(B, N, H, DH).permute(0, 2, 1, 3) != 0).cpu().numpy()
    assert np.array_equal(got, want[..., DH * w:DH * (w + 1)]), w
    assert torch.unique(o).numel() == 2           # 0 and one kept value


def test_rate_zero_gives_the_bits_of_the_masked_call():
  q, k, v, do = AM.make_inputs(3, 197, seed=31)
  mask = AM.make_mask(3, 197, "random", seed=32)
  for a, b in zip(run(q, k, v, do, mask, _key(0.0)), run(q, k, v, do, mask, None)):
    assert torch.equal(a, b)


def test_two_runs_give_the_same_bits():
  q, k, v, do = AM.make_inputs(4, 128, seed=41)
  mask = AM.make_mask(4, 128, "suffix", seed=42)
  key = _key(0.1)
  for a, b in zip(run(q, k, v, do, mask, key), run(q, k, v, do, mask, key)):
    assert torch.equal(a, b)
  # another step draws another mask
  assert not torch.equal(run(q, k, v, do, mask, _key(0.1, step=6))[0], run(q, k, v, do, mask, key)[0])


def test_a_batch_slice_at_its_global_rows_gives_that_slice_of_the_whole_batch():
  B, N, b0 = 4, 100, 2
  q, k, v, do = AM.make_inputs(B, N, seed=51)
  mask = AM.make_mask(B, N, "random", seed=52)
  whole = run(q, k, v, do, mask, _key(0.1))
  part = run(*(t[b0:].contiguous() for t in (q, k, v, do)), mask[b0:].contiguous(), _key(0.1, row0=b0 * H * N))
  for a, b in zip(whole, part):
    assert torch.equal(a[b0:], b)


# ---- the BERT tower ------------------------------------------------------------------------------------------
TINY = dict(width=128, depth=2, num_heads=2, mlp_dim=256, vocab_size=97, dropout_rate=0.1,
            attention_dropout_rate=0.1)
BASE_WIDTH = dict(width=768, depth=2, num_heads=12, mlp_dim=3072, vocab_size=30_522, dropout_rate=0.1,
                  attention_dropout_rate=0.1)
EMB = "BertEncoder_0/embedder/embedders_token_ids/embedding"


def _tower(cfg, n, length, classes=64, seed=0):
  from big_vision_b200.models.proj.flaxformer import bert
  model = bert.Model(cfg, num_classes=classes, head_zeroinit=False)
  P = model.init(seed, (n, length), device="cuda")
  rng = np.random.default_rng(seed + 1)
  P.flat.add_(torch.from_numpy(0.02 * rng.standard_normal(P.total).astype(np.float32)).cuda())
  P.sync_half()
  text = torch.from_numpy(BO.padded_text(n, length, cfg["vocab_size"], seed=seed + 2)).cuda()
  return model, P, text


def _fwd_bwd(model, P, text, cot, key):
  P.zero_grad()
  out, saved = model.fwd(P, text, dropout=key)
  model.bwd(P, cot, saved)
  torch.cuda.synchronize()
  return out.clone(), {k: v.clone() for k, v in P.tree("g").items()}


def _oracle(P, text, cfg, classes, cot, key, mm):
  leaves = {k: v.detach().double().cpu().clone().requires_grad_(True) for k, v in P.tree("f").items()}
  masks = BD.PhiloxMasks(cfg["dropout_rate"], cfg["attention_dropout_rate"], key.seed, key.step, key.sample0,
                         key.tower)
  y = BD.bert_forward(leaves, text.long().cpu(), dict(depth=cfg["depth"], num_heads=cfg["num_heads"],
                                                      num_classes=classes), masks, mm=mm)
  (y * cot.double().cpu()).sum().backward()
  return y.detach(), {k: v.grad for k, v in leaves.items()}


@pytest.mark.parametrize("cfg,n", [(TINY, 8), (BASE_WIDTH, 8)], ids=["tiny", "base_width"])
def test_tower_with_dropout_matches_the_oracle_with_the_same_masks(cfg, n):
  """The forward against the bf16-emulating oracle (2^-7 of the output scale) and float64 (3e-2), every
  gradient against float64 (6e-2 of the tensor's max), the oracle drawing the masks from numpy's Philox: the
  backward regenerates the forward's masks."""
  from big_vision_b200 import engine as E
  classes = 64
  model, P, text = _tower(cfg, n, 16, classes)
  assert (text == 0).any()
  key = E.DropoutKey(seed=7, step=11, sample0=n)
  cot = torch.from_numpy(np.random.default_rng(9).standard_normal((n, classes)).astype(np.float32)).cuda()
  out, grads = _fwd_bwd(model, P, text, cot, key)
  y16, _ = _oracle(P, text, cfg, classes, cot, key, "bfloat16")
  y64, g64 = _oracle(P, text, cfg, classes, cot, key, "float32")
  out = out.double().cpu()
  assert (out - y16).abs().max().item() <= 2.0 ** -7 * y16.abs().max().item()
  assert (out - y64).abs().max().item() <= 3e-2 * y64.abs().max().item()
  for name, g in grads.items():
    ref = g64[name]
    scale = ref.abs().max().item()
    if name.endswith("key/bias"):
      scale = g64[name.replace("key/bias", "value/bias")].abs().max().item()
    assert (g.double().cpu() - ref).abs().max().item() <= 6e-2 * scale + 1e-30, name
  assert not grads[EMB][0].any()           # the pad row reaches only padded positions


def test_steps_and_seeds_draw_different_masks_and_no_key_is_evaluation():
  from big_vision_b200 import engine as E
  model, P, text = _tower(TINY, 8, 16)
  outs = [model.fwd(P, text, dropout=k)[0].clone() for k in (E.DropoutKey(1, 2), E.DropoutKey(1, 3),
                                                              E.DropoutKey(2, 2), E.DropoutKey(1, 2))]
  assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], outs[2])
  assert torch.equal(outs[0], outs[3])
  x, _ = model.apply({"params": P}, text)
  assert torch.equal(x, model.fwd(P, text)[0]) and not torch.equal(x, outs[0])


# ---- SigLiT with dropout in the BERT tower -----------------------------------------------------------------
def _siglit_model(n=8):
  import test_bert_gpu as TB
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.models.proj.image_text import two_towers
  model = two_towers.Model(**dict(TB.SIGLIT, text=dict(config=TINY)))
  P = model.init(0, (n, 64, 64, 3), (n, 16), device="cuda")
  rng = np.random.default_rng(1)
  P.flat.add_(torch.from_numpy(0.02 * rng.standard_normal(P.total).astype(np.float32)).cuda())
  P.sync_half()
  image, _ = common.synthetic_batch((n, 64, 64, 3), (n, 16), 97)
  text = BO.padded_text(n, 16, TINY["vocab_size"], seed=2)
  tx, _ = bv_optax.make(dict(lr=1e-3, schedule=TB.LIT, optax=dict(b2=0.95)), P, sched_kw=dict(total_steps=100))
  return model, P, torch.from_numpy(image).cuda(), torch.from_numpy(text).cuda(), tx.frozen()


def test_siglit_bert_step_with_dropout_matches_the_oracle():
  from big_vision_b200 import engine as E
  from big_vision_b200.trainers.proj.image_text import siglip
  model, P, image, text, frozen = _siglit_model()
  key = E.DropoutKey(seed=4, step=3, sample0=0)
  loss, _ = siglip.loss_and_grads(model, P, image, text, frozen=frozen, dropout=key)
  leaves = {k: v.detach().double().cpu().requires_grad_(True) for k, v in P.tree("f").items()}
  img_cfg = dict(depth=2, num_heads=1, pool_type="tok", num_classes=None)
  zi = O.l2_normalize(O.vit_forward(O.sub(leaves, "img/"), image.double().cpu(), img_cfg))
  masks = BD.PhiloxMasks(0.1, 0.1, key.seed, key.step, 0, tower=1)
  zt = O.l2_normalize(BD.bert_forward(O.sub(leaves, "txt/"), text.long().cpu(),
                                      dict(depth=2, num_heads=2, num_classes=64), masks))
  ref = O.siglip_loss(zi, zt, torch.exp(leaves["t"]), leaves["b"])
  ref.backward()
  assert abs(float(loss) - ref.item()) <= 5e-3 * max(abs(ref.item()), 1.0)
  # without dropout the loss is another one: the masks are applied
  loss0, _ = siglip.loss_and_grads(model, P, image, text, frozen=frozen)
  assert float(loss0) != float(loss)
  siglip.loss_and_grads(model, P, image, text, frozen=frozen, dropout=key)
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
  import test_bert_dropout_gpu as T
  from big_vision_b200 import engine as E
  from big_vision_b200.trainers.proj.image_text import siglip
  model, P, image, text, frozen = T._siglit_model()   # pylint: disable=protected-access
  n = image.shape[0] // world
  loss, _ = siglip.loss_and_grads(model, P, image[rank * n:(rank + 1) * n], text[rank * n:(rank + 1) * n],
                                  frozen=frozen, dropout=E.DropoutKey(4, 3, rank * n))
  torch.cuda.synchronize()
  if rank == 0:
    ret["loss"] = float(loss)
    ret["grad"] = P.grad.cpu().numpy()
  dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_siglit_bert_step_with_dropout_equals_single_rank_global_batch():
  """Each rank draws the masks of its slice of the global batch, so 2 ranks compute the 1-rank step."""
  import torch.multiprocessing as mp
  from big_vision_b200 import engine as E
  from big_vision_b200.trainers.proj.image_text import siglip
  ctx = mp.get_context("spawn")
  ret = ctx.Manager().dict()
  port = 29730 + os.getpid() % 40
  procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  model, P, image, text, frozen = _siglit_model()
  loss, _ = siglip.loss_and_grads(model, P, image, text, frozen=frozen, dropout=E.DropoutKey(4, 3, 0))
  g1, g2 = P.grad.cpu().numpy(), ret["grad"]
  assert ret["loss"] == pytest.approx(float(loss), rel=1e-4)
  assert np.abs(g1 - g2).max() <= 2e-2 * np.abs(g1).max()
  assert np.linalg.norm(g1 - g2) <= 1e-2 * np.linalg.norm(g1)
