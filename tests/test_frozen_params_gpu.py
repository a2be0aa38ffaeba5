"""GPU: frozen parameters cost only a forward pass.

A SigLiT step (image tower frozen) and a ViT or MLP-Mixer linear probe (head only) against the same
step run the full way: the forward is bit-identical, every trained gradient matches, every frozen
gradient is exactly zero, the frozen parameters do not move in 3 optimizer steps and the trained ones
follow the full path.  The SigLiT step's peak memory drops by the image tower's saved activations;
apply() is the forward-only path and returns the training forward's bits, and so does a forward-only
Mixer run under stochastic-depth masks.  The single-output bias + GELU epilogue (EPI_BIAS_GELU_ACT)
writes the dual-output epilogue's first output bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch

import common

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCHED = dict(decay_type="cosine")
LIT = [("img/.*", None), (".*", SCHED)]

B16 = dict(image=dict(variant="B/16", pool_type="map"), text=dict(variant="B", vocab_size=32_000),
           out_dim=(None, 768), temperature_init=10.0, bias_init=-10.0)
B16_IMAGE_SHAPE, B16_TEXT_SHAPE = (4, 224, 224, 3), (4, 64)


class _FullPath:
  """The same optimizer, but the trainer sees nothing frozen: every backward runs (today's path)."""

  def __init__(self, tx):
    self.tx = tx

  def frozen(self):
    return frozenset()

  def update(self, *a, **kw):
    return self.tx.update(*a, **kw)


def _tx(P, schedule, lr=1e-3):
  from big_vision_b200 import optax as bv_optax
  tx, _ = bv_optax.make(dict(lr=lr, schedule=schedule, optax=dict(b2=0.95)), P,
                        sched_kw=dict(total_steps=100))
  return tx


def _two_towers(cfg, image_shape, text_shape, scan):
  from big_vision_b200.models.proj.image_text import two_towers
  kw = dict(cfg, image=dict(cfg["image"], scan=scan), text=dict(cfg["text"], scan=scan))
  model = two_towers.Model(**kw)
  P = model.init(0, image_shape, text_shape, device="cuda")
  image, text = common.synthetic_batch(image_shape, text_shape, kw["text"]["vocab_size"])
  return model, P, torch.from_numpy(image).cuda(), torch.from_numpy(text).cuda()


def _check_grads(P, g_cut, g_full, frozen):
  """Trained gradients within the fp32-atomics tolerance of the 2-rank test; frozen ones exactly 0."""
  tr = np.zeros(P.total, dtype=bool)
  for lo, hi in P.trained_ranges(frozen):
    tr[lo:hi] = True
  assert not g_cut[~tr].any(), "a frozen gradient is not zero"
  a, b = g_cut[tr], g_full[tr]
  assert np.abs(a - b).max() <= 2e-2 * np.abs(b).max()
  assert np.linalg.norm(a - b) <= 1e-2 * np.linalg.norm(b)


def _check_steps(P0, P_cut, P_full, frozen, lr):
  for name, (off, shape) in P0.offsets.items():
    n = int(np.prod(shape))
    a, b, init = (x[off:off + n] for x in (P_cut, P_full, P0.flat.cpu().numpy()))
    if name in frozen:
      assert np.array_equal(a, init), name
    else:
      assert np.abs(a - b).max() <= 6 * lr, name        # Adam moves a parameter by <= lr per step
  tr = np.zeros(P0.total, dtype=bool)
  for lo, hi in P0.trained_ranges(frozen):
    tr[lo:hi] = True
  init = P0.flat.cpu().numpy()
  assert np.linalg.norm(P_cut[tr] - P_full[tr]) <= 5e-2 * np.linalg.norm(P_full[tr] - init[tr])


def _siglit(cfg, image_shape, text_shape, scan):
  from big_vision_b200.trainers.proj.image_text import siglip
  model, P, image, text = _two_towers(cfg, image_shape, text_shape, scan)
  frozen = _tx(P, LIT).frozen()
  loss_f, out_f = siglip.loss_and_grads(model, P, image, text)
  g_full = P.grad.cpu().numpy()
  loss_c, out_c = siglip.loss_and_grads(model, P, image, text, frozen=frozen)
  g_cut = P.grad.cpu().numpy()
  assert torch.equal(loss_c, loss_f)
  assert torch.equal(out_c["zimg"], out_f["zimg"]) and torch.equal(out_c["ztxt"], out_f["ztxt"])
  assert out_c["dzimg"] is None and out_f["dzimg"] is not None
  _check_grads(P, g_cut, g_full, frozen)
  # 3 optimizer steps through make_update_fn, SigLiT vs the full path with the same schedule
  lr = 1e-3
  P0 = model.init(0, image_shape, text_shape, device="cuda")
  finals = []
  for full in (False, True):
    Pk = model.init(0, image_shape, text_shape, device="cuda")
    tx = _tx(Pk, LIT, lr)
    update_fn = siglip.make_update_fn(model, _FullPath(tx) if full else tx, {})
    state = {"params": Pk, "opt": tx.init(Pk)}
    for _ in range(3):
      state, _ = update_fn(state, None, {"image": image, "labels": text})
    finals.append(Pk.flat.cpu().numpy())
  _check_steps(P0, finals[0], finals[1], frozen, lr)


@pytest.mark.parametrize("scan", [False, True])
def test_siglit_step_tiny(scan):
  _siglit(common.TINY, common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE, scan)


@pytest.mark.parametrize("scan", [False, True])
def test_siglit_step_b16_width(scan):
  _siglit(B16, B16_IMAGE_SHAPE, B16_TEXT_SHAPE, scan)


def _image_saved_bytes(cfg, image_shape):
  """Bytes the full step keeps for the image tower's encoder blocks, from the shapes: per token
  x, ln1, qkv (3), o, x1, ln2 and GELU's act and pre-activation in bf16; two LayerNorms' mean and rstd
  and the attention's per-head log-sum-exp in fp32."""
  from big_vision_b200.models import vit
  v = vit.decode_variant(cfg["image"]["variant"])
  d, m, h, depth = v["width"], v["mlp_dim"], v["num_heads"], v["depth"]
  n, H, W, _ = image_shape
  tokens = n * (H // v["patch_size"][0]) * (W // v["patch_size"][1])
  return depth * tokens * (2 * (8 * d + 2 * m) + 4 * 4 + 4 * h)


def test_siglit_peak_memory_drops_by_the_image_activations():
  from big_vision_b200.trainers.proj.image_text import siglip
  model, P, image, text = _two_towers(B16, B16_IMAGE_SHAPE, B16_TEXT_SHAPE, False)
  frozen = _tx(P, LIT).frozen()
  peaks = {}
  for name, fz in (("full", None), ("lit", frozen), ("full2", None), ("lit2", frozen)):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    siglip.loss_and_grads(model, P, image, text, frozen=fz)
    torch.cuda.synchronize()
    peaks[name] = torch.cuda.max_memory_allocated()
  saved = _image_saved_bytes(B16, B16_IMAGE_SHAPE)
  drop = min(peaks["full"], peaks["full2"]) - max(peaks["lit"], peaks["lit2"])
  assert drop >= 0.9 * saved, (peaks, saved)


def test_apply_is_the_forward_bit_for_bit():
  model, P, image, text = _two_towers(B16, B16_IMAGE_SHAPE, B16_TEXT_SHAPE, False)
  zimg, ztxt, _ = model.fwd(P, image, text)
  zi, zt, out = model.apply({"params": P}, image, text)
  assert torch.equal(zi, zimg) and torch.equal(zt, ztxt)
  assert torch.equal(out["t"], P.f("t").exp())


# ---- ViT and MLP-Mixer linear probes through train.make_update_fn ----------------------------
def _probe_model(kind):
  from big_vision_b200.models import mlp_mixer, vit
  if kind == "mixer":        # 12 tokens: the token-mixing storage is padded to 16
    model = mlp_mixer.Model(16, patch_size=(16, 16), num_blocks=2, hidden_dim=64, tokens_mlp_dim=32,
                            channels_mlp_dim=128)
  else:
    model = vit.Model(16, width=64, depth=2, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type=kind)
  shape = (4, 64, 48, 3)
  P = model.init(0, shape, device="cuda")
  rng = np.random.default_rng(1)
  tree = {k: (v if np.any(v) else (rng.standard_normal(v.shape) * 0.05).astype(np.float32))
          for k, v in P.numpy_tree("f").items()}      # a zero-init head would zero the other gradients
  P.load_tree(tree)
  image = torch.from_numpy(rng.uniform(-1, 1, size=shape).astype(np.float32)).cuda()
  labels = torch.from_numpy(np.eye(16, dtype=np.float32)[rng.integers(0, 16, size=4)]).cuda()
  return model, P, tree, shape, image, labels


@pytest.mark.parametrize("kind", ["map", "tok", "gap", "mixer"])
def test_linear_probe_step(kind):
  from big_vision_b200 import train
  model, P, tree, shape, image, labels = _probe_model(kind)
  schedule = [("head/.*", SCHED), (".*", None)]
  frozen = _tx(P, schedule).frozen()
  assert model.cut(P, frozen) == len(model.stages()) - 1
  loss_f, logits_f = train.loss_and_grads(model, P, image, labels)
  g_full = P.grad.cpu().numpy()
  loss_c, logits_c = train.loss_and_grads(model, P, image, labels, frozen=frozen)
  g_cut = P.grad.cpu().numpy()
  assert torch.equal(loss_c, loss_f) and torch.equal(logits_c, logits_f)
  _check_grads(P, g_cut, g_full, frozen)
  lr = 1e-3
  finals = []
  for full in (False, True):
    Pk = model.init(0, shape, device="cuda")
    Pk.load_tree(tree)
    tx = _tx(Pk, schedule, lr)
    update_fn = train.make_update_fn(model, _FullPath(tx) if full else tx, {"loss": "sigmoid_xent"})
    state = {"params": Pk, "opt": tx.init(Pk)}
    for _ in range(3):
      state, _ = update_fn(state, None, {"image": image, "labels": labels})
    finals.append(Pk.flat.cpu().numpy())
  P0 = model.init(0, shape, device="cuda")
  P0.load_tree(tree)
  _check_steps(P0, finals[0], finals[1], frozen, lr)
  x, _ = model.apply({"params": P}, image)
  assert torch.equal(x, logits_f)
  if kind == "mixer":        # the stochastic-depth masks reach the forward-only blocks as well
    masks = torch.tensor([[[1, 1, 1, 1], [1, 1, 1, 1]], [[1, 0, 1, 0], [0, 1, 1, 0]]], dtype=torch.float32).cuda()
    x_saved, _ = model.fwd(P, image, masks=masks)
    x_fwd, _ = model.fwd(P, image, masks=masks, frozen=True)
    assert torch.equal(x_fwd, x_saved) and not torch.equal(x_fwd, x)


# ---- the single-output GELU epilogue ------------------------------------------------------------
@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M", [1, 65, 300])
def test_single_output_gelu_matches_the_dual_output_one(block_n, M):
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  g = torch.Generator(device="cuda").manual_seed(M + block_n)
  K, N = 192, 1000
  x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
  w = (torch.randn(K, N, device="cuda", generator=g) * 0.1).bfloat16()
  bias = torch.randn(N, device="cuda", generator=g)
  ref, _ = ops.gemm(x, w, b_mn=True, bias=bias, epilogue=L.EPI_BIAS_GELU, block_n=block_n)
  got = ops.gemm(x, w, b_mn=True, bias=bias, epilogue=L.EPI_BIAS_GELU_ACT, block_n=block_n)
  assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
  again = ops.gemm(x, w, b_mn=True, bias=bias, epilogue=L.EPI_BIAS_GELU_ACT, block_n=block_n)
  assert torch.equal(again.view(torch.int16), got.view(torch.int16))            # run to run
  # a strided output inside NaN sentinels: only the M x N window is written
  buf = torch.full((M + 2, N + 40), float("nan"), device="cuda", dtype=torch.bfloat16)
  out = buf[1:M + 1, 16:16 + N]
  ops.gemm(x, w, b_mn=True, bias=bias, out=out, epilogue=L.EPI_BIAS_GELU_ACT, block_n=block_n)
  assert torch.equal(out.view(torch.int16), ref.view(torch.int16))
  mask = torch.ones_like(buf, dtype=torch.bool)
  mask[1:M + 1, 16:16 + N] = False
  assert torch.isnan(buf[mask].float()).all()


def test_single_output_gelu_refuses_fp32_and_reduce():
  from big_vision_b200 import lib as L
  from big_vision_b200 import ops
  x = torch.zeros(8, 64, device="cuda", dtype=torch.bfloat16)
  w = torch.zeros(64, 64, device="cuda", dtype=torch.bfloat16)
  with pytest.raises(L.BvError):
    ops.gemm(x, w, b_mn=True, epilogue=L.EPI_BIAS_GELU_ACT, out_dtype=torch.float32)
  with pytest.raises(L.BvError):
    ops.gemm(x, w, b_mn=True, epilogue=L.EPI_BIAS_GELU_ACT, reduce_out=True)


# ---- 2 ranks --------------------------------------------------------------------------------------
def _worker(rank, world, port, ret):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  import common as c
  import test_frozen_params_gpu as T
  from big_vision_b200.trainers.proj.image_text import siglip
  model, P, image, text = T._two_towers(c.TINY, c.TINY_IMAGE_SHAPE, c.TINY_TEXT_SHAPE, False)
  frozen = T._tx(P, T.LIT).frozen()
  n = image.shape[0] // world
  loss, _ = siglip.loss_and_grads(model, P, image[rank * n:(rank + 1) * n], text[rank * n:(rank + 1) * n],
                                  frozen=frozen)
  torch.cuda.synchronize()
  if rank == 0:
    ret["loss"] = float(loss)
    ret["grad"] = P.grad.cpu().numpy()
  dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_siglit_step_equals_single_rank_global_batch():
  import torch.multiprocessing as mp
  from big_vision_b200.trainers.proj.image_text import siglip
  ctx = mp.get_context("spawn")
  ret = ctx.Manager().dict()
  port = 29650 + os.getpid() % 40
  procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  model, P, image, text = _two_towers(common.TINY, common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE, False)
  frozen = _tx(P, LIT).frozen()
  loss, _ = siglip.loss_and_grads(model, P, image, text, frozen=frozen)
  g1, g2 = P.grad.cpu().numpy(), ret["grad"]
  assert ret["loss"] == pytest.approx(float(loss), rel=1e-4)
  _check_grads(P, g2, g1, frozen)
