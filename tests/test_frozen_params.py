"""CPU: where the backward of a partly frozen model stops, and what the gradient all-reduce covers.

The parameters whose schedule is None (optax.Chain.frozen()) get no gradient.  Each model is a list of
backward stages, bottom-up; the backward runs down to the lowest stage holding a trained parameter
(the cut) and everything below runs forward-only.  Shapes only: nothing here runs a kernel."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import common

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCHED = dict(decay_type="cosine")
LIT = [("img/.*", None), (".*", SCHED)]


def _tx(P, schedule):
  from big_vision_b200 import optax as bv_optax
  tx, _ = bv_optax.make(dict(lr=1e-3, schedule=schedule), P, sched_kw=dict(total_steps=10))
  return tx


def _vit(pool="map", scan=False, rep=False, classes=10):
  from big_vision_b200 import engine as E
  from big_vision_b200.models import vit
  model = vit.Model(classes, width=64, depth=3, mlp_dim=128, num_heads=1, patch_size=(16, 16),
                    pool_type=pool, scan=scan, rep_size=rep)
  specs, aliases = model.specs((32, 32), 3)
  return model, E.FlatParams(specs, aliases, "cpu")


def _mixer():
  from big_vision_b200 import engine as E
  from big_vision_b200.models import mlp_mixer
  model = mlp_mixer.Model(10, patch_size=(16, 16), num_blocks=3, hidden_dim=64, tokens_mlp_dim=32,
                          channels_mlp_dim=128)
  specs, aliases = model.specs((32, 48), 3)
  return model, E.FlatParams(specs, aliases, "cpu")


def _two_towers(scan=False):
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.image_text import two_towers
  kw = dict(common.TINY, image=dict(common.TINY["image"], scan=scan), text=dict(common.TINY["text"], scan=scan))
  model = two_towers.Model(**kw)
  specs, aliases = model.specs(common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE)
  return model, E.FlatParams(specs, aliases, "cpu")


@pytest.mark.parametrize("scan", [False, True])
def test_lit_schedule_freezes_the_whole_image_tower(scan):
  model, P = _two_towers(scan)
  frozen = _tx(P, LIT).frozen()
  assert frozen == {k for k in P.offsets if k.startswith("img/")}
  assert model.img.cut(P, frozen) == len(model.img.stages())
  assert model.txt.cut(P, frozen) == 0
  assert model.tower_frozen(P, frozen) == (True, False)


@pytest.mark.parametrize("pool", ["map", "tok", "gap"])
def test_linear_probe_cuts_at_the_head(pool):
  model, P = _vit(pool)
  frozen = _tx(P, [("head/.*", SCHED), (".*", None)]).frozen()
  stages = model.stages()
  assert model.cut(P, frozen) == len(stages) - 1
  assert stages[-1] == ("head/",)


def test_head_and_map_head_cut_at_the_map_head():
  model, P = _vit("map")
  frozen = _tx(P, [("head/.*", SCHED), ("MAPHead_0/.*", SCHED), (".*", None)]).frozen()
  assert model.stages()[model.cut(P, frozen)] == ("MAPHead_0/",)


def test_frozen_middle_block_does_not_truncate():
  model, P = _vit("gap")
  frozen = _tx(P, [("Transformer/encoderblock_1/.*", None), (".*", SCHED)]).frozen()
  assert frozen and all(k.startswith("Transformer/encoderblock_1/") for k in frozen)
  assert model.cut(P, frozen) == 0


def test_blocks_are_stages_and_the_cut_falls_on_the_lowest_trained_block():
  model, P = _vit("gap")
  stages = model.stages()
  assert len(stages) == 1 + 3 + 1 + 1          # embedding, 3 blocks, encoder_norm, head
  frozen = _tx(P, [("embedding/.*|pos_embedding|Transformer/encoderblock_0/.*", None), (".*", SCHED)]).frozen()
  assert stages[model.cut(P, frozen)] == ("Transformer/encoderblock_1/",)


def test_mixer_stages_are_stem_blocks_pre_head_and_head():
  model, P = _mixer()
  assert model.stages() == [("stem/",), ("MixerBlock_0/",), ("MixerBlock_1/",), ("MixerBlock_2/",),
                            ("pre_head_layer_norm/",), ("head/",)]
  assert model.cut(P, _tx(P, [("head/.*", SCHED), (".*", None)]).frozen()) == 5
  frozen = _tx(P, [("stem/.*|MixerBlock_0/.*", None), (".*", SCHED)]).frozen()
  assert model.stages()[model.cut(P, frozen)] == ("MixerBlock_1/",)
  assert model.cut(P, _tx(P, [("MixerBlock_1/.*", None), (".*", SCHED)]).frozen()) == 0


def test_scan_stacked_encoder_is_one_stage():
  model, P = _vit("map", scan=True)
  stages = model.stages()
  assert len(stages) == 1 + 1 + 1 + 1 + 1      # embedding, the stacked encoder, encoder_norm, MAP head, head
  assert stages[1] == ("Transformer/encoderblock/",)
  # embedding frozen, encoder trained: the cut is the whole encoder
  frozen = _tx(P, [("embedding/.*|pos_embedding", None), (".*", SCHED)]).frozen()
  assert model.cut(P, frozen) == 1
  # encoder frozen as well: the cut moves above it
  frozen = _tx(P, [("embedding/.*|pos_embedding|Transformer/encoderblock/.*", None), (".*", SCHED)]).frozen()
  assert stages[model.cut(P, frozen)] == ("Transformer/encoder_norm/",)


def test_nothing_frozen_is_todays_path():
  from big_vision_b200.trainers.proj.image_text import siglip
  model, P = _two_towers()
  frozen = _tx(P, SCHED).frozen()
  assert frozen == frozenset()
  assert model.img.cut(P, frozen) == 0 and model.txt.cut(P, frozen) == 0
  assert siglip._frozen_plan(model, P, frozen) == (None, None, (False, False))
  vit_model, VP = _vit("tok", rep=True)
  assert vit_model.cut(VP, _tx(VP, SCHED).frozen()) == 0


def test_everything_frozen_cuts_above_the_top():
  model, P = _vit("map")
  assert model.cut(P, True) == len(model.stages())


def test_trained_ranges_cover_exactly_the_trained_storage():
  model, P = _two_towers()
  frozen = _tx(P, LIT).frozen()
  ranges = P.trained_ranges(frozen)
  mask = np.zeros(P.total, dtype=bool)
  for lo, hi in ranges:
    assert not mask[lo:hi].any()
    mask[lo:hi] = True
  assert all(a[1] < b[0] for a, b in zip(ranges, ranges[1:]))        # merged: no touching neighbours
  for name, (off, shape) in P.offsets.items():
    n = int(np.prod(shape))
    assert mask[off:off + n].all() == (name not in frozen)
    assert mask[off:off + n].any() == (name not in frozen)


def _reduce_worker(rank, world, port, ret, overlap):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  if overlap:
    os.environ["BV_GRAD_ALLREDUCE"] = "overlap"
  dist.init_process_group("gloo", rank=rank, world_size=world)
  import test_frozen_params as T
  from big_vision_b200.trainers.proj.image_text import siglip
  model, P = T._two_towers()
  frozen = T._tx(P, T.LIT).frozen()
  ranges = P.trained_ranges(frozen)
  launched = []
  orig = dist.all_reduce

  def spy(t, *a, **kw):
    lo = (t.data_ptr() - P.grad.data_ptr()) // P.grad.element_size()
    launched.append((lo, lo + t.numel()))
    return orig(t, *a, **kw)

  siglip.dist.all_reduce = spy
  rng = np.random.default_rng(7 + rank)
  full = torch.from_numpy(rng.standard_normal(P.total).astype(np.float32))

  def backward():     # a frozen stage writes nothing: trained slots only, in reverse spec order
    for spec in reversed(P.specs):
      if spec.name in frozen:
        continue
      off, shape = P.offsets[spec.name]
      n = int(np.prod(shape))
      P.grad[off:off + n] = full[off:off + n]
      if spec.name.endswith("LayerNorm_0/scale") and "encoderblock" in spec.name and P.on_ready:
        P.on_ready(spec.name)

  P.on_ready = None
  siglip.all_reduce_grads(P, siglip.Dist(), backward, ranges=ranges)
  siglip.dist.all_reduce = orig
  expect = full.clone()
  dist.all_reduce(expect)
  ok_trained, ok_frozen = True, True
  for name, (off, shape) in P.offsets.items():
    n = int(np.prod(shape))
    if name in frozen:
      ok_frozen &= bool((P.grad[off:off + n] == 0).all())
    else:
      ok_trained &= bool(torch.equal(P.grad[off:off + n], expect[off:off + n]))
  spans = sorted(launched)
  cover = np.zeros(P.total, dtype=np.int32)
  for lo, hi in spans:
    cover[lo:hi] += 1
  want = np.zeros(P.total, dtype=np.int32)
  for lo, hi in ranges:
    want[lo:hi] = 1
  ret[rank] = {"trained": ok_trained, "frozen_zero": ok_frozen, "exact_cover": bool((cover == want).all()),
               "n": len(spans)}
  dist.destroy_process_group()


@pytest.mark.parametrize("overlap", [False, True])
def test_all_reduce_reduces_only_the_trained_ranges(overlap):
  """gloo, world size 2: under the LiT schedule the all-reduce (one-shot and bucketed) launches over
  the trained ranges exactly once each, reduces them, and leaves the frozen ranges zero."""
  world = 2
  port = 29900 + os.getpid() % 50 + (50 if overlap else 0)
  ctx = mp.get_context("spawn")
  ret = ctx.Manager().dict()
  procs = [ctx.Process(target=_reduce_worker, args=(r, world, port, ret, overlap)) for r in range(world)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(120)
    assert p.exitcode == 0
  for r in range(world):
    res = dict(ret[r])
    assert res["trained"] and res["frozen_zero"] and res["exact_cover"], res
