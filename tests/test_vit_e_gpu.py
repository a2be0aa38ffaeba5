"""GPU: ViT-e/14.  Attention at head dim 112 against fp64 (exact and per-element bound cases, the split
backward, bit-reproducibility, the raw C ABI, in place in a fused [B, N, 3 * 1792] QKV buffer); tiny e-shaped
models and the real-width e/14 at depth 2 against the fp64 oracle; and the training step on a flat buffer
past 2^31 elements: the clip-norm sum of squares and a BV-Adafactor + weight-decay step against float64 on
both sides of 2^31, and one update_fn step of the full 56-block e/14."""
import json
import math

import numpy as np
import pytest
import torch

import test_attention_bwd_split_gpu as bsplit
import test_attention_elementwise_gpu as eattn
import test_classifier_gpu as cls_t
import test_head_dim_gpu as hd
from oracle import bv_oracle as O

pytestmark = pytest.mark.gpu

DH = 112
C = 29_593
TWO31 = 2 ** 31


@pytest.fixture(scope="module")
def ops():
  from big_vision_b200 import lib, ops as _ops
  assert lib.load().bv_device_supported() == 1
  return _ops


@pytest.fixture(autouse=True)
def _release_memory():
  yield
  torch.cuda.synchronize()
  torch.cuda.empty_cache()


# ---- attention at head dim 112 -------------------------------------------------------------------
@pytest.mark.parametrize("Nk", [1, 64, 197, 256, 2048])
def test_zero_queries_average_every_key_once(ops, Nk):
  eattn.test_zero_queries_average_every_key_once(ops, DH, Nk)


@pytest.mark.parametrize("placement,Nk", [("first", 197), ("last", 197), ("last", 577), ("moving", 2048),
                                          ("moving", 577), ("moving", 65)])
def test_dominant_key_gives_its_value(ops, placement, Nk):
  eattn.test_dominant_key_gives_its_value(ops, DH, placement, Nk)


# (B, H, Nq, Nk): a single key, the MAP probe (Nq = 1) at the small and the e/14 geometry, Nq != Nk both
# ways, and the e/14 encoder (16 heads, 256 tokens)
BOUND_SHAPES = {"e_nk1": (2, 2, 65, 1), "e_probe": (2, 2, 1, 197), "e_map": (3, 16, 1, 256),
                "e_nk64": (2, 2, 577, 64), "e_nk2048": (1, 2, 63, 2048), "e_nq2048": (1, 1, 2048, 65),
                "e14": (2, 16, 256, 256)}


@pytest.mark.parametrize("sname,scale", [("e_nk1", None), ("e_probe", None), ("e_map", None), ("e_nk64", 1.0),
                                         ("e_nk2048", None), ("e_nq2048", 0.05), ("e14", None)])
def test_forward_and_backward_within_bound(ops, monkeypatch, sname, scale):
  """The per-element fp64 bounds of test_attention_elementwise_gpu at dh 112 on these shapes."""
  monkeypatch.setitem(eattn.SHAPES, sname, BOUND_SHAPES[sname])
  eattn.test_forward_and_backward_within_bound(ops, (DH, sname, scale))


@pytest.mark.parametrize("B,H,Nq,Nk", bsplit.SHAPES)
def test_backward_matches_fp64(ops, B, H, Nq, Nk):
  bsplit.test_backward_matches_fp64(ops, DH, B, H, Nq, Nk)


def test_backward_is_bitwise_reproducible(ops):
  bsplit.test_backward_is_bitwise_reproducible(ops, DH)


def test_raw_abi_without_dq_accum(ops):
  bsplit.test_raw_abi_without_dq_accum(ops, DH)


def test_in_place_in_the_fused_e14_qkv_buffer(ops):
  """q/k/v and dq/dk/dv as column views of [B, N + 5, 3 * 1792 + 8] buffers at the e/14 geometry (16 heads
  of 112).  The 8 columns past the views hold NaN in the input and a sentinel in the gradient buffer; rows
  past N and the sentinel columns must come back untouched."""
  B, H, N = 2, 16, 256
  d = H * DH
  qkv, g = hd._qkv(B, N + 5, d, 112)
  buf = torch.cat([qkv, torch.full((B, N + 5, 8), float("nan"), dtype=torch.bfloat16)], 2).cuda()
  do = hd._bf(torch.randn(B, N, d, generator=g))
  qr = qkv[:, :N, 0:d].double().requires_grad_(True)
  kr = qkv[:, :N, d:2 * d].double().requires_grad_(True)
  vr = qkv[:, :N, 2 * d:].double().requires_grad_(True)
  o_ref, lse_ref = hd._ref_attention(qr, kr, vr, H)
  o_ref.backward(do.double())
  q, k, v = buf[:, :N, 0:d], buf[:, :N, d:2 * d], buf[:, :N, 2 * d:3 * d]
  o, lse = ops.attention_fwd(q, k, v, H)
  sentinel = 1234.0
  dbuf = torch.full((B, N + 5, 3 * d + 8), sentinel, dtype=torch.bfloat16, device="cuda")
  ops.attention_bwd(do.cuda(), q, k, v, o, lse, H, dq=dbuf[:, :N, 0:d], dk=dbuf[:, :N, d:2 * d],
                    dv=dbuf[:, :N, 2 * d:3 * d])
  torch.cuda.synchronize()
  hd._close(o, o_ref, 2 ** -6)
  hd._close(lse, lse_ref, 1e-5)
  hd._close(dbuf[:, :N, 0:d], qr.grad, 2 ** -5)
  hd._close(dbuf[:, :N, d:2 * d], kr.grad, 2 ** -5)
  hd._close(dbuf[:, :N, 2 * d:3 * d], vr.grad, 2 ** -5)
  assert bool((dbuf[:, N:, :] == sentinel).all())
  assert bool((dbuf[:, :, 3 * d:] == sentinel).all())


# ---- tiny e-shaped models --------------------------------------------------------------------------
TINY_E = dict(width=2 * DH, depth=2, mlp_dim=4 * DH, num_heads=2, patch_size=(16, 16))
TINY_C = 37


def _unstacked(p, depth):
  """A scan-stacked tree as the per-block names the oracle reads (views, so gradients reach the stack)."""
  out = {}
  for k, v in p.items():
    if k.startswith("Transformer/encoderblock/"):
      for i in range(depth):
        out[k.replace("encoderblock/", f"encoderblock_{i}/")] = v[i]
    else:
      out[k] = v
  return out


def _tiny(pool, scan):
  from big_vision_b200.models import vit
  model = vit.Model(TINY_C, pool_type=pool, scan=scan, **TINY_E)
  cfg = dict(depth=2, num_heads=2, pool_type=pool, posemb="learn", rep_size=False, num_classes=TINY_C)
  return model, (lambda p, img, mm: O.vit_forward(_unstacked(p, 2) if scan else p, img, cfg, mm))


@pytest.mark.parametrize("scan", [False, True])
@pytest.mark.parametrize("pool", ["map", "gap"])
def test_tiny_e_shaped_vit_matches_oracle(pool, scan):
  model, fwd = _tiny(pool, scan)
  assert model.width // model.num_heads == DH
  cls_t._check(model, fwd, (4, 64, 48, 3), "sigmoid_xent", TINY_C)


@pytest.mark.parametrize("scan", [False, True])
@pytest.mark.parametrize("pool", ["map", "gap"])
def test_tiny_e_shaped_vit_adafactor_step(pool, scan):
  """One update_fn step with the e/14 config's optimizer (BV-Adafactor, clip 1, wd_mults): the gradient norm
  against the fp64 oracle, l2_params / l2_updates against the reference-shaped trees, every trained tensor
  moved."""
  from big_vision_b200 import optax as bv_optax, train
  model, fwd = _tiny(pool, scan)
  n, shape = 4, (4, 64, 48, 3)
  P = model.init(0, shape, device="cuda")
  tree = cls_t._randomize_zero_inits(P.numpy_tree("f"), 1)
  P.load_tree(tree)
  config = dict(optax_name="big_vision.scale_by_adafactor", grad_clip_norm=1.0, lr=1e-2, wd=1e-2 * 0.03,
                wd_mults=[(".*head/kernel", 100.0), (".*/kernel", 1.0)], loss="sigmoid_xent",
                schedule=dict(decay_type="cosine", warmup_steps=0))
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=100, batch_size=n, data_size=1000))
  state = {"params": P, "opt": tx.init(P)}
  rng = np.random.default_rng(3)
  image = rng.uniform(-1, 1, shape).astype(np.float32)
  labels = np.eye(TINY_C, dtype=np.float32)[rng.integers(0, TINY_C, n)]
  batch = {"image": torch.from_numpy(image).cuda(), "labels": torch.from_numpy(labels).cuda()}
  state, m = train.make_update_fn(model, tx, config)(state, None, batch)
  torch.cuda.synchronize()
  after = P.numpy_tree("f")
  l2 = lambda t: np.sqrt(sum(float(np.sum(np.asarray(v, np.float64) ** 2)) for v in t.values()))  # noqa: E731
  assert float(m["l2_params"]) == pytest.approx(l2(after), rel=1e-4)
  assert float(m["l2_updates"]) == pytest.approx(l2({k: after[k] - tree[k] for k in after}), rel=2e-3)
  p64 = O.to_f64_tree(tree, requires_grad=True)
  ref = O.sigmoid_xent(fwd(p64, torch.from_numpy(image), "float32"), torch.from_numpy(labels).double())
  ref.backward()
  assert float(m["training_loss"]) == pytest.approx(float(ref), rel=2e-2)
  assert float(m["l2_grads"]) == pytest.approx(
      np.sqrt(sum(float((v.grad ** 2).sum()) for v in p64.values() if v.grad is not None)), rel=3e-2)
  still = [k for k in after if np.array_equal(after[k], tree[k])]
  assert not still, still


# ---- real-width e/14 ----------------------------------------------------------------------------------
def test_vit_e14_real_width_with_jft_head_precision():
  """ViT-e/14 at its real width (1792, 16 heads of 112, mlp 15360, 256 tokens, MAP head, the 29,593-class
  head), depth cut to 2 so the fp64 oracle stays short; the bounds of the G/14 and So400m/14 tests."""
  from big_vision_b200 import train
  from big_vision_b200.models import vit
  n, depth = 4, 2
  shape = (n, 224, 224, 3)
  model = vit.Model(C, variant="e/14", depth=depth, pool_type="map")
  assert model.width == 1792 and model.mlp_dim == 15360 and model.num_heads == 16
  P = model.init(0, shape, device="cuda")
  rng = np.random.default_rng(1)
  tree = P.numpy_tree("f")
  for k, v in tree.items():                      # zero-initialised head: small values instead
    if not np.any(v):
      tree[k] = (rng.standard_normal(v.shape) * 0.02).astype(np.float32)
  P.load_tree(tree)
  image = rng.uniform(-1, 1, size=shape).astype(np.float32)
  labels = np.eye(C, dtype=np.float32)[rng.integers(0, C, size=n)]
  loss, logits = train.loss_and_grads(model, P, torch.from_numpy(image).cuda(), torch.from_numpy(labels).cuda(),
                                      "sigmoid_xent")
  cfg = dict(depth=depth, num_heads=16, pool_type="map", posemb="learn", rep_size=False, num_classes=C)
  with torch.no_grad():
    ref16 = O.vit_forward(O.to_f64_tree(tree), torch.from_numpy(image), cfg, "bfloat16").numpy()
  p64 = O.to_f64_tree(tree, requires_grad=True)
  ref64 = O.vit_forward(p64, torch.from_numpy(image), cfg, "float32")
  ref_loss = O.sigmoid_xent(ref64, torch.from_numpy(labels).double())
  ref_loss.backward()
  got = logits.double().cpu().numpy()
  res = {"logits_vs_bf16_oracle_max": hd._rel(got, ref16), "logits_vs_fp64_oracle_max": hd._rel(got, ref64.detach().numpy()),
         "loss_rel": abs(float(loss) - float(ref_loss)) / abs(float(ref_loss))}
  grads = P.numpy_tree("g")
  worst, l2s = ("", 0.0), []
  gmax = max(float(v.grad.abs().max()) for v in p64.values() if v.grad is not None)
  for k, g in grads.items():
    ref = p64[k].grad.numpy() if p64[k].grad is not None else np.zeros_like(g)
    e = float(np.abs(g - ref).max() / (np.abs(ref).max() + 1e-3 * gmax))
    l2s.append(hd._rel_l2(g, ref) if np.abs(ref).max() > 1e-3 * gmax else 0.0)
    if e > worst[1]:
      worst = (k, e)
  res.update(grad_worst_tensor=worst[0], grad_worst_rel_max=worst[1], grad_median_rel_l2=float(np.median(l2s)))
  print(json.dumps({f"vit_e14_depth{depth}_map_jft_n{n}": res}))
  assert res["logits_vs_bf16_oracle_max"] <= 1.5e-2, res
  assert res["logits_vs_fp64_oracle_max"] <= 3e-2 and res["loss_rel"] <= 2e-3, res
  assert res["grad_worst_rel_max"] <= 1.2e-1 and res["grad_median_rel_l2"] <= 3e-2, res


# ---- past 2^31 elements ---------------------------------------------------------------------------------
ROWS, COLS = 2 ** 15, 2 ** 16       # x/kernel: 2^31 elements at offset 0, its last one at 2^31 - 1
YN = 2 ** 12                        # y/kernel [4096, 4096] at offset 2^31, y/bias [4096] at the end


def _row_col_sumsq(x, gs, chunk=2048):
  """float64 row and column sums of (x * gs)^2 of a [ROWS, COLS] fp32 tensor, a few rows at a time."""
  rows = torch.empty(x.shape[0], dtype=torch.float64, device=x.device)
  cols = torch.zeros(x.shape[1], dtype=torch.float64, device=x.device)
  for r in range(0, x.shape[0], chunk):
    sq = (x[r:r + chunk].double() * gs) ** 2
    rows[r:r + chunk] = sq.sum(1)
    cols += sq.sum(0)
  return rows, cols


def _sumsq64(flat, chunk=2 ** 27):
  return sum(float((flat[i:i + chunk].double() ** 2).sum()) for i in range(0, flat.numel(), chunk))


def _bf16(x):
  return x.to(torch.bfloat16).double()


def test_flat_buffer_past_2_31_clip_norm_and_adafactor_step(ops):
  """A flat buffer of 2^31 + 2^24 + 4096 elements: x/kernel [32768, 65536] fills [0, 2^31), y/kernel
  [4096, 4096] starts at 2^31, y/bias ends the buffer.  Two BV-Adafactor steps with clip norm 1 and weight
  decay (x, y factored; y/bias a full second moment): the clip-norm sum of squares (one launch over a range of
  2^31 + 2^24 elements) against float64, and the parameters, bf16 shadow and momentum against a float64
  restatement of the update on x's rows 0 and 32767 (the latter ends at flat index 2^31 - 1) and column 65535,
  and on all of y/kernel and y/bias (flat indices 2^31 .. the end).

  Device memory: 10 bytes per element for the parameters, gradients and bf16 shadow, plus 2 bytes of bf16
  momentum, about 25.2 GiB, and 1 GiB of float64 scratch."""
  from big_vision_b200 import engine as E
  from big_vision_b200 import optax as bv_optax
  specs = [E.ParamSpec("x/kernel", (ROWS, COLS), E.zeros), E.ParamSpec("y/kernel", (YN, YN), E.zeros),
           E.ParamSpec("y/bias", (YN,), E.zeros)]
  P = E.FlatParams(specs, [], "cuda")
  assert P.offsets["y/kernel"][0] == TWO31 and P.total == TWO31 + YN * YN + YN
  lr, wd, beta = 1e-3, 1e-4, 0.9
  config = dict(optax_name="big_vision.scale_by_adafactor", grad_clip_norm=1.0, lr=lr, wd=wd,
                schedule=dict(decay_type="cosine", warmup_steps=0))
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=10, batch_size=1, data_size=10))
  assert [(lo, hi) for lo, hi, *_ in tx.ranges] == [(0, TWO31 + YN * YN), (TWO31 + YN * YN, P.total)]
  assert [t.mode for t, *_ in tx.tensors] == [1, 1, 0]
  opt = tx.init(P)
  gen = torch.Generator(device="cuda").manual_seed(31)
  P.flat.normal_(0.0, 0.02, generator=gen)
  P.sync_half()
  x, y, yb = P.f("x/kernel"), P.f("y/kernel"), P.f("y/bias")
  # float64 reference state: x on the checked rows and column, y and y/bias whole
  rows_chk, col_chk = [0, ROWS - 1], COLS - 1
  ref = {"x_rows": x[rows_chk].double(), "x_col": x[:, col_chk].double(), "y": y.double(), "yb": yb.double()}
  mom = {k: torch.zeros_like(v) for k, v in ref.items()}
  # error bounds: a bf16 rounding of the momentum may go the other way on the device (2^-7 of the terms it
  # sums, per step); the parameters carry the momentum's bound times lr plus fp32 rounding
  mtol = {k: torch.zeros_like(v) for k, v in ref.items()}
  ptol = {k: torch.zeros_like(v) for k, v in ref.items()}
  red = {}                                    # factored second moments: (rows, cols) of x and y; vfull of yb
  eps = 1e-30
  for step in range(2):
    P.grad.normal_(0.0, 1.0, generator=gen)
    gx, gy, gyb = P.g("x/kernel"), P.g("y/kernel"), P.g("y/bias")
    gsq = _sumsq64(P.grad)
    sc = tx.update(P, opt)
    torch.cuda.synchronize()
    # the clip norm's sum of squares over the whole buffer (one sumsq launch over > 2^31 elements)
    assert float(sc[0]) == pytest.approx(gsq, rel=1e-5)
    gs = min(1.0, 1.0 / math.sqrt(gsq))
    t = np.float32(step) + np.float32(1.0)
    decay = float(min(np.float32(0.999), np.float32(1.0) - t ** np.float32(-0.8)))
    lr_eff, wd_eff = tx.sched_fns[0](step) * lr, tx.sched_fns[0](step) * wd
    xr, xc = _row_col_sumsq(gx, gs)
    yr, yc = _row_col_sumsq(gy, gs)
    new = {"x": (xr / COLS + eps, xc / ROWS + eps), "y": (yr / YN + eps, yc / YN + eps),
           "yb": (gyb.double() * gs) ** 2 + eps}
    for k, v in new.items():                  # ema, decay 0 on the first step
      red[k] = v if step == 0 else (tuple(decay * a + (1 - decay) * b for a, b in zip(red[k], v))
                                    if k != "yb" else decay * red[k] + (1 - decay) * v)

    def factored(g, k, rows, cols):
      r, c = red[k]                           # mode 1: R0 = row means (d0 = the last axis), normaliser mean_L(R0)
      return g.double() * gs * torch.rsqrt(r[rows].unsqueeze(1) / r.mean()) * torch.rsqrt(c[cols].unsqueeze(0))

    everything, last = slice(None), slice(col_chk, None)
    u = {"x_rows": factored(gx[rows_chk], "x", rows_chk, everything),
         "x_col": factored(gx[:, last], "x", everything, last)[:, 0],
         "y": factored(gy, "y", everything, everything), "yb": gyb.double() * gs * torch.rsqrt(red["yb"])}
    for k in ref:
      mtol[k] = beta * mtol[k] + 2 ** -6 * (beta * mom[k].abs() + (1 - beta) * u[k].abs()) + 1e-12
      mom[k] = _bf16(beta * mom[k] + (1 - beta) * u[k])
      ref[k] = ref[k] - (lr_eff * mom[k] + (wd_eff if k != "yb" else 0.0) * ref[k])
      ptol[k] = ptol[k] + 1e-6 * ref[k].abs() + lr_eff * mtol[k]
    got = {"x_rows": x[rows_chk], "x_col": x[:, col_chk], "y": y, "yb": yb}
    half = {"x_rows": P.h("x/kernel")[rows_chk], "x_col": P.h("x/kernel")[:, col_chk], "y": P.h("y/kernel"),
            "yb": P.h("y/bias")}
    moms = {"x_rows": opt["af"][0]["momentum"].view(ROWS, COLS)[rows_chk],
            "x_col": opt["af"][0]["momentum"].view(ROWS, COLS)[:, col_chk],
            "y": opt["af"][1]["momentum"].view(YN, YN), "yb": opt["af"][2]["momentum"]}
    for k in ref:
      err = (got[k].double() - ref[k]).abs()
      assert bool((err <= ptol[k]).all()), (step, k, float((err / ptol[k]).max()))
      assert torch.equal(half[k], got[k].to(torch.bfloat16)), (step, k)
      merr = (moms[k].double() - mom[k]).abs()
      assert bool((merr <= mtol[k]).all()), (step, k, float((merr / mtol[k]).max()))
    # l2_params over the whole buffer
    assert float(sc[2]) == pytest.approx(_sumsq64(P.flat), rel=1e-5)
  del P, opt, tx


def test_vit_e14_update_fn_step_updates_parameters_past_2_31():
  """One update_fn step of the full 56-block e/14 (MAP head, 29,593 classes, scan) at batch 2 with the
  config's optimizer (BV-Adafactor, clip 1, wd_mults; a schedule without warmup so the step moves the
  weights): the loss is finite, and every reference element at a flat index >= 2^31 moved while the storage
  padding there stayed as it was.  Device memory: about 47 GiB of parameters, gradients, bf16 shadow and
  momentum, and 9 GiB for the copy of the buffer's tail and its masks."""
  from big_vision_b200 import engine as E
  from big_vision_b200 import optax as bv_optax, train
  from big_vision_b200.models import vit
  model = vit.Model(C, variant="e/14", pool_type="map", scan=True)
  n, shape = 2, (2, 224, 224, 3)
  P = E.FlatParams(*model.specs(shape[1:3], shape[3]), "cuda")
  assert P.total > TWO31
  for v in P.tree("f").values():             # marks the reference elements; the storage padding stays 0
    v.fill_(1.0)
  ref_elem = P.flat[TWO31:] != 0
  gen = torch.Generator(device="cuda").manual_seed(5)
  for k, v in P.tree("f").items():
    if not k.endswith("/scale"):
      v.normal_(0.0, 0.02, generator=gen)
  P.sync_half()
  config = dict(optax_name="big_vision.scale_by_adafactor", grad_clip_norm=1.0, lr=8e-4, wd=0.03 * 8e-4,
                wd_mults=[(".*head/kernel", 100.0), (".*/kernel", 1.0)], loss="sigmoid_xent",
                schedule=dict(decay_type="rsqrt", timescale=1_000, warmup_steps=0, cooldown_steps=5))
  tx, _ = bv_optax.make(config, P, sched_kw=dict(total_steps=10, batch_size=n, data_size=1000))
  state = {"params": P, "opt": tx.init(P)}
  rng = np.random.default_rng(7)
  batch = {"image": torch.from_numpy(rng.uniform(-1, 1, shape).astype(np.float32)).cuda(),
           "labels": torch.from_numpy(np.eye(C, dtype=np.float32)[rng.integers(0, C, n)]).cuda()}
  tail0 = P.flat[TWO31:].clone()
  state, m = train.make_update_fn(model, tx, config)(state, None, batch)
  torch.cuda.synchronize()
  assert math.isfinite(float(m["training_loss"])) and float(m["training_loss"]) > 0
  assert all(math.isfinite(float(m[k])) for k in ("l2_grads", "l2_params", "l2_updates"))
  tail = P.flat[TWO31:]
  # the class head and the MAP head lie wholly past 2^31: (nearly) every element of each moved
  for name in ("head/kernel", "head/bias", "MAPHead_0/probe", "MAPHead_0/MlpBlock_0/Dense_1/kernel"):
    cur = P.tree("f")[name]
    off = cur.storage_offset() - TWO31
    assert off >= 0
    assert float((cur != torch.as_strided(tail0, cur.shape, cur.stride(), off)).float().mean()) >= 0.999, name
  moved = tail != tail0
  del tail0
  n_ref = int(torch.count_nonzero(ref_elem))
  assert n_ref > 1_700_000_000
  assert not bool((moved & ~ref_elem).any())                # the padding was not written
  moved &= ref_elem
  assert int(torch.count_nonzero(moved)) >= (1 - 1e-3) * n_ref
  del moved, ref_elem
  assert bool(torch.isfinite(tail).all())
  assert torch.equal(P.half[TWO31:], tail.to(torch.bfloat16))
