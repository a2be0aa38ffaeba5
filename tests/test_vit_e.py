"""CPU: ViT-e/14 (head dim 112, 3,926.4 M parameters) builds the reference's parameter names and shapes,
the text tower builds at `e`, the head-dim entry points accept 112 and still refuse 88 and a key mask at
112 before any CUDA call, the e/14 benchmark workload counts its FLOPs by the SURVEY.md 8d formula, and
Adafactor takes the scan-stacked q / k / v biases of a small e-shaped model as strided unfactored views."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

from big_vision_b200 import engine as E
from big_vision_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C = 29_593


def _shapes(model, hw=(224, 224)):
  return {k: tuple(v.shape) for k, v in E.FlatParams(*model.specs(hw, 3), "meta").tree("f").items()}


@pytest.mark.parametrize("scan", [False, True])
def test_vit_e14_builds_reference_shapes(scan):
  from big_vision_b200.models import vit
  v = vit.decode_variant("e/14")
  assert v == dict(width=1792, depth=56, mlp_dim=15360, num_heads=16, patch_size=(14, 14))
  model = vit.Model(None, variant="e/14", pool_type="map", scan=scan)
  assert model.width // model.num_heads == 112
  got = _shapes(model)
  d, h, dh, m, depth = v["width"], v["num_heads"], 112, v["mlp_dim"], v["depth"]
  blk, lead = ("Transformer/encoderblock/", (depth,)) if scan else (f"Transformer/encoderblock_{depth - 1}/", ())
  if not scan:
    assert f"Transformer/encoderblock_{depth}/LayerNorm_0/scale" not in got
  for name in ("query", "key", "value"):
    assert got[blk + f"MultiHeadDotProductAttention_0/{name}/kernel"] == lead + (d, h, dh)
    assert got[blk + f"MultiHeadDotProductAttention_0/{name}/bias"] == lead + (h, dh)
    assert got[f"MAPHead_0/MultiHeadDotProductAttention_0/{name}/kernel"] == (d, h, dh)
  assert got[blk + "MultiHeadDotProductAttention_0/out/kernel"] == lead + (h, dh, d)
  assert got[blk + "MlpBlock_0/Dense_0/kernel"] == lead + (d, m)
  assert got[blk + "MlpBlock_0/Dense_1/kernel"] == lead + (m, d)
  assert got["MAPHead_0/MultiHeadDotProductAttention_0/out/kernel"] == (h, dh, d)
  assert got["MAPHead_0/MlpBlock_0/Dense_0/kernel"] == (d, m) and got["MAPHead_0/probe"] == (1, 1, d)
  assert got["embedding/kernel"] == (14, 14, 3, d) and got["pos_embedding"] == (1, 256, d)
  assert not any(k.startswith("head/") for k in got)


@pytest.mark.parametrize("scan", [False, True])
def test_vit_e14_with_the_jft_head_has_3926_4_m_parameters(scan):
  """The 29,593-class head is stored padded; the flat buffer passes 2^31 elements."""
  from big_vision_b200.models import vit
  model = vit.Model(C, variant="e/14", pool_type="map", scan=scan)
  P = E.FlatParams(*model.specs((224, 224), 3), "meta")
  got = {k: tuple(v.shape) for k, v in P.tree("f").items()}
  assert got["head/kernel"] == (1792, C) and got["head/bias"] == (C,)
  assert abs(sum(int(np.prod(s)) for s in got.values()) / 1e6 - 3926.4) < 0.05
  assert P.total > 2 ** 31
  # the reference tensors that lie wholly past 2^31 include the MAP head and the class head
  assert min(P.offsets["head/kernel_pad"][0], P.offsets["MAPHead_0/probe"][0]) >= 2 ** 31


@pytest.mark.parametrize("scan", [False, True])
def test_text_tower_builds_at_e(scan):
  from big_vision_b200.models.proj.image_text import text_transformer
  model = text_transformer.Model(None, variant="e", vocab_size=32_000, scan=scan)
  assert model.width == 1792 and model.width // model.num_heads == 112


@pytest.mark.parametrize("fn,args", [("bv_attention_fwd_hd", L.AttnArgs), ("bv_attention_bwd_hd", L.AttnBwdArgs)])
def test_hd_entry_points_accept_112(fn, args):
  """A zero-filled args struct at head dim 112 passes the head-dim check and is refused by the argument
  check (B = 0), before any CUDA call: BV_ERR_INVALID, not BV_ERR_UNSUPPORTED."""
  lib = L.load()
  assert getattr(lib, fn)(ctypes.byref(args()), 112, None) == -1
  msg = lib.bv_last_error_string().decode()
  assert msg.startswith(fn + ":") and "not supported" not in msg, msg


def test_head_dim_88_is_still_refused_and_the_message_lists_112():
  lib = L.load()
  for fn, args in (("bv_attention_fwd_hd", L.AttnArgs), ("bv_attention_bwd_hd", L.AttnBwdArgs)):
    assert getattr(lib, fn)(ctypes.byref(args()), 88, None) == -3
    assert "head_dim 88" in lib.bv_last_error_string().decode()
    assert "64, 72, 80, 96, 104, 112" in lib.bv_last_error_string().decode()


def test_a_key_mask_at_112_is_refused():
  lib = L.load()
  mask = (ctypes.c_uint8 * 4)(1, 1, 1, 1)
  m = L.AttnMaskedArgs(key_mask=ctypes.cast(mask, ctypes.c_void_p), bsmask=4)
  assert lib.bv_attention_fwd_hd(ctypes.byref(m.attn), 112 | L.ATTN_KEY_MASK, None) == -1
  assert "head_dim 64 only" in lib.bv_last_error_string().decode()
  mb = L.AttnMaskedBwdArgs(key_mask=ctypes.cast(mask, ctypes.c_void_p), bsmask=4)
  assert lib.bv_attention_bwd_hd(ctypes.byref(mb.attn), 112 | L.ATTN_KEY_MASK, None) == -1
  assert "head_dim 64 only" in lib.bv_last_error_string().decode()


def _bench():
  spec = importlib.util.spec_from_file_location("bench_vit_G14", os.path.join(ROOT, "tools", "bench_vit_G14.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def test_vit_e14_workload_registers_and_counts_flops():
  mod = _bench()
  opt_before = mod.bench.OPT_CONFIG
  try:
    wl = mod.register("e/14")
    assert mod.bench.WORKLOADS["scaling_laws_vit_e14"] is wl
    assert "scaling_laws_vit_G14" not in mod.bench.WORKLOADS
    assert mod.bench.OPT_CONFIG["optax_name"] == "big_vision.scale_by_adafactor"
    assert wl["remat"] and wl["loss"] == "sigmoid_xent" and wl["num_classes"] == C
    model = mod.bench.build_model(wl)
    assert model.scan and model.pool_type == "map" and model.num_classes == C
    assert model.width == 1792 and model.depth == 56 and model.mlp_dim == 15360 and model.num_heads == 16
    # SURVEY.md 8d: per block 8*N*d^2 + 4*N*d*m + 4*N^2*d; patch embedding, MAP head and class head once;
    # training = 3 x forward
    d, m, depth, N = 1792, 15360, 56, 256
    block = 8 * N * d * d + 4 * N * d * m + 4 * N * N * d
    fwd = 2 * N * 14 * 14 * 3 * d + depth * block + (4 * N * d * d + 4 * d * d + 4 * N * d + 4 * d * m) + 2 * d * C
    assert wl["flops"] == 3 * fwd
    assert abs(wl["flops"] / 1e9 - 5931.2) < 0.05
    counts = mod.param_counts(wl)
    assert abs(counts["total"] / 1e6 - 3926.4) < 0.05 and counts["head"] == 1792 * C + C
    # the default variant is still G/14
    assert mod.VARIANTS["G/14"][1] is mod.WORKLOAD and mod.WORKLOAD["per_gpu_batch"] == 512
  finally:
    mod.bench.OPT_CONFIG = opt_before
    mod.bench.WORKLOADS.pop("scaling_laws_vit_e14", None)


def test_adafactor_takes_scan_stacked_unfactored_qkv_biases():
  """With depth and heads below min_dim_size_to_factor, a scan-stacked q / k / v bias [depth, heads, dh] is a
  strided view of the fused bias storage and keeps a full second moment over that view."""
  from big_vision_b200 import optax as bv_optax
  from big_vision_b200.models import vit
  model = vit.Model(37, width=224, depth=2, mlp_dim=448, num_heads=2, patch_size=(16, 16), pool_type="map", scan=True)
  P = E.FlatParams(*model.specs((64, 48), 3), "meta")
  tx, _ = bv_optax.make(dict(optax_name="big_vision.scale_by_adafactor", lr=1e-3), P,
                        sched_kw=dict(total_steps=10, batch_size=1, data_size=10))
  tens = {t.name: t for t, *_ in tx.tensors}
  blk = "Transformer/encoderblock/MultiHeadDotProductAttention_0/"
  q, k = tens[blk + "query/bias"], tens[blk + "key/bias"]
  assert q.mode == 0 and q.dims == (2, 2, 1, 112) and q.strides == (3 * 224, 112, 0)
  assert k.offset == q.offset + 224 and q.state_sizes() == {"vfull": 2 * 2 * 112}
