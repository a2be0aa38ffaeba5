"""CPU: the head-dim entry points refuse unsupported head dims before any CUDA call, the So400m models
build the reference's parameter shapes, head dims without kernels are refused at model construction,
and the So400m benchmark workload builds and counts its FLOPs by the SURVEY.md 8d formula."""
import ctypes
import importlib.util
import os

import pytest

from big_vision_b200 import engine as E
from big_vision_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("head_dim", [68, 88, 128])
def test_hd_entry_points_refuse_unsupported_head_dims(head_dim):
  lib = L.load()
  rc = lib.bv_attention_fwd_hd(ctypes.byref(L.AttnArgs()), head_dim, None)
  assert rc == -3
  msg = lib.bv_last_error_string().decode()
  assert f"head_dim {head_dim}" in msg and "64, 72, 80, 96" in msg
  rc = lib.bv_attention_bwd_hd(ctypes.byref(L.AttnBwdArgs()), head_dim, None)
  assert rc == -3
  assert "64, 72, 80, 96" in lib.bv_last_error_string().decode()


def _shapes(specs, aliases):
  return {k: tuple(v.shape) for k, v in E.FlatParams(specs, aliases, "meta").tree("f").items()}


@pytest.mark.parametrize("scan", [False, True])
def test_so400m_image_tower_builds_reference_shapes(scan):
  from big_vision_b200.models import vit
  model = vit.Model(None, variant="So400m/14", pool_type="map", scan=scan)
  got = _shapes(*model.specs((224, 224), 3))
  if scan:
    blk, lead = "Transformer/encoderblock/", (27,)
  else:
    blk, lead = "Transformer/encoderblock_26/", ()
    assert "Transformer/encoderblock_27/LayerNorm_0/scale" not in got
  assert got[blk + "MultiHeadDotProductAttention_0/query/kernel"] == lead + (1152, 16, 72)
  assert got[blk + "MultiHeadDotProductAttention_0/out/kernel"] == lead + (16, 72, 1152)
  assert got[blk + "MlpBlock_0/Dense_0/kernel"] == lead + (1152, 4304)
  assert got["MAPHead_0/MultiHeadDotProductAttention_0/query/kernel"] == (1152, 16, 72)
  assert got["embedding/kernel"] == (14, 14, 3, 1152) and got["pos_embedding"] == (1, 256, 1152)


@pytest.mark.parametrize("scan", [False, True])
def test_so400m_two_towers_build_reference_shapes(scan):
  from big_vision_b200.models.proj.image_text import two_towers
  model = two_towers.Model(image=dict(variant="So400m/14", pool_type="map", scan=scan),
                           text=dict(variant="So400m", vocab_size=32_000, scan=scan), out_dim=(None, 1152))
  got = _shapes(*model.specs((2, 224, 224, 3), (2, 16)))
  blk, lead = ("txt/Encoder_0/encoderblock/", (27,)) if scan else ("txt/Encoder_0/encoderblock_0/", ())
  assert got[blk + "MultiHeadDotProductAttention_0/query/kernel"] == lead + (1152, 16, 72)
  assert got[blk + "MultiHeadDotProductAttention_0/out/kernel"] == lead + (16, 72, 1152)
  assert got[blk + "MlpBlock_0/Dense_0/kernel"] == lead + (1152, 4304)
  assert got["txt/head/kernel"] == (1152, 1152) and got["txt/Embed_0/embedding"] == (32_000, 1152)


@pytest.mark.parametrize("variant", ["mu", "g"])
def test_head_dims_without_kernels_are_refused(variant):
  from big_vision_b200.models import vit
  from big_vision_b200.models.proj.image_text import text_transformer
  with pytest.raises(NotImplementedError, match="64, 72, 80, 96"):
    vit.Model(None, variant=f"{variant}/16")
  with pytest.raises(NotImplementedError, match="64, 72, 80, 96"):
    text_transformer.Model(None, variant=variant)


def test_supported_variants_build():
  from big_vision_b200.models import vit
  for variant, dh in (("B", 64), ("So400m", 72), ("H", 80), ("g-opt", 96), ("G-opt", 96)):
    m = vit.Model(None, variant=f"{variant}/14")
    assert m.width // m.num_heads == dh


def _bench_so400m():
  spec = importlib.util.spec_from_file_location("bench_so400m", os.path.join(ROOT, "tools", "bench_so400m.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def test_so400m_workload_builds_and_counts_flops():
  mod = _bench_so400m()
  wl = mod.register()
  assert mod.bench.WORKLOADS["siglip_so400m14_224"] is wl
  model = mod.bench.build_model(wl)
  assert model.img.scan and model.txt.scan and model.img.width == 1152 and model.img.patch_size == (14, 14)
  assert model.img.num_heads == 16 and model.txt.width == 1152 and model.txt.mlp_dim == 4304
  b = mod.bench.synthetic_batch(wl, 2, seed=0)
  assert b["image"].shape == (2, 224, 224, 3) and b["labels"].shape == (2, 64)
  # SURVEY.md 8d per block: 24*N*d^2 + 4*N^2*d when m = 4d, i.e. 8*N*d^2 + 4*N*d*m + 4*N^2*d in general
  d, m, depth, N, T = 1152, 4304, 27, 256, 64
  block = lambda n: 8 * n * d * d + 4 * n * d * m + 4 * n * n * d  # noqa: E731
  img = 2 * N * 14 * 14 * 3 * d + depth * block(N) + (4 * N * d * d + 4 * d * d + 4 * N * d + 4 * d * m)
  txt = depth * block(T) + 2 * d * d
  assert wl["flops"] == 3 * (img + txt)
  assert abs(wl["flops"] / 1e9 - 820.4) < 0.1
  counts = mod.param_counts()
  assert abs(counts["img"] / 1e6 - 428) < 1 and abs(counts["txt"] / 1e6 - 450) < 1
