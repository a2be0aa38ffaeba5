"""CPU: classifier heads of any class count (padded storage exposed under the reference names and
shapes, unchanged layout when C % 8 == 0, optimizer masks and Adafactor factoring on the reference
tensors), the strided xent entry points' refusal of ld < C, ViT-G/14 (head dim 104) shapes and
parameter count, and the ViT-G/14 benchmark workload."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

from big_vision_b200 import engine as E
from big_vision_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLASS_COUNTS = [21843, 29593, 37]


def _model(kind, C, **kw):
  from big_vision_b200.models import mlp_mixer, vit
  if kind == "mixer":
    return mlp_mixer.Model(C, patch_size=(16, 16), num_blocks=2, hidden_dim=64, tokens_mlp_dim=32,
                           channels_mlp_dim=128, **kw)
  return vit.Model(C, width=64, depth=2, mlp_dim=128, num_heads=1, patch_size=(16, 16), pool_type=kind, **kw)


def _flat(model, hw=(64, 64)):
  return E.FlatParams(*model.specs(hw, 3), "meta")


@pytest.mark.parametrize("C", CLASS_COUNTS)
@pytest.mark.parametrize("kind", ["map", "gap", "tok", "mixer"])
def test_padded_head_has_reference_names_and_shapes(kind, C):
  P = _flat(_model(kind, C))
  shapes = {k: tuple(v.shape) for k, v in P.tree("f").items()}
  assert shapes["head/kernel"] == (64, C) and shapes["head/bias"] == (C,)
  assert not any(k.startswith("head/") and k not in ("head/kernel", "head/bias") for k in shapes)
  Cp = (C + 7) // 8 * 8
  assert P.offsets["head/kernel_pad"][1] == (64, Cp) and P.offsets["head/bias_pad"][1] == (Cp,)
  assert P.tree("f")["head/kernel"].stride() == (Cp, 1)


@pytest.mark.parametrize("C", CLASS_COUNTS)
def test_padded_head_init_is_zero_in_the_padding(C):
  from big_vision_b200.models import vit
  model = vit.Model(C, width=64, depth=1, mlp_dim=128, num_heads=1, patch_size=(16, 16), head_zeroinit=False)
  P = E.FlatParams(*model.specs((32, 32), 3), "cpu").init(0)
  k = P.f("head/kernel_pad")
  assert float(k[:, C:].abs().max()) == 0.0 and float(P.f("head/bias_pad").abs().max()) == 0.0
  assert float(k[:, :C].abs().max()) > 0.0


# FlatParams layout of the parent layout at C = 1000 (B/16 at 224): (total, n_decay, head/kernel offset,
# head/bias offset, number of specs, number of aliases)
PARENT_LAYOUT_1000 = {
    "vit_map": (93653224, 93370368, 92602368, 93652224, 164, 92),
    "vit_tok": (87157480, 86882304, 86114304, 87156480, 154, 85),
    "mixer": (59898952, 59805696, 59037696, 59897952, 150, 25),
}


@pytest.mark.parametrize("name", sorted(PARENT_LAYOUT_1000))
def test_class_count_multiple_of_8_keeps_the_layout(name):
  from big_vision_b200.models import mlp_mixer, vit
  model = {"vit_map": lambda: vit.Model(1000, variant="B/16", pool_type="map"),
           "vit_tok": lambda: vit.Model(1000, variant="B/16", pool_type="tok", rep_size=True),
           "mixer": lambda: mlp_mixer.Model(1000, variant="B/16")}[name]()
  specs, aliases = model.specs((224, 224), 3)
  P = E.FlatParams(specs, aliases, "meta")
  got = (P.total, P.n_decay, P.offsets["head/kernel"][0], P.offsets["head/bias"][0], len(specs), len(aliases))
  assert got == PARENT_LAYOUT_1000[name]
  assert P.offsets["head/kernel"][1] == (768, 1000) and "head/kernel_pad" not in P.offsets
  assert not any(a.name.startswith("head/") for a in aliases)


def _chain(P, **config):
  from big_vision_b200 import optax as bv_optax
  config.setdefault("schedule", dict(decay_type="cosine", warmup_steps=0))
  return bv_optax.Chain(config, P, dict(total_steps=100, batch_size=8, data_size=1000))


@pytest.mark.parametrize("kind", ["map", "mixer"])
def test_optimizer_masks_select_the_padded_head(kind):
  P = _flat(_model(kind, 21843))
  tx = _chain(P, optax_name="scale_by_adam", lr=1e-3, wd=0.1, wd_mults=[(".*head/kernel", 100.0), (".*/kernel", 1.0)])
  wd = {storage: w for storage, _, _, w in tx.per_storage}
  assert wd["head/kernel_pad"] == pytest.approx(10.0) and wd["head/bias_pad"] == 0.0
  # the padded storage lies whole inside the launch range whose setting its names select
  for storage, want in (("head/kernel_pad", 10.0), ("head/bias_pad", 0.0)):
    off, shape = P.offsets[storage]
    n = int(np.prod(shape))
    (lo, hi, _, _, w), = [r for r in tx.ranges if r[0] <= off < r[1]]
    assert off + n <= hi and w == pytest.approx(want)
  # the default decay mask (.*/kernel$, on the reference names) puts the padded kernel in the decayed range
  off, shape = P.offsets["head/kernel_pad"]
  assert off + int(np.prod(shape)) <= P.n_decay and P.offsets["head/bias_pad"][0] >= P.n_decay


@pytest.mark.parametrize("C", [21843, 37, 12])
def test_adafactor_factors_the_head_over_the_reference_shape(C):
  P = _flat(_model("map", C))
  tx = _chain(P, optax_name="big_vision.scale_by_adafactor", lr=1e-3, wd=1e-4)
  tens = {t.name: t for t, *_ in tx.tensors}
  k, b = tens["head/kernel"], tens["head/bias"]
  Cp = (C + 7) // 8 * 8
  assert k.numel == 64 * C and b.numel == C
  assert k.offset == P.offsets["head/kernel_pad"][0] and k.strides[1] == Cp
  if C >= 32:        # min_dim_size_to_factor: both axes factored over (rep, C)
    assert k.mode in (1, 2) and k.dims == (1, 64, 1, C)
  else:              # unfactored, a [rep, C] view with row stride Cp
    assert k.mode == 0 and k.dims == (1, 64, 1, C)
  assert "head/kernel_pad" not in tens and "head/bias_pad" not in tens


@pytest.mark.parametrize("scan", [False, True])
def test_vit_G14_builds_reference_shapes(scan):
  from big_vision_b200.models import vit
  model = vit.Model(29_593, variant="G/14", pool_type="map", scan=scan)
  assert model.width // model.num_heads == 104
  got = {k: tuple(v.shape) for k, v in _flat(model, (224, 224)).tree("f").items()}
  blk, lead = ("Transformer/encoderblock/", (48,)) if scan else ("Transformer/encoderblock_47/", ())
  assert got[blk + "MultiHeadDotProductAttention_0/query/kernel"] == lead + (1664, 16, 104)
  assert got[blk + "MultiHeadDotProductAttention_0/out/kernel"] == lead + (16, 104, 1664)
  assert got[blk + "MlpBlock_0/Dense_0/kernel"] == lead + (1664, 8192)
  assert got["MAPHead_0/MultiHeadDotProductAttention_0/query/kernel"] == (1664, 16, 104)
  assert got["head/kernel"] == (1664, 29_593) and got["head/bias"] == (29_593,)
  assert got["embedding/kernel"] == (14, 14, 3, 1664) and got["pos_embedding"] == (1, 256, 1664)
  assert abs(sum(int(np.prod(s)) for s in got.values()) / 1e6 - 1930.4) < 0.05


def test_g_and_mu_are_still_refused():
  from big_vision_b200.models import vit
  for variant in ("g", "mu"):
    with pytest.raises(NotImplementedError, match="64, 72, 80, 96"):
      vit.Model(None, variant=f"{variant}/14")


def test_hd_entry_points_list_104():
  lib = L.load()
  assert lib.bv_attention_fwd_hd(ctypes.byref(L.AttnArgs()), 88, None) == -3
  assert "64, 72, 80, 96, 104" in lib.bv_last_error_string().decode()


@pytest.mark.parametrize("name", ["bv_sigmoid_xent_ld", "bv_softmax_xent_ld"])
@pytest.mark.parametrize("which", [0, 1, 2])
def test_xent_ld_refuses_row_stride_below_C(name, which):
  """Refused before any CUDA call: the pointers are dangling on purpose and the machine needs no GPU."""
  lib = L.load()
  ld = [37, 37, 40]
  ld[which] = 36
  bogus = ctypes.c_void_p(16)
  rc = getattr(lib, name)(bogus, ld[0], bogus, ld[1], bogus, bogus, ld[2], None, 4, 37, None)
  assert rc == -1
  assert "row strides must be >= C" in lib.bv_last_error_string().decode()


def _bench_G14():
  spec = importlib.util.spec_from_file_location("bench_vit_G14", os.path.join(ROOT, "tools", "bench_vit_G14.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def test_vit_G14_workload_registers_and_counts_flops():
  mod = _bench_G14()
  opt_before = mod.bench.OPT_CONFIG
  try:
    wl = mod.register()
    assert mod.bench.WORKLOADS["scaling_laws_vit_G14"] is wl
    assert mod.bench.OPT_CONFIG["optax_name"] == "big_vision.scale_by_adafactor"
    assert mod.bench.OPT_CONFIG["wd_mults"] == [(".*head/kernel", 100.0), (".*/kernel", 1.0)]
    model = mod.bench.build_model(wl)
    assert model.scan and model.pool_type == "map" and model.num_classes == 29_593
    assert model.width == 1664 and model.num_heads == 16 and model.patch_size == (14, 14)
    b = mod.bench.synthetic_batch(wl, 2, seed=0)
    assert b["image"].shape == (2, 224, 224, 3) and b["labels"].shape == (2, 29_593)
    assert abs(wl["flops"] / 1e9 - 2899.9) < 0.05
    counts = mod.param_counts()
    assert abs(counts["total"] / 1e6 - 1930.4) < 0.05 and counts["head"] == 1664 * 29_593 + 29_593
  finally:
    mod.bench.OPT_CONFIG = opt_before
    mod.bench.WORKLOADS.pop("scaling_laws_vit_G14", None)
