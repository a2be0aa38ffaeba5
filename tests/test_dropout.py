"""CPU: dropout for the ViT and text towers.  The C ABI of include/bv_dropout.h (its functions exported and
bound one to one, plain C that a C program links against, each entry point named with the GPU tests that
call its ops function), the numpy restatement of the mask stream (its realized rate, its independence across
sites, steps, seeds and rows, and its separation from Jet's noise), the refusals of the entry points and of
the models, the key struct's layout against a C program, and what the models launch and keep with dropout,
recorded by tests/golden/make_model_traces.py's recorder."""
import ctypes
import importlib.util
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import dropout_oracle as D
from common import header_functions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "bv_dropout.h")

# entry point -> the GPU tests of tests/test_dropout_gpu.py that check it directly against numpy / float64
COVERAGE = {
    "bv_dropout": ["test_dropout_is_numpy_bit_for_bit", "test_column_sums_match_fp64_and_runs_repeat",
                   "test_realized_rate_at_b16_shapes"],
    "bv_dropout_add": ["test_dropout_add_is_numpy_bit_for_bit"],
}


# ---- the C ABI of include/bv_dropout.h ------------------------------------------------------------------
def test_header_functions_are_exported_and_bound_one_to_one():
  from big_vision_b200 import lib as L
  declared = header_functions(HEADER)
  assert declared == set(L.DROPOUT_SIGNATURES) == set(COVERAGE)
  assert not declared & set(L.SIGNATURES)
  lib = L.load()
  for name in declared:
    assert tuple(getattr(lib, name).argtypes) == tuple(L.DROPOUT_SIGNATURES[name])


def test_every_entry_point_has_gpu_tests_that_call_its_op():
  import ast
  tree = ast.parse(open(os.path.join(ROOT, "tests", "test_dropout_gpu.py")).read())
  gpu_module = any(isinstance(n, ast.Assign) and any(getattr(t, "id", "") == "pytestmark" for t in n.targets)
                   and ast.unparse(n.value) == "pytest.mark.gpu" for n in tree.body)
  assert gpu_module
  tests = {n.name: ast.unparse(n) for n in tree.body if isinstance(n, ast.FunctionDef) and n.name.startswith("test_")}
  for fn, names in COVERAGE.items():
    for t in names:
      assert t in tests, (fn, t)
      assert fn.replace("bv_", "ops.", 1) + "(" in tests[t], (fn, t)


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no gcc")
def test_header_is_plain_c_and_a_c_program_links(tmp_path):
  """The header compiles as C99 and C++, and a C program that includes it links against libbv_b200.so and
  gets the refusals that need no GPU."""
  from big_vision_b200 import lib as L
  L.load()
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c", HEADER], check=True)
  subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", HEADER], check=True)
  src = tmp_path / "main.c"
  src.write_text("""#include <stdio.h>
#include "bv_dropout.h"
int main(void) {
  /* a rate of 1, then site 0 */
  unsigned short buf[64];
  bv_dropout_key key = {1, 2, 3, 0, 1.f};
  int a = bv_dropout(buf, 8, buf, 8, 4, 8, &key, NULL);
  key.rate = 0.1f;
  key.site = 0;
  int b = bv_dropout_add(buf, 8, buf, 8, buf, 8, 4, 8, &key, NULL);
  printf("%d %d %s\\n", a, b, bv_last_error_string());
  return 0;
}
""")
  libdir = os.path.dirname(os.path.abspath(L.LIB_PATH))
  exe = tmp_path / "main"
  subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                  "-L", libdir, "-lbv_b200", f"-Wl,-rpath,{libdir}"], check=True)
  out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split(None, 2)
  assert [int(v) for v in out[:2]] == [-1, -1] and "bv_dropout_add" in out[2] and "site 0" in out[2], out


# ---- the mask stream ------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate", [0.1, 0.5, 0.03])
def test_realized_rate_is_within_the_binomial_bound(rate):
  n = 10_000_000
  dropped = int((D.lanes(7, 3, 5, 0, n) < D.threshold(rate)).sum())
  p = D.threshold(rate) / 65536
  assert abs(p - rate) <= 2.0 ** -17 + 1e-8
  assert abs(dropped / n - p) <= 5 * math.sqrt(p * (1 - p) / n)


def test_the_stream_is_numpys_philox_in_16_bit_lanes():
  raw = np.random.Philox(key=11, counter=[0, 4, 9, 0]).random_raw(8)   # blocks 0 and 1
  got = D.lanes(11, 4, 9, 0, 32)
  for e in range(32):
    assert got[e] == (int(raw[4 * (e // 16) + (e % 16) // 4]) >> (16 * (e % 4))) & 0xFFFF
  # any window of the stream is the same stream
  assert np.array_equal(D.lanes(11, 4, 9, 5, 29), got[5:29])


def test_sites_steps_seeds_and_rows_give_different_masks():
  rate, rows, cols = 0.1, 64, 96
  base = D.keep_mask(1, 2, 3, 0, rows, cols, rate)
  others = [D.keep_mask(1, 2, 4, 0, rows, cols, rate), D.keep_mask(1, 3, 3, 0, rows, cols, rate),
            D.keep_mask(2, 2, 3, 0, rows, cols, rate), D.keep_mask(1, 2, 3, rows, rows, cols, rate)]
  p = D.threshold(rate) / 65536
  for m in others:
    # independent masks agree on both being dropped at about p^2, far from the p of identical ones
    both = float((~base & ~m).mean())
    assert both < 3 * p * p + 0.005, both
  # the rows of a later rank are the continuation of the global stream
  assert np.array_equal(D.keep_mask(1, 2, 3, 0, 2 * rows, cols, rate)[rows:], others[3])


def test_no_site_meets_jets_stream():
  from big_vision_b200 import engine as E
  sites = [E.dropout_site(t, layer, k) for t in range(2) for layer in range(64) for k in range(4)]
  assert min(sites) >= 1 and len(set(sites)) == len(sites)
  # Jet's noise runs at counter word 2 = 0; the first dropout site never draws those words
  jet = np.random.Philox(key=0, counter=[0, 0, 0, 0]).random_raw(64)
  assert not np.array_equal(D.lanes(0, 0, min(sites), 0, 256).view("<u8"), jet)


# ---- refusals -----------------------------------------------------------------------------------------
def _key(**kw):
  from big_vision_b200 import lib as L
  return L.DropoutKey(**{"seed": 1, "step": 2, "site": 3, "row0": 0, "rate": 0.1, **kw})


@pytest.mark.parametrize("what,kw,args,message", [
    ("rate < 0", dict(rate=-0.1), {}, "outside [0, 1)"),
    ("rate 1", dict(rate=1.0), {}, "outside [0, 1)"),
    ("rate nan", dict(rate=float("nan")), {}, "outside [0, 1)"),
    ("site 0", dict(site=0), {}, "site 0"),
    ("row0 < 0", dict(row0=-1), {}, "row0 >= 0"),
    ("stride < cols", {}, dict(ldx=4), "stride >= cols"),
    ("no cols", {}, dict(cols=0), "cols >= 1"),
    ("misaligned", {}, dict(off=1), "2-byte aligned"),
    ("alias, other stride", {}, dict(alias=True, ldy=16), "aliasing"),
])
def test_bv_dropout_refusals(what, kw, args, message):
  from big_vision_b200 import lib as L
  lib = L.load()
  buf = (ctypes.c_uint16 * 256)()
  base = ctypes.addressof(buf) + args.get("off", 0)
  x, y = base, (base if args.get("alias") else ctypes.addressof(buf) + 256)
  rc = lib.bv_dropout(x, args.get("ldx", 8), y, args.get("ldy", 8), 4, args.get("cols", 8),
                      ctypes.byref(_key(**kw)), None)
  assert rc == -1, what
  err = lib.bv_last_error_string().decode()
  assert "bv_dropout" in err and message in err, err


def test_bv_dropout_add_refusals():
  from big_vision_b200 import lib as L
  lib = L.load()
  buf = (ctypes.c_uint16 * 256)()
  p = ctypes.addressof(buf)
  assert lib.bv_dropout_add(None, 8, p, 8, p + 64, 8, 4, 8, ctypes.byref(_key()), None) == -1
  assert b"null resid" in lib.bv_last_error_string()
  assert lib.bv_dropout_add(p, 8, p, 8, p + 64, 8, 4, 8, None, None) == -1
  assert b"null key" in lib.bv_last_error_string()
  assert lib.bv_dropout_add(p, 8, p + 128, 8, p, 16, 4, 8, ctypes.byref(_key()), None) == -1
  assert b"bv_dropout_add" in lib.bv_last_error_string()
  # rows = 0 launches nothing and succeeds without a device
  assert lib.bv_dropout(p, 8, p, 8, 0, 8, ctypes.byref(_key()), None) == 0


def test_ops_refuse_other_dtypes():
  from big_vision_b200 import lib as L, ops
  with pytest.raises(L.BvError):
    ops.dropout(torch.zeros(4, 8), _key())


@pytest.mark.parametrize("rate", [-0.1, 1.0, 1.5])
def test_models_refuse_a_rate_outside_0_1(rate):
  from big_vision_b200.models import vit
  from big_vision_b200.models.proj.image_text import text_transformer
  with pytest.raises(ValueError):
    vit.Model(10, width=64, depth=1, mlp_dim=128, num_heads=1, dropout=rate)
  with pytest.raises(ValueError):
    text_transformer.Model(10, width=64, depth=1, mlp_dim=128, num_heads=1, dropout=rate)


def test_apply_train_with_dropout_has_no_key():
  from big_vision_b200.models import vit
  from big_vision_b200.models.proj.image_text import text_transformer, two_towers
  m = vit.Model(10, width=64, depth=1, mlp_dim=128, num_heads=1, dropout=0.1)
  with pytest.raises(ValueError, match="dropout key"):
    m.apply({"params": None}, None, train=True)
  t = text_transformer.Model(10, width=64, depth=1, mlp_dim=128, num_heads=1, dropout=0.1)
  with pytest.raises(ValueError, match="dropout key"):
    t.apply({"params": None}, None, train=True)
  tt = two_towers.Model(image=dict(width=64, depth=1, mlp_dim=128, num_heads=1),
                        text=dict(width=64, depth=1, mlp_dim=128, num_heads=1, dropout=0.1))
  with pytest.raises(ValueError, match="dropout key"):
    tt.apply({"params": None}, None, None, train=True)


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no gcc")
def test_key_struct_layout_matches_the_header(tmp_path):
  from big_vision_b200 import lib as L
  prog = tmp_path / "layout.c"
  prog.write_text("""#include <stddef.h>
#include <stdio.h>
#include "bv_dropout.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(bv_dropout_key), offsetof(bv_dropout_key, seed),
         offsetof(bv_dropout_key, step), offsetof(bv_dropout_key, site), offsetof(bv_dropout_key, row0),
         offsetof(bv_dropout_key, rate));
  return 0;
}
""")
  exe = tmp_path / "layout"
  subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
  got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
  K = L.DropoutKey
  assert got == [ctypes.sizeof(K), K.seed.offset, K.step.offset, K.site.offset, K.row0.offset, K.rate.offset]


# ---- what the models launch and keep --------------------------------------------------------------------
def _generator():
  spec = importlib.util.spec_from_file_location("make_model_traces", os.path.join(ROOT, "tests", "golden",
                                                                                   "make_model_traces.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def _count(lines, name):
  return sum(1 for line in lines if line.split(" ", 1)[0] == name)


def _sites(lines):
  return [int(m) for m in re.findall(r"site=(\d+)", " ".join(lines))]


DEPTH = 3


def _vit(rate, **kw):
  from big_vision_b200 import engine as E
  from big_vision_b200.models import vit
  model = vit.Model(37, width=64, depth=DEPTH, mlp_dim=128, num_heads=1, patch_size=(16, 16), dropout=rate, **kw)
  return model, E.FlatParams(*model.specs((32, 32), 3), "cpu")


def _vit_step(gen, mp, model, P, frozen=None, dropout=None):
  image = torch.zeros((2, 32, 32, 3))
  out = {}

  def fwd():
    y, saved = model.fwd(P, image, frozen=frozen, dropout=dropout)
    out["y"], out["saved"] = y, saved
    return gen.saved_bytes(saved, P, image)

  fwd_lines, nbytes = gen._run(P, mp.setattr, fwd)   # pylint: disable=protected-access
  y, saved = out["y"], out["saved"]
  bwd_lines, _ = gen._run(P, mp.setattr,             # pylint: disable=protected-access
                          lambda: model.bwd(P, torch.zeros(y.shape[:-1] + (model.head.Cp,)), saved))
  return fwd_lines, bwd_lines, nbytes


@pytest.mark.parametrize("pool_type,scan", [("gap", False), ("tok", False), ("map", False), ("gap", True),
                                            ("tok", True)])
def test_dropout_adds_the_expected_calls_and_no_saved_bytes(pool_type, scan):
  from big_vision_b200 import engine as E
  gen = _generator()
  key = E.DropoutKey(seed=5, step=7, sample0=4)
  with pytest.MonkeyPatch.context() as mp:
    f0, b0, n0 = _vit_step(gen, mp, *_vit(0.0, pool_type=pool_type, scan=scan), dropout=key)
    model, P = _vit(0.1, pool_type=pool_type, scan=scan)
    f1, b1, n1 = _vit_step(gen, mp, model, P, dropout=key)
    # no key: the evaluation path, the same calls as rate 0
    fe, be, ne = _vit_step(gen, mp, model, P)
  assert (fe, be, ne) == (f0, b0, n0)
  assert n1 == n0
  assert _count(f0, "bv_dropout") == _count(b0, "bv_dropout") == _count(f0, "bv_dropout_add") == 0
  # forward: the embedding and each block's GELU output, and each block's two residual adds
  assert _count(f1, "bv_dropout") == 1 + DEPTH and _count(f1, "bv_dropout_add") == 2 * DEPTH
  assert _count(f1, "bv_gemm") == _count(f0, "bv_gemm")
  # backward: three masked gradients per block and the embedding's; with scan, the recompute's forward too
  recompute = 1 if scan else 0
  assert _count(b1, "bv_dropout") == 3 * DEPTH + 1 + recompute * DEPTH
  assert _count(b1, "bv_dropout_add") == recompute * 2 * DEPTH
  assert _count(b1, "bv_gemm") == _count(b0, "bv_gemm")
  # the bias gradients of the masked gradients (Dense_1, Dense_0, out and the patch embedding's without [cls])
  # are summed by their own pass instead of a neighbour's epilogue
  bias_sums = 3 * DEPTH + (0 if pool_type == "tok" else 1)
  assert _count(b1, "bv_colsum") == _count(b0, "bv_colsum") + bias_sums
  # every mask is drawn at this rank's rows and the step's key, at the model's sites
  N = 4 + (pool_type == "tok")
  assert all(f"row0={4 * N} " in line and "seed=5 " in line and "step=7 " in line
             for line in f1 + b1 if line.startswith("bv_dropout"))
  want = {E.dropout_site(0, 0, E.DROP_EMBED)} | {E.dropout_site(0, layer, k) for layer in range(DEPTH)
                                                  for k in (E.DROP_ATTN, E.DROP_GELU, E.DROP_MLP)}
  assert set(_sites(f1)) == set(_sites(b1)) == want


def test_forward_only_stages_drop_and_save_nothing():
  from big_vision_b200 import engine as E
  gen = _generator()
  key = E.DropoutKey(seed=5, step=7)
  model, P = _vit(0.1, pool_type="gap")
  image = torch.zeros((2, 32, 32, 3))
  with pytest.MonkeyPatch.context() as mp:
    lines, saved = gen._run(P, mp.setattr,   # pylint: disable=protected-access
                            lambda: model.fwd(P, image, frozen=True, dropout=key)[1])
    # a linear probe: every stage but the head runs forward-only
    frozen = frozenset(k for k in P.offsets if not k.startswith("head/"))
    probe, probe_saved = gen._run(P, mp.setattr,   # pylint: disable=protected-access
                                  lambda: model.fwd(P, image, frozen=frozen, dropout=key)[1])
  assert all(s is None for s in saved["stages"])
  assert _count(lines, "bv_dropout") == 1 + DEPTH and _count(lines, "bv_dropout_add") == 2 * DEPTH
  assert all(s is None for s in probe_saved["stages"][:-1])
  assert _count(probe, "bv_dropout") == 1 + DEPTH


def test_text_tower_drops_in_the_blocks_only_and_two_towers_use_their_own_sites():
  import common
  from big_vision_b200 import engine as E
  from big_vision_b200.models.proj.image_text import two_towers
  gen = _generator()
  kw = dict(common.TINY, image=dict(common.TINY["image"], dropout=0.1),
            text=dict(common.TINY["text"], dropout=0.2))
  model = two_towers.Model(**kw)
  P = E.FlatParams(*model.specs(common.TINY_IMAGE_SHAPE, common.TINY_TEXT_SHAPE), "cpu")
  image, text = torch.zeros(common.TINY_IMAGE_SHAPE), torch.ones(common.TINY_TEXT_SHAPE, dtype=torch.int32)
  with pytest.MonkeyPatch.context() as mp:
    lines, _ = gen._run(P, mp.setattr,   # pylint: disable=protected-access
                        lambda: model.fwd(P, image, text, dropout=E.DropoutKey(1, 2)))
  depth = common.TINY["text"]["depth"]
  sites = _sites(lines)
  txt = {E.dropout_site(1, layer, k) for layer in range(depth) for k in (E.DROP_ATTN, E.DROP_GELU, E.DROP_MLP)}
  img = {E.dropout_site(0, 0, E.DROP_EMBED)} | {E.dropout_site(0, layer, k) for layer in range(depth)
                                                for k in (E.DROP_ATTN, E.DROP_GELU, E.DROP_MLP)}
  assert set(sites) == txt | img and not txt & img
  assert "rate=0.20000000298023224" in " ".join(lines) and "rate=0.10000000149011612" in " ".join(lines)
