"""CPU: the C ABI of include/bv_conv.h (the BiT ResNet-v2 kernels): its functions exported and bound one to
one, each named with the GPU tests that call its ops function, the argument struct's layout against a C
program, and every refusal returned before any CUDA call."""
import ast
import ctypes
import os
import shutil
import subprocess

import pytest

from common import header_functions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "bv_conv.h")

# entry point -> the GPU tests of tests/test_conv_gpu.py that check it against float64
COVERAGE = {
    "bv_conv_fwd": ["test_convolutions_match_fp64"],
    "bv_conv_dgrad": ["test_convolutions_match_fp64"],
    "bv_conv_wgrad": ["test_convolutions_match_fp64"],
    "bv_weight_std_fwd": ["test_weight_standardisation_matches_fp64"],
    "bv_weight_std_bwd": ["test_weight_standardisation_matches_fp64"],
    "bv_groupnorm_fwd": ["test_groupnorm_relu_matches_fp64"],
    "bv_groupnorm_bwd": ["test_groupnorm_relu_matches_fp64"],
    "bv_maxpool_fwd": ["test_maxpool_forward_and_first_max_backward"],
    "bv_maxpool_bwd": ["test_maxpool_forward_and_first_max_backward"],
    "bv_stem_im2col": ["test_stem_convolution_matches_fp64"],
}
# ops functions that reach an entry point through a helper of the same family
VIA = {"bv_stem_im2col": "ops.stem_conv_fwd("}


def test_header_functions_are_exported_and_bound_one_to_one():
  from big_vision_b200 import lib as L
  declared = header_functions(HEADER)
  assert declared == set(L.CONV_SIGNATURES) == set(COVERAGE)
  assert not declared & (set(L.SIGNATURES) | set(L.DROPOUT_SIGNATURES))
  lib = L.load()
  for name in declared:
    assert tuple(getattr(lib, name).argtypes) == tuple(L.CONV_SIGNATURES[name])


def test_every_entry_point_has_gpu_tests_that_call_its_op():
  tree = ast.parse(open(os.path.join(ROOT, "tests", "test_conv_gpu.py")).read())
  assert any(isinstance(n, ast.Assign) and any(getattr(t, "id", "") == "pytestmark" for t in n.targets)
             and ast.unparse(n.value) == "pytest.mark.gpu" for n in tree.body)
  tests = {n.name: ast.unparse(n) for n in tree.body if isinstance(n, ast.FunctionDef) and n.name.startswith("test_")}
  for fn, names in COVERAGE.items():
    for t in names:
      assert t in tests, (fn, t)
      assert VIA.get(fn, fn.replace("bv_", "ops.", 1) + "(") in tests[t], (fn, t)


def test_the_build_hashes_the_header():
  from big_vision_b200 import build
  assert HEADER in build._headers()
  assert "conv.cu" in build.SOURCES


def _c_program(tmp_path, body):
  from big_vision_b200 import lib as L
  L.load()
  src = tmp_path / "main.c"
  src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "bv_conv.h"\nint main(void) {\n' + body +
                 "  return 0;\n}\n")
  libdir = os.path.dirname(os.path.abspath(L.LIB_PATH))
  exe = tmp_path / "main"
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                  str(exe), "-L", libdir, "-lbv_b200", f"-Wl,-rpath,{libdir}"], check=True)
  return subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no gcc")
def test_header_is_plain_c_and_the_struct_layout_matches(tmp_path):
  from big_vision_b200 import lib as L
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c", HEADER], check=True)
  subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", HEADER], check=True)
  fields = [f for f, _ in L.ConvArgs._fields_]
  body = "".join(f'  printf("%zu ", offsetof(bv_conv_args, {f}));\n' for f in fields)
  body += '  printf("%zu %d %d\\n", sizeof(bv_conv_args), BV_STEM_K, BV_STEM_K_PAD);\n'
  got = [int(v) for v in _c_program(tmp_path, body).split()]
  assert got[:-3] == [getattr(L.ConvArgs, f).offset for f in fields]
  assert got[-3:] == [ctypes.sizeof(L.ConvArgs), L.STEM_K, L.STEM_K_PAD]


# each refusal: a C statement that returns the code into rc, and a phrase of its message
REFUSALS = [
    ("rc = bv_conv_fwd(NULL, NULL);", "null args"),
    ("a.k = 5; rc = bv_conv_fwd(&a, NULL);", "k = 5"),
    ("a.stride = 3; rc = bv_conv_dgrad(&a, NULL);", "stride 3"),
    ("a.cin = 96; rc = bv_conv_wgrad(&a, NULL);", "multiples of 64"),
    ("a.cout = 0; rc = bv_conv_fwd(&a, NULL);", "multiples of 64"),
    ("a.h = 0; rc = bv_conv_fwd(&a, NULL);", "h, w <= 32767"),
    ("a.w = 40000; rc = bv_conv_fwd(&a, NULL);", "h, w <= 32767"),
    ("a.n = 0; rc = bv_conv_fwd(&a, NULL);", "n >= 1"),
    ("a.n = 1 << 30; rc = bv_conv_fwd(&a, NULL);", "too large"),
    ("a.x = NULL; rc = bv_conv_fwd(&a, NULL);", "null x"),
    ("a.y = (char*)buf + 2; rc = bv_conv_fwd(&a, NULL);", "y must be 16-byte aligned"),
    ("a.resid = (char*)buf + 8; rc = bv_conv_fwd(&a, NULL);", "resid must be 16-byte aligned"),
    ("a.kernel = NULL; rc = bv_conv_dgrad(&a, NULL);", "null kernel"),
    ("a.stride = 2; a.workspace = NULL; rc = bv_conv_dgrad(&a, NULL);", "null workspace"),
    ("a.dy = NULL; rc = bv_conv_wgrad(&a, NULL);", "null dy"),
    ("a.dkernel = NULL; rc = bv_conv_wgrad(&a, NULL);", "null dkernel"),
    ("rc = bv_weight_std_fwd(NULL, 9, 64, buf, (float*)buf, (float*)buf, NULL);", "null pointer"),
    ("rc = bv_weight_std_fwd((float*)buf, 0, 64, buf, (float*)buf, (float*)buf, NULL);", "rows, cout >= 1"),
    ("rc = bv_weight_std_bwd((float*)buf, (float*)buf, (float*)buf, (float*)buf, 9, 0, (float*)buf, NULL);",
     "rows, cout >= 1"),
    ("rc = bv_groupnorm_fwd(buf, (float*)buf, (float*)buf, buf, (float*)buf, (float*)buf, 1, 4, 48, 1, NULL);",
     "multiple of 32"),
    ("rc = bv_groupnorm_fwd(buf, (float*)buf, (float*)buf, buf, (float*)buf, NULL, 1, 4, 64, 1, NULL);",
     "null pointer"),
    ("rc = bv_groupnorm_bwd(buf, buf, (float*)buf, (float*)buf, (float*)buf, (float*)buf, NULL, buf, (float*)buf,"
     " (float*)buf, 0, 4, 64, 1, NULL);", "n <= 65535"),
    ("rc = bv_groupnorm_bwd(buf, buf, (float*)buf, (float*)buf, (float*)buf, (float*)buf, NULL, buf, NULL,"
     " (float*)buf, 1, 4, 64, 1, NULL);", "null pointer"),
    ("rc = bv_maxpool_fwd(buf, buf, 1, 0, 4, 8, NULL);", "n, h, w, c >= 1"),
    ("rc = bv_maxpool_bwd(buf, NULL, buf, 1, 4, 4, 8, NULL);", "null pointer"),
    ("rc = bv_stem_im2col((float*)buf, buf, 1, 4, 0, NULL);", "n, h, w >= 1"),
    ("rc = bv_stem_im2col(NULL, buf, 1, 4, 4, NULL);", "null pointer"),
]


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no gcc")
def test_every_refusal_returns_invalid_before_any_cuda_call(tmp_path):
  """Host pointers stand in for device ones: a call that got past its checks would fault or fail in CUDA, so
  -1 with the named message shows the refusal came first."""
  body = "  static double buf[64];\n  int rc;\n  bv_conv_args a;\n"
  for stmt, _ in REFUSALS:
    body += ("  { bv_conv_args d = {buf, buf, buf, buf, buf, (float*)buf, NULL, buf, 2, 8, 8, 64, 64, 3, 1, 0};"
             f" a = d; }}\n  {stmt}\n  printf(\"%d|%s\\n\", rc, bv_last_error_string());\n")
  lines = _c_program(tmp_path, body).strip().split("\n")
  assert len(lines) == len(REFUSALS)
  for (stmt, phrase), line in zip(REFUSALS, lines):
    rc, msg = line.split("|", 1)
    assert int(rc) == -1 and phrase in msg, (stmt, line)
