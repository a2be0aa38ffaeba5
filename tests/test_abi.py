"""CPU: the C-ABI library builds, loads and exports every symbol include/bv_b200*.h declare, the binding
and the header constants match the headers, each header is plain C that a C program can link against, and
argument validation fails loudly (no compute without a GPU)."""
import ctypes
import os
import re

import pytest

from big_vision_b200 import lib as L
from common import HEADERS, ROOT, header_functions


def _declared():
  return set().union(*(header_functions(h) for h in HEADERS))


def test_header_symbols_exported():
  lib = L.load()
  names = _declared()
  assert len(names) >= 50
  for n in names:
    assert hasattr(lib, n), f"{n} declared in include/ but not exported"


def test_binding_covers_header():
  """The entry points are defined across the kernel sources, so the headers together must match the binding
  one to one."""
  declared = _declared() - {"bv_last_error_string"}
  assert declared == set(L.SIGNATURES), declared ^ set(L.SIGNATURES)


def test_header_constants_equal_their_python_mirrors():
  defines = {}
  for h in HEADERS:
    defines.update((k, int(v)) for k, v in re.findall(r"#define BV_([A-Z0-9_]+)\s+(\d+)\b", open(h).read()))
  prefixed = lambda pre: {k[len(pre):].lower(): v for k, v in defines.items() if k.startswith(pre)}
  for name in ("F32", "BF16", "LOSS_WS_FLOATS", "SAM_WS_FLOATS"):
    assert defines[name] == getattr(L, name), name
  assert prefixed("EPI_") == {k[4:].lower(): getattr(L, k) for k in dir(L) if k.startswith("EPI_")}
  assert prefixed("DIST_") == L.DIST_KINDS
  outs = prefixed("DISTILL_")
  assert outs.pop("outputs") == len(L.DISTILL_OUTPUTS)
  assert outs == {k.replace("task_loss_", "task_"): i for i, k in enumerate(L.DISTILL_OUTPUTS)}


@pytest.mark.parametrize("name,args,message", [
    ("bv_gemm", (None, None), "bv_gemm: null args"),
    ("bv_attention_fwd_hd", (None, 96, None), "bv_attention_fwd_hd: null args"),
    ("bv_attention_bwd_hd", (None, 96, None), "bv_attention_bwd_hd: null args"),
    ("bv_adam_step", (None, None), "bv_adam_step: null args"),
    ("bv_adafactor_step", (None, None), "bv_adafactor_step: null args"),
])
def test_null_struct_args_are_refused(name, args, message):
  lib = L.load()
  assert getattr(lib, name)(*args) == -1
  assert lib.bv_last_error_string().decode() == message


def test_version_and_no_gpu_support_flag():
  lib = L.load()
  assert lib.bv_version() == 101
  assert lib.bv_device_supported() in (0, 1)


def test_invalid_arguments_fail_loudly():
  lib = L.load()
  args = L.GemmArgs(M=0, N=8, K=8)
  rc = lib.bv_gemm(ctypes.byref(args), None)
  assert rc == -1
  assert b"empty" in lib.bv_last_error_string()
  args = L.GemmArgs(M=8, N=8, K=8, ldd=12, out_dtype=L.BF16)   # bf16 row stride not 16B-aligned
  assert lib.bv_gemm(ctypes.byref(args), None) == -1
  with pytest.raises(L.BvError):
    L.call("bv_layernorm_fwd", None, 1, None, None, None, 1, None, None, 4, 12, 1e-6, None)


def test_ops_refuse_cpu_tensors():
  import torch
  from big_vision_b200 import ops
  with pytest.raises(L.BvError):
    ops.layernorm_fwd(torch.zeros(4, 64), torch.ones(64), torch.zeros(64))


def test_bench_workloads_cover_the_five_baseline_configs():
  """bench.py --workload: one entry per BASELINE.json config, synthetic batches of the SURVEY 8d shapes."""
  import importlib.util
  import json
  import os
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  spec = importlib.util.spec_from_file_location("bench", os.path.join(root, "bench.py"))
  bench = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(bench)
  assert len(json.load(open(os.path.join(root, "BASELINE.json")))["configs"]) == len(bench.WORKLOADS) == 5
  wl = bench.WORKLOADS["siglip_b16"]
  b = bench.synthetic_batch(wl, 4, seed=0)
  assert b["image"].shape == (4, 224, 224, 3) and b["image"].dtype.name == "float32"
  assert -1.0 <= b["image"].min() and b["image"].max() < 1.0
  assert b["labels"].shape == (4, 64) and b["labels"].dtype.name == "int32" and (b["labels"][:, -1] == 1).all()
  assert bench.synthetic_batch(wl, 2, seed=0, uint8=True)["image"].dtype.name == "uint8"
  c = bench.synthetic_batch(bench.WORKLOADS["vit_b16_cls"], 4, seed=0)
  assert c["labels"].shape == (4, 1000) and (c["labels"].sum(1) == 1).all()
  assert bench.WORKLOADS["siglip_l14_336"]["per_gpu_batch"] * 8 == 4096 and wl["per_gpu_batch"] * 8 == 6144
  model = bench.build_model(bench.WORKLOADS["siglip_l14_336"])
  assert model.img.scan and model.txt.scan and model.img.width == 1024 and model.img.patch_size == (14, 14)


# header -> (body of the main() of a C program that calls entry points refused before any launch, the integers
# it prints, the names in the error strings it prints after them)
C_PROGRAMS = {
    "bv_b200.h": (
        '  /* 7 columns; the losses without their workspace */\n'
        '  char e[2][512];\n'
        '  int a = bv_colsum(NULL, 1, NULL, 4, 7, 7, NULL);\n'
        '  snprintf(e[0], sizeof e[0], "%s", bv_last_error_string());\n'
        '  int b = bv_siglip_loss(NULL, 1, 4, 4, 0, NULL, NULL, 4, NULL, 4, NULL, NULL, NULL, NULL, NULL);\n'
        '  snprintf(e[1], sizeof e[1], "%s", bv_last_error_string());\n'
        '  int c = bv_sigmoid_xent_ld(NULL, 8, NULL, 8, NULL, NULL, 8, NULL, 2, 8, NULL);\n'
        '  printf("%d %d %d %d %s %s %s\\n", bv_version(), a, b, c, e[0], e[1], bv_last_error_string());\n',
        [101, -1, -1, -1], ("bv_colsum", "bv_siglip_loss", "bv_sigmoid_xent_ld")),
    "bv_b200_sam.h": (
        '  int rc = bv_sam_dots(NULL, NULL, NULL, NULL, 8, NULL);\n'
        '  printf("%d %d %s\\n", BV_SAM_WS_FLOATS, rc, bv_last_error_string());\n',
        [L.SAM_WS_FLOATS, -1], ("bv_sam_dots",)),
    "bv_b200_distill.h": (
        '  /* a distance without a training kernel, a stride < C */\n'
        '  int a = bv_distill_loss(NULL, 8, NULL, 8, NULL, 0, BV_DIST_L2, 1.f, 0.f, 0, NULL, 0, NULL, NULL, 4, 8,'
        ' NULL);\n'
        '  int b = bv_distance(NULL, 4, NULL, 8, BV_DIST_AGREE, 0.f, 1.f, 0.f, 1, NULL, 4, 8, NULL);\n'
        '  printf("%d %d %d %s\\n", BV_DISTILL_OUTPUTS, a, b, bv_last_error_string());\n',
        [len(L.DISTILL_OUTPUTS), -3, -1], ("bv_distance",)),
    "bv_b200_flexi.h": (
        '  /* J not a multiple of 4, a null matrix */\n'
        '  float m = 1.f;\n'
        '  int a = bv_resample_fwd(&m, &m, &m, 1, 1, 6, NULL);\n'
        '  int b = bv_resample_bwd(NULL, &m, &m, 1, 1, 4, NULL);\n'
        '  printf("%d %d %s\\n", a, b, bv_last_error_string());\n',
        [-1, -1], ("bv_resample_bwd",)),
    "bv_b200_jet.h": (
        '  /* H not a multiple of ps, a null buffer */\n'
        '  float m = 1.f;\n'
        '  int a = bv_jet_unpatchify(&m, &m, 1, 6, 8, 3, 4, NULL);\n'
        '  int b = bv_jet_bits(&m, NULL, &m, &m, NULL, 1.f, 1, 1, NULL);\n'
        '  printf("%d %d %s\\n", a, b, bv_last_error_string());\n',
        [-1, -1], ("bv_jet_bits",)),
}


@pytest.mark.parametrize("header", [os.path.basename(h) for h in HEADERS])
def test_header_is_plain_c_and_a_c_program_links(tmp_path, header):
  """The boundary is a C ABI: each header must compile as C99 (and C++), and a C program that includes it
  links against libbv_b200.so and can call the entry points that need no GPU."""
  import shutil
  import subprocess
  if shutil.which("gcc") is None:
    pytest.skip("no gcc")
  L.load()
  hdr = os.path.join(ROOT, "include", header)
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c", hdr], check=True)
  subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", hdr], check=True)
  body, ints, names = C_PROGRAMS[header]
  src = tmp_path / "main.c"
  src.write_text(f'#include <stdio.h>\n#include "{header}"\nint main(void) {{\n{body}  return 0;\n}}\n')
  libdir = os.path.dirname(os.path.abspath(L.LIB_PATH))
  exe = tmp_path / "main"
  subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                  "-L", libdir, "-lbv_b200", f"-Wl,-rpath,{libdir}"], check=True)
  out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
  fields = out.split(None, len(ints))
  assert [int(v) for v in fields[:-1]] == ints and all(name in fields[-1] for name in names), out


def test_bench_refuses_to_run_the_product_arm_without_a_gpu():
  """No CPU fallback: the product arm of bench.py exits non-zero on a box without a GPU instead of timing
  something else (the reference arm is the only thing that may run on the host cores)."""
  import subprocess
  import sys
  import torch
  if torch.cuda.is_available():
    pytest.skip("a GPU is present")
  r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "1",
                      "--no-cpu-baseline", "--no-gpu-baseline"], capture_output=True, text=True, timeout=600)
  assert r.returncode != 0 and r.stdout.strip() == "" and "needs a GPU" in r.stderr


def test_reference_arm_prints_the_contract_line():
  """`bench.py --impl reference`: the oracle port on the host cores, one JSON line with the same metric /
  unit / config keys as the product arm plus impl, cpu_baseline and an e2e block with zero copies."""
  import json
  import subprocess
  import sys
  r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                      "--warmup", "1"], capture_output=True, text=True, timeout=900)
  assert r.returncode == 0, r.stderr[-2000:]
  line = json.loads(r.stdout.strip().splitlines()[-1])
  assert line["impl"] == "reference" and line["metric"] == "siglip_vit_b16_pairs_per_sec" and line["unit"] == "pairs/s"
  assert line["higher_is_better"] is True and line["steps"] == 1 and line["value"] > 0
  assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["value"] == line["value"]
  assert line["cpu_baseline"]["cores"] >= 1 and "sample" in line["cpu_baseline"]
  assert line["e2e"] == {"value": line["value"], "unit": "pairs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
  assert "workload" in line["config"] and "model" not in line["config"]
