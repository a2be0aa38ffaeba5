"""CPU: the C-ABI library builds, loads and exports every symbol include/bv_*.h declare, the binding and
the header constants match the headers, the build compiles every source and hashes every header, the C
compiler agrees with every ctypes prototype and argument struct of the binding, each header is plain C that
a C program can link against, and argument validation fails loudly (no compute without a GPU)."""
import ctypes
import os
import re

import pytest

from big_vision_b200 import lib as L
from common import HEADERS, ROOT, header_functions, run_c


def _declared():
  return set().union(*(header_functions(h) for h in HEADERS))


def test_header_symbols_exported():
  lib = L.load()
  names = _declared()
  assert len(names) >= 50
  for n in names:
    assert hasattr(lib, n), f"{n} declared in include/ but not exported"


def test_binding_covers_every_header():
  """The entry points are defined across the kernel sources, so the headers together must match the one
  binding table one to one, and the loaded library must carry its argtypes."""
  declared = _declared() - {"bv_last_error_string"}
  assert declared == set(L.SIGNATURES), declared ^ set(L.SIGNATURES)
  lib = L.load()
  for name, argtypes in L.SIGNATURES.items():
    assert tuple(getattr(lib, name).argtypes) == tuple(argtypes), name


def test_the_build_compiles_every_source_and_hashes_every_header():
  from big_vision_b200 import build
  assert set(HEADERS) <= set(build._headers())   # pylint: disable=protected-access
  assert {f for f in os.listdir(build.CSRC) if f.endswith(".cu")} <= set(build.SOURCES)


def test_header_constants_equal_their_python_mirrors():
  defines = {}
  for h in HEADERS:
    defines.update((k, int(v)) for k, v in re.findall(r"#define BV_([A-Z0-9_]+)\s+(\d+)\b", open(h).read()))
  prefixed = lambda pre: {k[len(pre):].lower(): v for k, v in defines.items() if k.startswith(pre)}
  for name in ("F32", "BF16", "LOSS_WS_FLOATS", "SAM_WS_FLOATS", "ATTN_KEY_MASK", "ATTN_DROPOUT", "STEM_K",
               "STEM_K_PAD"):
    assert defines[name] == getattr(L, name), name
  # the attention flags sit above every head dim, apart from each other
  from big_vision_b200 import ops
  assert L.ATTN_KEY_MASK > max(ops.ATTN_HEAD_DIMS) and L.ATTN_KEY_MASK & 0xffff == 0
  assert L.ATTN_DROPOUT & 0xffff == 0 and L.ATTN_DROPOUT & L.ATTN_KEY_MASK == 0
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
    "bv_dropout.h": (
        '  /* a rate of 1, then site 0 */\n'
        '  unsigned short buf[64] = {0};\n'
        '  bv_dropout_key key = {1, 2, 3, 0, 1.f};\n'
        '  int a = bv_dropout(buf, 8, buf, 8, 4, 8, &key, NULL);\n'
        '  key.rate = 0.1f;\n'
        '  key.site = 0;\n'
        '  int b = bv_dropout_add(buf, 8, buf, 8, buf, 8, 4, 8, &key, NULL);\n'
        '  printf("%d %d %s\\n", a, b, bv_last_error_string());\n',
        [-1, -1], ("bv_dropout_add", "site 0")),
    "bv_conv.h": (
        '  int rc = bv_conv_fwd(NULL, NULL);\n'
        '  printf("%d %d %d %s\\n", BV_STEM_K, BV_STEM_K_PAD, rc, bv_last_error_string());\n',
        [L.STEM_K, L.STEM_K_PAD, -1], ("bv_conv_fwd", "null args")),
}


@pytest.mark.parametrize("header", [os.path.basename(h) for h in HEADERS])
def test_header_is_plain_c_and_a_c_program_links(tmp_path, header):
  """The boundary is a C ABI: each header must compile as C99 (and C++), and a C program that includes it
  links against libbv_b200.so and can call the entry points that need no GPU."""
  import subprocess
  body, ints, names = C_PROGRAMS[header]
  out = run_c(tmp_path, f'#include <stdio.h>\n#include "{header}"\nint main(void) {{\n{body}  return 0;\n}}\n',
              link=True)
  hdr = os.path.join(ROOT, "include", header)
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c", hdr], check=True)
  subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", hdr], check=True)
  fields = out.split(None, len(ints))
  assert [int(v) for v in fields[:-1]] == ints and all(name in fields[-1] for name in names), out


# ---- the C compiler against the ctypes binding ------------------------------------------------------------
# A type's kind, as both sides print it: i32, i64, u64, f32; a struct's typedef name; a pointer "p", or
# "p:<typedef>" when it points to a struct.
_KINDS = {L.c_i32: "i32", L.c_i64: "i64", ctypes.c_uint64: "u64", L.c_f32: "f32", L.c_vp: "p"}


def _c_name(struct):
  """GemmArgs -> bv_gemm_args: the typedef a ctypes.Structure of lib mirrors."""
  return "bv" + re.sub(r"[A-Z]", lambda m: "_" + m.group(0).lower(), struct.__name__)


def _kind(t):
  if issubclass(t, ctypes._Pointer):   # pylint: disable=protected-access
    return "p:" + _c_name(t._type_) if issubclass(t._type_, ctypes.Structure) else "p"
  if issubclass(t, ctypes.Structure):
    return _c_name(t)
  return _KINDS.get(t, repr(t))


def _structs():
  """Every ctypes.Structure subclass that lib defines."""
  return [v for v in vars(L).values()
          if isinstance(v, type) and issubclass(v, ctypes.Structure) and v.__module__ == L.__name__]


# put<T>() prints T's kind.  Name<T> is specialised for each mirrored struct after the headers are included,
# before main() instantiates put().
_PRELUDE = r"""#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <type_traits>
template <class T> struct Name { static constexpr const char* v = "?"; };
template <> struct Name<int32_t> { static constexpr const char* v = "i32"; };
template <> struct Name<int64_t> { static constexpr const char* v = "i64"; };
template <> struct Name<uint64_t> { static constexpr const char* v = "u64"; };
template <> struct Name<float> { static constexpr const char* v = "f32"; };
template <class T> void put() {
  using U = std::remove_cv_t<T>;
  if constexpr (std::is_pointer_v<U>) {
    using P = std::remove_cv_t<std::remove_pointer_t<U>>;
    if constexpr (std::is_class_v<P>) std::printf(" p:%s", Name<P>::v); else std::printf(" p");
  } else {
    std::printf(" %s", Name<U>::v);
  }
}
template <class F> struct Sig;
template <class R, class... A> struct Sig<R(A...)> {
  static void print(const char* name) { std::printf("%s", name); put<R>(); (put<A>(), ...); std::printf("\n"); }
};
"""


def _abi_mismatches(tmp_path, signatures, structs):
  """Compiles a C++ program that includes every header and prints, from the declarations alone (nothing is
  linked), the return and parameter kinds of each function of `signatures`, and sizeof, each member's offset
  and kind of the typedef each ctypes.Structure of `structs` mirrors.  Returns what differs from ctypes, one
  line each.  A name the headers do not declare, or a member they do not have, fails the compile."""
  src = _PRELUDE + "".join(f'#include "{os.path.basename(h)}"\n' for h in HEADERS)
  for S in structs:
    src += f'template <> struct Name<{_c_name(S)}> {{ static constexpr const char* v = "{_c_name(S)}"; }};\n'
  src += "int main() {\n" + "".join(f'  Sig<decltype({fn})>::print("{fn}");\n' for fn in signatures)
  for S in structs:
    c = _c_name(S)
    src += f'  std::printf("{c} %zu", sizeof({c}));\n'
    for f, _ in S._fields_:   # pylint: disable=protected-access
      src += f'  std::printf(" {f}@%zu", offsetof({c}, {f})); put<decltype({c}::{f})>();\n'
    src += '  std::printf("\\n");\n'
  got = dict(line.split(" ", 1) for line in run_c(tmp_path, src + "  return 0;\n}\n", cxx=True).splitlines())
  want = {fn: " ".join(_kind(t) for t in [ctypes.c_int] + list(argtypes)) for fn, argtypes in signatures.items()}
  for S in structs:
    want[_c_name(S)] = f"{ctypes.sizeof(S)} " + " ".join(
        f"{f}@{getattr(S, f).offset} {_kind(t)}" for f, t in S._fields_)   # pylint: disable=protected-access
  return [f"{k}: C has '{got[k]}', ctypes '{want[k]}'" for k in want if got[k] != want[k]]


def test_every_prototype_and_argument_struct_matches_the_headers(tmp_path):
  """ctypes cannot see the C declarations: a c_int32 bound where the header says int64_t, or a field off by
  a member, passes garbage to a kernel without any error.  So the compiler states each declaration's kinds
  and each struct's layout, and they must be those of lib.SIGNATURES and lib's structs."""
  structs = _structs()
  assert len(structs) >= 11 and len(L.SIGNATURES) >= 65
  assert _abi_mismatches(tmp_path, L.SIGNATURES, structs) == []


def test_a_planted_wrong_argtype_and_swapped_fields_are_reported(tmp_path):
  class DropoutKey(ctypes.Structure):   # seed and step swapped
    _fields_ = [("step", ctypes.c_uint64), ("seed", ctypes.c_uint64), ("site", ctypes.c_uint64),
                ("row0", L.c_i64), ("rate", L.c_f32)]

  signatures = dict(L.SIGNATURES, bv_dropout=[L.c_vp, L.c_i32] + L.SIGNATURES["bv_dropout"][2:])   # ldx
  structs = [DropoutKey if S is L.DropoutKey else S for S in _structs()]
  got = _abi_mismatches(tmp_path, signatures, structs)
  assert len(got) == 2, got
  assert got[0].startswith("bv_dropout: ") and got[1].startswith("bv_dropout_key: "), got


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
