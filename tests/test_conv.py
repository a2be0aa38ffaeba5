"""CPU: every refusal of the C ABI of include/bv_conv.h (the BiT ResNet-v2 kernels) returned before any CUDA
call.  The header's binding, coverage table, layout and C program are checked with the other headers' in
tests/test_abi.py and tests/test_kernel_coverage.py."""
from common import run_c

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


def test_every_refusal_returns_invalid_before_any_cuda_call(tmp_path):
  """Host pointers stand in for device ones: a call that got past its checks would fault or fail in CUDA, so
  -1 with the named message shows the refusal came first."""
  body = "  static double buf[64];\n  int rc;\n  bv_conv_args a;\n"
  for stmt, _ in REFUSALS:
    body += ("  { bv_conv_args d = {buf, buf, buf, buf, buf, (float*)buf, NULL, buf, 2, 8, 8, 64, 64, 3, 1, 0};"
             f" a = d; }}\n  {stmt}\n  printf(\"%d|%s\\n\", rc, bv_last_error_string());\n")
  src = '#include <stdio.h>\n#include "bv_conv.h"\nint main(void) {\n' + body + "  return 0;\n}\n"
  lines = run_c(tmp_path, src, link=True).strip().split("\n")
  assert len(lines) == len(REFUSALS)
  for (stmt, phrase), line in zip(REFUSALS, lines):
    rc, msg = line.split("|", 1)
    assert int(rc) == -1 and phrase in msg, (stmt, line)
