"""CPU: the key-masked attention arguments.  The ctypes mirrors of bv_attn_masked_args /
bv_attn_masked_bwd_args have the header's layout (checked against a C program), the BV_ATTN_KEY_MASK
flag is mirrored, and the flag is refused at head dims other than 64 and with a NULL mask, before any
CUDA call."""
import ctypes
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _masked_fwd(key_mask):
  from big_vision_b200 import lib as L
  return L.AttnMaskedArgs(key_mask=key_mask, bsmask=4)


@pytest.mark.parametrize("head_dim", [72, 80, 96, 104])
def test_a_mask_at_another_head_dim_is_refused(head_dim):
  from big_vision_b200 import lib as L
  lib = L.load()
  mask = (ctypes.c_uint8 * 4)(1, 1, 1, 1)
  m = _masked_fwd(ctypes.cast(mask, ctypes.c_void_p))
  assert lib.bv_attention_fwd_hd(ctypes.byref(m.attn), head_dim | L.ATTN_KEY_MASK, None) == -1
  assert b"head_dim 64 only" in lib.bv_last_error_string()
  mb = L.AttnMaskedBwdArgs(key_mask=ctypes.cast(mask, ctypes.c_void_p), bsmask=4)
  assert lib.bv_attention_bwd_hd(ctypes.byref(mb.attn), head_dim | L.ATTN_KEY_MASK, None) == -1
  assert b"bv_attention_bwd_hd" in lib.bv_last_error_string()


def test_the_flag_without_a_mask_is_refused():
  from big_vision_b200 import lib as L
  lib = L.load()
  m = _masked_fwd(None)
  assert lib.bv_attention_fwd_hd(ctypes.byref(m.attn), 64 | L.ATTN_KEY_MASK, None) == -1
  assert b"non-null key_mask" in lib.bv_last_error_string()


def test_the_unmasked_arguments_are_unchanged_and_the_flag_is_mirrored():
  from big_vision_b200 import lib as L
  assert [f[0] for f in L.AttnArgs._fields_][-1] == "scale"
  src = open(os.path.join(ROOT, "include", "bv_b200.h")).read()
  assert f"#define BV_ATTN_KEY_MASK {L.ATTN_KEY_MASK} " in src
  assert L.ATTN_KEY_MASK > max(104, 0) and L.ATTN_KEY_MASK & 0xffff == 0


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no gcc")
def test_masked_struct_layout_matches_the_header(tmp_path):
  from big_vision_b200 import lib as L
  prog = tmp_path / "layout.c"
  prog.write_text("""#include <stddef.h>
#include <stdio.h>
#include "bv_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(bv_attn_masked_args), offsetof(bv_attn_masked_args, key_mask),
         offsetof(bv_attn_masked_args, bsmask), sizeof(bv_attn_masked_bwd_args),
         offsetof(bv_attn_masked_bwd_args, key_mask), offsetof(bv_attn_masked_bwd_args, bsmask));
  return 0;
}
""")
  exe = tmp_path / "layout"
  subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
  got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
  want = [ctypes.sizeof(L.AttnMaskedArgs), L.AttnMaskedArgs.key_mask.offset, L.AttnMaskedArgs.bsmask.offset,
          ctypes.sizeof(L.AttnMaskedBwdArgs), L.AttnMaskedBwdArgs.key_mask.offset, L.AttnMaskedBwdArgs.bsmask.offset]
  assert got == want
