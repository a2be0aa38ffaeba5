"""CPU: the key-masked attention arguments.  The unmasked arguments still end in `scale`, and the
BV_ATTN_KEY_MASK flag is refused at head dims other than 64 and with a NULL mask, before any CUDA call.
The masked structs' layout and the flag's mirror are checked with the other headers' in tests/test_abi.py."""
import ctypes

import pytest


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
  """The masked structs append to bv_attn_args; the flag's mirror is checked with the other header
  constants in tests/test_abi.py."""
  from big_vision_b200 import lib as L
  assert [f[0] for f in L.AttnArgs._fields_][-1] == "scale"
