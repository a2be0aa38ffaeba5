"""ctypes binding of libbv_b200.so (C ABI declared in include/bv_b200*.h, include/bv_dropout.h and
include/bv_conv.h).

The product path has no fallback: if the library is missing, or a call is made
without a compute-capability-9.x device, this module raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# BV_LIB_PATH selects an experimental build of the same sources (tools / A-B measurements only)
LIB_PATH = os.environ.get("BV_LIB_PATH") or os.path.join(_HERE, "libbv_b200.so")

c_i32, c_i64, c_f32, c_vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p

# the #defines of include/bv_b200*.h that Python needs
F32, BF16 = 0, 1
EPI_NONE, EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_RESID, EPI_DGELU, EPI_BIAS_GELU_ACT = 0, 1, 2, 3, 4, 5
LOSS_WS_FLOATS = 8192      # BV_LOSS_WS_FLOATS
SAM_WS_FLOATS = 2048       # BV_SAM_WS_FLOATS
# BV_DIST_*: the kinds of dist(); BV_DISTILL_*: the outputs of bv_distill_loss, in order
DIST_KINDS = {"euclidean": 0, "l2": 1, "hard": 2, "kl": 3, "logsoftmax_euclidean": 4, "agree": 5}
ATTN_KEY_MASK = 65536      # BV_ATTN_KEY_MASK: head_dim flag of a key-masked attention call
ATTN_DROPOUT = 131072      # BV_ATTN_DROPOUT (include/bv_dropout.h): head_dim flag of attention-probability dropout
DISTILL_OUTPUTS = ("distance", "entropy_student", "entropy_teacher", "task_loss_student", "task_loss_teacher")


class GemmArgs(ctypes.Structure):
  _fields_ = [("A", c_vp), ("B", c_vp), ("D", c_vp), ("D2", c_vp), ("bias", c_vp), ("aux", c_vp),
              ("colsum", c_vp), ("M", c_i64), ("N", c_i64), ("K", c_i64),
              ("lda", c_i64), ("ldb", c_i64), ("ldd", c_i64), ("ldd2", c_i64), ("ldaux", c_i64),
              ("a_mn", c_i32), ("b_mn", c_i32),
              ("epilogue", c_i32), ("out_dtype", c_i32), ("reduce_out", c_i32), ("splits", c_i32),
              ("block_n", c_i32), ("aux_row_mod", c_i32), ("alpha", c_f32)]


class AttnArgs(ctypes.Structure):
  _fields_ = [("q", c_vp), ("k", c_vp), ("v", c_vp), ("o", c_vp), ("lse", c_vp),
              ("B", c_i64), ("H", c_i32), ("Nq", c_i32), ("Nk", c_i32),
              ("ldq", c_i64), ("ldk", c_i64), ("ldv", c_i64), ("ldo", c_i64),
              ("bsq", c_i64), ("bsk", c_i64), ("bsv", c_i64), ("bso", c_i64),
              ("scale", c_f32)]


class AttnBwdArgs(ctypes.Structure):
  _fields_ = [("fwd", AttnArgs), ("d_o", c_vp), ("lddo", c_i64), ("bsdo", c_i64),
              ("dq", c_vp), ("dk", c_vp), ("dv", c_vp),
              ("lddq", c_i64), ("lddk", c_i64), ("lddv", c_i64),
              ("bsdq", c_i64), ("bsdk", c_i64), ("bsdv", c_i64),
              ("dq_colsum", c_vp), ("dk_colsum", c_vp), ("dv_colsum", c_vp),
              ("delta", c_vp)]


# head_dim | ATTN_KEY_MASK: the attention arguments are the first member of one of these
class AttnMaskedArgs(ctypes.Structure):
  _fields_ = [("attn", AttnArgs), ("key_mask", c_vp), ("bsmask", c_i64)]


class AttnMaskedBwdArgs(ctypes.Structure):
  _fields_ = [("attn", AttnBwdArgs), ("key_mask", c_vp), ("bsmask", c_i64)]


class DropoutKey(ctypes.Structure):
  _fields_ = [("seed", ctypes.c_uint64), ("step", ctypes.c_uint64), ("site", ctypes.c_uint64), ("row0", c_i64),
              ("rate", c_f32)]


# head_dim | ATTN_KEY_MASK | ATTN_DROPOUT: the masked arguments are the first member of one of these
class AttnDropoutArgs(ctypes.Structure):
  _fields_ = [("masked", AttnMaskedArgs), ("drop", DropoutKey)]


class AttnDropoutBwdArgs(ctypes.Structure):
  _fields_ = [("masked", AttnMaskedBwdArgs), ("drop", DropoutKey)]


# include/bv_conv.h
STEM_K, STEM_K_PAD = 147, 152   # BV_STEM_K, BV_STEM_K_PAD


class ConvArgs(ctypes.Structure):
  _fields_ = [("x", c_vp), ("kernel", c_vp), ("dy", c_vp), ("y", c_vp), ("dx", c_vp), ("dkernel", c_vp),
              ("resid", c_vp), ("workspace", c_vp), ("n", c_i64),
              ("h", c_i32), ("w", c_i32), ("cin", c_i32), ("cout", c_i32), ("k", c_i32), ("stride", c_i32),
              ("accumulate", c_i32)]


class AdamArgs(ctypes.Structure):
  _fields_ = [("params", c_vp), ("grads", c_vp), ("mu", c_vp), ("nu", c_vp), ("params_bf16", c_vp),
              ("n", c_i64), ("mu_dtype", c_i32),
              ("lr_eff", c_f32), ("b1", c_f32), ("b2", c_f32), ("eps", c_f32), ("wd_eff", c_f32),
              ("grad_mult", c_f32), ("clip_norm", c_f32),
              ("gnorm_sq", c_vp), ("step", c_i64), ("upd_sq", c_vp), ("param_sq", c_vp)]


class AdafactorArgs(ctypes.Structure):
  _fields_ = [("params", c_vp), ("grads", c_vp), ("params_bf16", c_vp),
              ("A", c_i64), ("L", c_i64), ("M", c_i64), ("H", c_i64), ("sA", c_i64), ("sL", c_i64), ("sM", c_i64),
              ("mode", c_i32),
              ("vfull", c_vp), ("red_h", c_vp), ("red_l", c_vp), ("nrm", c_vp), ("momentum", c_vp),
              ("decay", c_f32), ("eps", c_f32), ("beta", c_f32), ("lr_eff", c_f32), ("wd_eff", c_f32),
              ("grad_mult", c_f32), ("clip_norm", c_f32),
              ("gnorm_sq", c_vp), ("upd_sq", c_vp), ("param_sq", c_vp)]


# name -> argtypes (restype is int).  Mirrors the functions of include/bv_b200*.h one to one, all exported
# from the same library.
SIGNATURES = {
    # include/bv_b200.h
    "bv_gemm": [ctypes.POINTER(GemmArgs), c_vp],
    "bv_layernorm_fwd": [c_vp, c_i32, c_vp, c_vp, c_vp, c_i32, c_vp, c_vp, c_i64, c_i32, c_f32, c_vp],
    "bv_layernorm_bwd": [c_vp, c_i32, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_vp, c_vp,
                         c_vp, c_i64, c_i32, c_vp],
    "bv_attention_fwd_hd": [ctypes.POINTER(AttnArgs), c_i32, c_vp],
    "bv_attention_bwd_hd": [ctypes.POINTER(AttnBwdArgs), c_i32, c_vp],
    "bv_patchify": [c_vp, c_vp, c_i64, c_i32, c_i32, c_i32, c_i32, c_vp],
    "bv_patchify_u8": [c_vp, c_vp, c_i64, c_i32, c_i32, c_i32, c_i32, c_f32, c_f32, c_f32, c_f32, c_i32, c_vp],
    "bv_embed_fwd": [c_vp, c_vp, c_vp, c_vp, c_i32, c_i64, c_i32, c_i32, c_i32, c_vp],
    "bv_embed_bwd": [c_vp, c_vp, c_i32, c_vp, c_vp, c_i64, c_i32, c_i32, c_i32, c_vp],
    "bv_colsum": [c_vp, c_i32, c_vp, c_i64, c_i64, c_i64, c_vp],
    "bv_cast": [c_vp, c_i32, c_vp, c_i32, c_i64, c_vp],
    "bv_l2norm_fwd": [c_vp, c_i32, c_vp, c_vp, c_i64, c_i32, c_f32, c_vp],
    "bv_l2norm_bwd": [c_vp, c_vp, c_vp, c_vp, c_i32, c_i64, c_i32, c_f32, c_vp],
    "bv_pool_fwd": [c_vp, c_i32, c_vp, c_i32, c_i64, c_i32, c_i32, c_i32, c_i32, c_vp],
    "bv_pool_bwd": [c_vp, c_i32, c_vp, c_i32, c_i64, c_i32, c_i32, c_i32, c_i32, c_vp],
    "bv_pool_max_bwd": [c_vp, c_i32, c_vp, c_i32, c_vp, c_i32, c_i64, c_i32, c_i32, c_vp],
    "bv_broadcast_row": [c_vp, c_i32, c_vp, c_vp, c_i32, c_i64, c_i32, c_vp],
    "bv_tanh_fwd": [c_vp, c_vp, c_i32, c_i64, c_vp],
    "bv_tanh_bwd": [c_vp, c_vp, c_vp, c_i32, c_i64, c_vp],
    "bv_gelu_fwd": [c_vp, c_vp, c_i32, c_i64, c_vp],
    "bv_mixup": [c_vp, c_vp, c_i64, c_i64, c_f32, c_vp],
    "bv_axpby": [c_vp, c_vp, c_vp, c_i32, c_f32, c_f32, c_i64, c_vp],
    "bv_transpose_tokens": [c_vp, c_vp, c_i64, c_i32, c_i32, c_vp],
    "bv_untranspose_add": [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp],
    "bv_row_select": [c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp],
    "bv_concat_cls": [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp],
    "bv_drop_cls": [c_vp, c_vp, c_i64, c_i32, c_i32, c_vp],
    "bv_siglip_loss": [c_vp, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp,
                       c_vp, c_vp, c_vp],
    "bv_softmax_contrastive_loss": [c_vp, c_i64, c_i64, c_i64, c_i64, c_vp, c_i64, c_f32, c_vp, c_i64, c_vp, c_vp,
                                    c_vp, c_vp, c_vp],
    "bv_sigmoid_xent_ld": [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_i64, c_i32, c_vp],
    "bv_softmax_xent_ld": [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_i64, c_i32, c_vp],
    "bv_adam_step": [ctypes.POINTER(AdamArgs), c_vp],
    "bv_sumsq": [c_vp, c_vp, c_i64, c_vp],
    "bv_adafactor_step": [ctypes.POINTER(AdafactorArgs), c_vp],
    "bv_scale_step": [c_vp, c_vp, c_vp, c_i64, c_f32, c_f32, c_f32, c_f32, c_vp, c_vp, c_vp, c_vp],
    "bv_top1": [c_vp, c_i32, c_i64, c_i32, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp],
    "bv_retrieval_ranks": [c_vp, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp],
    "bv_version": [],
    "bv_device_supported": [],
    # include/bv_b200_sam.h (GSAM / SAM)
    "bv_sam_perturb": [c_vp, c_vp, c_vp, c_f32, c_f32, c_i32, c_vp, c_vp, c_i64, c_vp],
    "bv_sam_dots": [c_vp, c_vp, c_vp, c_vp, c_i64, c_vp],
    "bv_gsam_combine": [c_vp, c_vp, c_vp, c_vp, c_f32, c_i32, c_i64, c_vp],
    # include/bv_b200_distill.h (distillation)
    "bv_distill_loss": [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i32, c_f32, c_f32, c_i32, c_vp, c_i64, c_vp, c_vp,
                        c_i64, c_i32, c_vp],
    "bv_distance": [c_vp, c_i64, c_vp, c_i64, c_i32, c_f32, c_f32, c_f32, c_i32, c_vp, c_i64, c_i32, c_vp],
    # include/bv_b200_flexi.h (FlexiViT resampling)
    "bv_resample_fwd": [c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp],
    "bv_resample_bwd": [c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp],
    # include/bv_b200_jet.h (Jet normalizing flow)
    "bv_jet_dequantize_patchify": [c_vp, c_vp, c_i64, c_i32, c_i32, c_i32, c_i32, ctypes.c_uint64, ctypes.c_uint64,
                                   c_i64, c_f32, c_vp],
    "bv_jet_unpatchify": [c_vp, c_vp, c_i64, c_i32, c_i32, c_i32, c_i32, c_vp],
    "bv_jet_split": [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp],
    "bv_jet_coupling_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_f32, c_i32, c_vp],
    "bv_jet_coupling_bwd": [c_vp, c_vp, c_vp, c_vp, c_f32, c_vp, c_vp, c_i64, c_i32, c_i32, c_f32, c_vp],
    "bv_jet_merge_grad": [c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp],
    "bv_jet_bits": [c_vp, c_vp, c_vp, c_vp, c_vp, c_f32, c_i64, c_i64, c_vp],
}

# The same for include/bv_dropout.h, the one header outside the bv_b200*.h set: its functions, binding and C
# link test are checked by tests/test_dropout.py rather than by the tests of the bv_b200*.h headers.
DROPOUT_SIGNATURES = {
    "bv_dropout": [c_vp, c_i64, c_vp, c_i64, c_i64, c_i64, ctypes.POINTER(DropoutKey), c_vp],
    "bv_dropout_add": [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i64, c_i64, ctypes.POINTER(DropoutKey), c_vp],
}

# include/bv_conv.h (BiT ResNet-v2), also outside the bv_b200*.h set; checked by tests/test_conv.py.
CONV_SIGNATURES = {
    "bv_conv_fwd": [ctypes.POINTER(ConvArgs), c_vp],
    "bv_conv_dgrad": [ctypes.POINTER(ConvArgs), c_vp],
    "bv_conv_wgrad": [ctypes.POINTER(ConvArgs), c_vp],
    "bv_weight_std_fwd": [c_vp, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp],
    "bv_weight_std_bwd": [c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_vp, c_vp],
    "bv_groupnorm_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i32, c_i32, c_vp],
    "bv_groupnorm_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i32, c_i32,
                         c_vp],
    "bv_maxpool_fwd": [c_vp, c_vp, c_i64, c_i32, c_i32, c_i32, c_vp],
    "bv_maxpool_bwd": [c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_i32, c_vp],
    "bv_stem_im2col": [c_vp, c_vp, c_i64, c_i32, c_i32, c_vp],
}

_lib = None


class BvError(RuntimeError):
  pass


def load():
  """Loads the shared library (once) and declares every prototype."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise BvError(
        f"{LIB_PATH} not found: build it with `python -m big_vision_b200.build` "
        "(there is no CPU or eager fallback for the kernels).")
  lib = ctypes.CDLL(LIB_PATH)
  for name, argtypes in {**SIGNATURES, **DROPOUT_SIGNATURES, **CONV_SIGNATURES}.items():
    fn = getattr(lib, name)   # raises AttributeError if the symbol is missing
    fn.argtypes = argtypes
    fn.restype = ctypes.c_int
  lib.bv_last_error_string.argtypes = []
  lib.bv_last_error_string.restype = ctypes.c_char_p
  _lib = lib
  return lib


def check(rc, what):
  if rc != 0:
    msg = load().bv_last_error_string().decode("utf-8", "replace")
    raise BvError(f"{what} failed (code {rc}): {msg}")


# kernels launched by this process through the C ABI (bench.py reports it as gpu_launches)
LAUNCHES = [0]
_LAUNCHES_PER_CALL = {"bv_attention_bwd_hd": 3, "bv_embed_bwd": 2, "bv_retrieval_ranks": 2, "bv_siglip_loss": 2,
                      "bv_sigmoid_xent_ld": 2, "bv_softmax_xent_ld": 2,
                      "bv_softmax_contrastive_loss": 2, "bv_adafactor_step": 4, "bv_sam_dots": 2,
                      "bv_distill_loss": 2, "bv_jet_bits": 2}


# optional in-situ timing of every C-ABI call (bench.py --profile-calls): list of (name, e0, e1)
PROFILE = None


def call(name, *args, tag=None):
  lib = load()
  if PROFILE is not None:
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    check(getattr(lib, name)(*args), name)
    e1.record()
    PROFILE.append((tag[0] if tag else name, e0, e1, tag[1] if tag else 0.0))
  else:
    check(getattr(lib, name)(*args), name)
  LAUNCHES[0] += _LAUNCHES_PER_CALL.get(name, 1)
