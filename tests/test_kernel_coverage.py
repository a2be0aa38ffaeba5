"""CPU: every entry point of include/bv_*.h is named here with the GPU test(s) that check it directly
against a reference of the same operation (not only through a whole-model test, whose tolerances are far
too loose to pin one kernel).  A new ABI function without such a test, or a table row that names a test
that does not exist, fails this file on a machine without a GPU."""
import ast
import os

from common import HEADERS, ROOT, header_functions

TESTS = os.path.join(ROOT, "tests")

# entry points with nothing to compute on the device
EXEMPT = {"bv_version", "bv_device_supported", "bv_last_error_string"}

KE = "test_kernel_edges_gpu"
KG = "test_kernels_gpu"
GE = "test_gemm_elementwise_gpu"
AE = "test_attention_elementwise_gpu"
SG = "test_gsam_gpu"
DG = "test_distill_gpu"
FG = "test_flexi_gpu"
JG = "test_jet_gpu"
DR = "test_dropout_gpu"
CV = "test_conv_gpu"
COVERAGE = {
    "bv_gemm": [f"{KG}::test_dense_forward_epilogues", f"{KG}::test_dense_backward_contractions",
                "test_gemm_aux_tma_gpu::test_resid_matches_fp32_oracle",
                f"{KE}::test_gemm_gelu_epilogues_over_every_bf16_input",
                f"{KE}::test_resid_epilogue_position_embedding_periods",
                f"{GE}::test_tier1_exact", f"{GE}::test_tier2_bound", f"{GE}::test_colsum_of_the_stored_output",
                f"{GE}::test_split_k_adds_bias_once"],
    "bv_layernorm_fwd": [f"{KG}::test_layernorm", f"{KG}::test_layernorm_constant_rows_hit_the_variance_clamp"],
    "bv_layernorm_bwd": [f"{KG}::test_layernorm"],
    "bv_attention_fwd_hd": [f"{KG}::test_attention_forward_backward", "test_head_dim_gpu::test_forward_matches_fp64",
                            f"{AE}::test_zero_queries_average_every_key_once",
                            f"{AE}::test_dominant_key_gives_its_value",
                            f"{AE}::test_forward_and_backward_within_bound"],
    "bv_attention_bwd_hd": [f"{KG}::test_attention_forward_backward",
                            "test_attention_bwd_split_gpu::test_backward_matches_fp64",
                            f"{AE}::test_forward_and_backward_within_bound"],
    "bv_patchify": [f"{KG}::test_patchify_embed_pool_l2norm", f"{KE}::test_patchify_layout_and_zero_pad"],
    "bv_patchify_u8": [f"{KG}::test_patchify_u8_fuses_value_range_bit_exactly",
                       f"{KE}::test_patchify_layout_and_zero_pad"],
    "bv_embed_fwd": [f"{KE}::test_embed_fwd_and_bwd"],
    "bv_embed_bwd": [f"{KE}::test_embed_fwd_and_bwd"],
    "bv_colsum": [f"{KE}::test_colsum", f"{KE}::test_colsum_of_the_patch_embedding_view"],
    "bv_cast": [f"{KE}::test_cast_both_directions_bit_exact"],
    "bv_l2norm_fwd": [f"{KE}::test_l2norm"],
    "bv_l2norm_bwd": [f"{KE}::test_l2norm"],
    "bv_pool_fwd": [f"{KE}::test_pool_fwd_mean", f"{KE}::test_pool_token_mode_and_pool_bwd"],
    "bv_pool_bwd": [f"{KE}::test_pool_token_mode_and_pool_bwd"],
    "bv_pool_max_bwd": [f"{KG}::test_patchify_embed_pool_l2norm"],
    "bv_broadcast_row": [f"{KE}::test_broadcast_row"],
    "bv_tanh_fwd": [f"{KE}::test_standalone_gelu_and_tanh_over_every_bf16_input"],
    "bv_tanh_bwd": [f"{KE}::test_standalone_gelu_and_tanh_over_every_bf16_input"],
    "bv_gelu_fwd": [f"{KE}::test_standalone_gelu_and_tanh_over_every_bf16_input"],
    "bv_mixup": ["test_classifier_gpu::test_mixup_kernel_is_bit_exact",
                 "test_class_count_gpu::test_mixup_scalar_path_is_bit_exact"],
    "bv_axpby": [f"{KE}::test_axpby"],
    "bv_concat_cls": [f"{KE}::test_concat_and_drop_cls_bit_exact"],
    "bv_drop_cls": [f"{KE}::test_concat_and_drop_cls_bit_exact"],
    "bv_transpose_tokens": [f"{KG}::test_token_transposes_are_exact"],
    "bv_untranspose_add": [f"{KG}::test_token_transposes_are_exact"],
    "bv_row_select": [f"{KE}::test_row_select_bit_exact"],
    "bv_siglip_loss": [f"{KG}::test_siglip_loss_slab", f"{KE}::test_siglip_loss_elementwise"],
    "bv_softmax_contrastive_loss": [f"{KG}::test_softmax_contrastive_slab",
                                    f"{KE}::test_softmax_contrastive_at_batch_6144"],
    "bv_sigmoid_xent_ld": [f"{KG}::test_classification_losses", f"{KE}::test_classification_losses_wide_logits"],
    "bv_softmax_xent_ld": [f"{KG}::test_classification_losses", f"{KE}::test_classification_losses_wide_logits"],
    "bv_adam_step": [f"{KG}::test_adam_matches_optax_chain", f"{KE}::test_adam_step_state_and_norms"],
    "bv_sumsq": [f"{KE}::test_sumsq"],
    "bv_scale_step": [f"{KE}::test_scale_step_state_and_norms"],
    "bv_adafactor_step": ["test_optax_gpu::test_adafactor_matches_oracle"],
    "bv_top1": ["test_eval_paths::test_top1_matches_oracle", "test_eval_paths::test_top1_nan_and_zero_shot"],
    "bv_retrieval_ranks": ["test_eval_paths::test_retrieval_ranks_match_stable_argsort",
                           "test_eval_paths::test_retrieval_golden_on_device"],
    # include/bv_b200_sam.h
    "bv_sam_perturb": [f"{SG}::test_sam_perturb_elementwise"],
    "bv_sam_dots": [f"{SG}::test_sam_dots_elementwise", f"{SG}::test_sam_dots_bit_identical_across_runs"],
    "bv_gsam_combine": [f"{SG}::test_gsam_combine_elementwise", f"{SG}::test_gsam_combine_zero_robust_gradient_is_nan"],
    # include/bv_b200_distill.h
    "bv_distill_loss": [f"{DG}::test_distill_loss_elementwise", f"{DG}::test_distill_loss_scalar_path_and_accumulate",
                        f"{DG}::test_distill_loss_extreme_logits_and_clip",
                        f"{DG}::test_distill_loss_bit_identical_across_runs"],
    "bv_distance": [f"{DG}::test_distance_every_kind", f"{DG}::test_distance_agree_is_exact_on_ties"],
    # include/bv_b200_flexi.h
    "bv_resample_fwd": [f"{FG}::test_resample_fwd_elementwise", f"{FG}::test_resample_bit_identical_across_runs",
                        f"{FG}::test_resample_refusals"],
    "bv_resample_bwd": [f"{FG}::test_resample_bwd_elementwise", f"{FG}::test_resample_bit_identical_across_runs",
                        f"{FG}::test_resample_refusals"],
    # include/bv_b200_jet.h
    "bv_jet_dequantize_patchify": [f"{JG}::test_dequantize_patchify_is_numpy_bit_for_bit",
                                   f"{JG}::test_noise_of_a_global_batch_does_not_depend_on_the_rank_count",
                                   f"{JG}::test_refusals"],
    "bv_jet_unpatchify": [f"{JG}::test_unpatchify_and_plain_patchify_are_exact", f"{JG}::test_refusals"],
    "bv_jet_split": [f"{JG}::test_split_and_merge_grad_are_exact", f"{JG}::test_refusals"],
    "bv_jet_coupling_fwd": [f"{JG}::test_coupling_fwd_elementwise",
                            f"{JG}::test_logdet_and_bits_are_bit_identical_across_runs",
                            f"{JG}::test_extreme_raw_scales_stay_finite", f"{JG}::test_refusals"],
    "bv_jet_coupling_bwd": [f"{JG}::test_coupling_bwd_elementwise", f"{JG}::test_extreme_raw_scales_stay_finite"],
    "bv_jet_merge_grad": [f"{JG}::test_split_and_merge_grad_are_exact"],
    "bv_jet_bits": [f"{JG}::test_bits_elementwise", f"{JG}::test_logdet_and_bits_are_bit_identical_across_runs"],
    # include/bv_dropout.h
    "bv_dropout": [f"{DR}::test_dropout_is_numpy_bit_for_bit", f"{DR}::test_column_sums_match_fp64_and_runs_repeat",
                   f"{DR}::test_realized_rate_at_b16_shapes"],
    "bv_dropout_add": [f"{DR}::test_dropout_add_is_numpy_bit_for_bit"],
    # include/bv_conv.h
    "bv_conv_fwd": [f"{CV}::test_convolutions_match_fp64"],
    "bv_conv_dgrad": [f"{CV}::test_convolutions_match_fp64"],
    "bv_conv_wgrad": [f"{CV}::test_convolutions_match_fp64"],
    "bv_weight_std_fwd": [f"{CV}::test_weight_standardisation_matches_fp64"],
    "bv_weight_std_bwd": [f"{CV}::test_weight_standardisation_matches_fp64"],
    "bv_groupnorm_fwd": [f"{CV}::test_groupnorm_relu_matches_fp64"],
    "bv_groupnorm_bwd": [f"{CV}::test_groupnorm_relu_matches_fp64"],
    "bv_maxpool_fwd": [f"{CV}::test_maxpool_forward_and_first_max_backward"],
    "bv_maxpool_bwd": [f"{CV}::test_maxpool_forward_and_first_max_backward"],
    "bv_stem_im2col": [f"{CV}::test_stem_convolution_matches_fp64"],
}
# entry points whose op is reached through another ops function of the same family
VIA = {"bv_stem_im2col": "ops.stem_conv_fwd("}


def _is_gpu_mark(dec):
  """`pytest.mark.gpu` (bare or called)."""
  if isinstance(dec, ast.Call):
    dec = dec.func
  return isinstance(dec, ast.Attribute) and dec.attr == "gpu"


def _gpu_tests():
  """module::name -> source of every top-level test function in tests/ that is marked gpu, by its module's
  pytestmark or by its own decorator."""
  out = {}
  for fn in sorted(os.listdir(TESTS)):
    mod, ext = os.path.splitext(fn)
    if ext != ".py" or not mod.startswith("test_"):
      continue
    tree = ast.parse(open(os.path.join(TESTS, fn)).read())
    gpu_module = any(isinstance(n, ast.Assign) and any(getattr(t, "id", "") == "pytestmark" for t in n.targets)
                     and _is_gpu_mark(n.value) for n in tree.body)
    for node in tree.body:
      if isinstance(node, ast.FunctionDef) and node.name.startswith("test_") and (
          gpu_module or any(_is_gpu_mark(d) for d in node.decorator_list)):
        out[f"{mod}::{node.name}"] = ast.unparse(node)
  return out


def test_table_keys_are_exactly_the_header_entry_points():
  declared = set().union(*(header_functions(h) for h in HEADERS)) - EXEMPT
  assert len(declared) >= 50
  missing, extra = declared - set(COVERAGE), set(COVERAGE) - declared
  assert not missing, f"entry points without a direct GPU test in COVERAGE: {sorted(missing)}"
  assert not extra, f"COVERAGE rows for functions the header does not declare: {sorted(extra)}"


def test_every_named_test_exists_as_a_gpu_test():
  known = _gpu_tests()
  assert len(known) > 50
  for fn, tests in COVERAGE.items():
    assert tests, fn
    for t in tests:
      assert t in known, f"{fn}: {t} is not a GPU test function in tests/"


def test_feature_header_rows_name_tests_that_call_the_op():
  """Each entry point of the feature headers (all but bv_b200.h) has one ops function of the same name (or
  the one VIA names), and every test its row names calls that function."""
  known = _gpu_tests()
  for h in HEADERS:
    if os.path.basename(h) != "bv_b200.h":
      for fn in header_functions(h):
        for t in COVERAGE[fn]:
          assert VIA.get(fn, fn.replace("bv_", "ops.", 1) + "(") in known[t], (fn, t)


def test_gemm_and_attention_rows_name_an_element_wise_test():
  """The GEMM and attention entry points are checked per element against fp64, not only against the
  tensor maximum: each of their rows names a test of the element-wise files."""
  for fn in ("bv_gemm", "bv_attention_fwd_hd", "bv_attention_bwd_hd"):
    assert any(t.split("::")[0] in (GE, AE) for t in COVERAGE[fn]), fn
