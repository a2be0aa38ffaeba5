"""Top-1 classification counting on the device.

Mirror of the arithmetic of big_vision/evaluators/classification.py:36-53 (`_eval_fn`):
  mask *= labels.max(axis=1); top1_idx = argmax(logits, axis=1);
  top1_correct = take_along_axis(labels, top1_idx); ncorrect = sum(top1_correct * mask);
  nseen = sum(mask)
as one kernel (`bv_top1`).  The per-example loss of the reference's `_eval_fn` is not computed here.
"""
from big_vision_b200 import ops


def top1_counts(logits, labels, mask=None):
  """logits [n, C] (fp32 or bf16), labels [n, C] fp32 (one/multi-hot), mask [n] or None.
  Returns (ncorrect, nseen) as Python floats and the argmax indices (int32 device tensor)."""
  idx, _, sums = ops.top1(logits, labels, mask)
  ncorrect, nseen = (float(x) for x in sums.tolist())
  return ncorrect, nseen, idx


def zero_shot_best_text(zimg, ztxt):
  """best_txt = (zimg @ ztxt.T).argmax(axis=1)
  (evaluators/proj/image_text/discriminative_classifier.py:284-288): wgmma GEMM + argmax."""
  import torch
  scores = ops.gemm(zimg.to(torch.bfloat16).contiguous(), ztxt.to(torch.bfloat16).contiguous(),
                    out_dtype=torch.float32)
  idx, _, _ = ops.top1(scores)
  return idx
