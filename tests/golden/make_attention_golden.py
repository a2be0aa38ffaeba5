"""Writes tests/golden/attention_unmasked.json: sha256 digests of the unmasked attention kernels' outputs
(o, lse, dq, dk, dv) at the shapes of test_attention_mask_gpu.GOLDEN_CASES, on seeded inputs.  Run it on an
H100 in the tree whose kernels' bits are to be kept:

  python tests/golden/make_attention_golden.py

The committed file was written by the kernels before the key mask was added (the same generator and
test module copied into that tree).
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import torch  # noqa: E402  pylint: disable=wrong-import-position

import test_attention_mask_gpu as T  # noqa: E402  pylint: disable=wrong-import-position


def main():
  out = {"device": torch.cuda.get_device_name(0), "digests": T.golden_results()}
  with open(T.GOLDEN, "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
  print(json.dumps(out))


if __name__ == "__main__":
  main()
