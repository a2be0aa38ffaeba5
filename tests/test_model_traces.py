"""CPU: what the ViT, two-tower and MLP-Mixer models launch, where they accumulate and what they keep.

The models run on CPU tensors with the C-ABI call replaced by a recorder (tests/golden/make_model_traces.py)
over every pool, with and without scan, the ViT with and without a class head, the Mixer with and without
token padding and stochastic-depth masks, under the freezing schedules that place the backward's cut on
each kind of stage, and under apply().  The traces must equal the committed ones call for call: every entry point, scalar argument and
argument-struct field, every parameter pointer, the P.on_ready calls and the bytes kept for the backward.
So must each configuration's parameter layout and the checksum of its seed-0 init."""
import difflib
import importlib.util
import json
import os

import pytest

_GEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_model_traces.py")


def _generator():
  spec = importlib.util.spec_from_file_location("make_model_traces", _GEN)
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def test_model_traces_match_the_golden():
  gen = _generator()
  with pytest.MonkeyPatch.context() as mp:
    got = gen.traces(mp.setattr)
  want = gen.load()
  assert sorted(got) == sorted(want)
  bad = [k for k in want if got[k] != want[k]]
  if bad:
    k = bad[0]
    lines = lambda entry: json.dumps(entry, indent=0, sort_keys=True).splitlines()
    diff = "\n".join(difflib.unified_diff(lines(want[k]), lines(got[k]), "golden", "now", n=1, lineterm=""))
    pytest.fail(f"{len(bad)} of {len(want)} traces differ, first {k!r}:\n{diff}")
