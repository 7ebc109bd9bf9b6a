"""The float64 training-step reference (tests/train_step_ref.py) on its own, without a GPU.

* Its ray chunking is exact: chunks with the criterion's denominators held fixed give the same loss terms, outputs
  and gradients as one evaluation of the whole batch, to rounding (measured 7e-15 relative on edges_occ1).
* With the library's nets swapped in, in mode "exact" and float32, it is the oracle's fp32 training step
  differentiated by torch autograd (tests/test_train_gpu.py's reference) to fp32 rounding (measured 5e-6, on `s`).
* The edges cases contain what they are meant to: rays with no valid static view, rays whose samples have fewer than
  2 valid dynamic views, basis rows that wrap.
"""

import pytest
import torch

import train_step_ref as T


def _worst(errs):
  return max(errs.items(), key=lambda kv: max(kv[1]))


def test_chunked_reference_equals_unchunked():
  c = T.make_case("edges_occ1")
  whole = T.reference(c, "cpu", "exact")
  chunked = T.reference(c, "cpu", "exact", chunk=40)
  errs = T.errors(chunked, whole, c["V_st"])
  assert set(errs) == set(T.errors(whole, whole, c["V_st"]))
  name, (rel, mx) = _worst(errs)
  assert rel <= 1e-12 and mx <= 1e-12, (name, rel, mx)
  assert len(errs) > 130  # terms, criterion inputs, every parameter, the basis and the feature maps


def test_float32_reference_matches_oracle_autograd():
  c = T.make_case("edges_occ2")
  oracle = T.reference(c, "cpu", None, dtype=torch.float32)
  ref = T.reference(c, "cpu", "exact", dtype=torch.float32)
  name, (rel, mx) = _worst(T.errors(ref, oracle, c["V_st"]))
  assert rel <= 5e-5 and mx <= 5e-5, (name, rel, mx)


@pytest.mark.parametrize("name", ["edges_occ1", "edges_occ2"])
def test_edges_cases_reach_their_edges(name):
  c = T.make_case(name)
  st, dy = T.view_counts(c)
  assert (st.sum(1) == 0).sum() >= 2  # rays no static view sees at any sample
  assert (dy.max(1).values < 2).sum() >= 2  # rays whose samples all have fewer than 2 valid dynamic views
  assert ((dy == 1).sum(1) > 0).sum() >= 1  # samples with exactly one valid view: a masked attention query row
  ref_idx, anc_idx = c["frame"]
  assert abs(ref_idx - anc_idx) == 1 and min(c["offs"][0]) + ref_idx < 0  # basis rows wrap
  assert c["aa"] == 1 and "s" in c["model"].net_coarse_st.state_dict()


def test_chunks_must_keep_the_dispatch():
  T._check_chunk(1024, 128, 64)
  with pytest.raises(AssertionError):
    T._check_chunk(1024, 64, 64)  # ref_feature_fc's forward would leave the tensor cores
  with pytest.raises(AssertionError):
    T._check_chunk(4096, 1024, 64)  # its weight gradient would too
