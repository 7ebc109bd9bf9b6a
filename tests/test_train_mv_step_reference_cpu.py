"""The float64 fine-stage training-step reference (tests/train_mv_step_ref.py) on its own, without a GPU.

* Its ray chunking is exact: chunks of the stand-in loss give the same loss, outputs and gradients as one evaluation
  of the whole batch, to rounding.
* With the library's nets swapped in, in mode "exact" and float32, it is the oracle's own fp32 fine step (mode None)
  differentiated by torch autograd, to fp32 rounding.
* The cases contain what they are meant to: rays no static view sees, samples with exactly one valid dynamic view and
  basis rows that wrap (edges), exp_sf tied on every ray (fresh, short), every coefficient zeroed (short).
* Every plant changes the float64 result.
"""

import pytest
import torch

import train_mv_step_ref as T


def _worst(errs):
  return max(errs.items(), key=lambda kv: max(kv[1]))


def test_chunked_reference_equals_unchunked():
  c = T.make_case("edges", rays=24)
  whole = T.reference(c, "cpu", "exact")
  chunked = T.reference(c, "cpu", "exact", chunk=10)
  assert len(T.spans(c["R"], 10)) == 3
  errs = T.errors(chunked, whole, c["V_st"])
  name, (rel, mx) = _worst(errs)
  assert rel <= 1e-12 and mx <= 1e-12, (name, rel, mx)
  assert len(errs) > 100  # the loss, the fine outputs, every parameter, the basis and the feature maps
  assert not T.zero_violations(chunked, whole)


def test_library_fine_depths_are_used():
  """z_fine replaces the oracle's resampling: the fine pass is evaluated at exactly the depths handed in."""
  c = T.make_case("short")
  own = T.reference(c, "cpu", "exact")
  z = own["coarse"]["z_vals"]
  zf = torch.sort(torch.cat([z, z[:, :2] + 0.25 * (z[:, 1:3] - z[:, :2])], 1), 1).values
  moved = T.reference(c, "cpu", "exact", z_fine=zf)
  assert not torch.equal(moved["out"]["fine/depth"], own["out"]["fine/depth"])
  want = (moved["out"]["fine/weights"] * zf.double()).sum(1)
  torch.testing.assert_close(moved["out"]["fine/depth"], want, rtol=1e-12, atol=1e-12)


def test_float32_reference_matches_oracle_autograd():
  c = T.make_case("edges", rays=16)
  oracle = T.reference(c, "cpu", None, dtype=torch.float32)
  ref = T.reference(c, "cpu", "exact", dtype=torch.float32)
  name, (rel, mx) = _worst(T.errors(ref, oracle, c["V_st"]))
  assert rel <= 5e-5 and mx <= 5e-5, (name, rel, mx)


def test_edges_case_reaches_its_edges():
  c = T.make_case("edges")
  st, dy = T.view_counts(c)
  assert (st.sum(1) == 0).sum() >= 2  # rays no static view sees at any sample
  assert (dy.max(1).values < 2).sum() >= 2  # rays whose samples all have fewer than 2 valid dynamic views
  assert ((dy == 1).sum(1) > 0).sum() >= 1  # samples with exactly one valid view: a masked attention query row
  f = c["frame"][0]
  assert f + min(c["offs"][0]) < 0 and f - 2 < 0  # displacement rows f - 3 (and exp_sf's f - 2) wrap
  assert c["aa"] == 1 and "s" in c["model"].net_fine_st.state_dict()
  assert not torch.equal(c["model"].trajectory_basis_fine, c["model"].trajectory_basis)


@pytest.mark.parametrize("name", ["fresh", "short"])
def test_motion_free_cases_tie_and_zero(name):
  """fresh: coeff_linear zero, so motion is 0 and exp_sf ties on every ray; the MotionMLP trunk and the basis get
  exactly zero gradient, coeff_linear a non-zero one (the half-split tie gradient).  short: fine S = 5, every sample's
  coefficients zeroed, so the whole MotionMLP and the basis get exactly zero gradient."""
  c = T.make_case(name, rays=12)
  ref = T.reference(c, "cpu", "exact")
  assert (ref["out"]["fine/exp_sf"] == 0).all()
  zeros, rows = T.zero_tensors(ref)
  trunk = ["grad.motion_mlp_fine.pts_linears.%d.%s" % (i, k) for i in range(8) for k in ("weight", "bias")]
  assert set(trunk + ["grad.trajectory_basis_fine"]) <= set(zeros)
  head = {"grad.motion_mlp_fine.coeff_linear.weight", "grad.motion_mlp_fine.coeff_linear.bias"}
  assert head <= set(zeros) if name == "short" else not head & set(zeros)
  assert len(rows) == c["model"].trajectory_basis_fine.shape[0]
  if name == "fresh":
    assert torch.equal(c["model"].trajectory_basis_fine, c["model"].trajectory_basis)


def test_every_plant_changes_the_result():
  c = T.make_case(T.PLANT_CASE, rays=12)
  clean = T.reference(c, "cpu", "exact")
  for plant in T.PLANTS:
    name, (rel, mx) = _worst(T.errors(T.reference(c, "cpu", "exact", plant=plant), clean, c["V_st"]))
    assert rel >= 1e-6, (plant, name, rel, mx)


def test_chunks_are_near_equal_and_keep_the_dispatch():
  assert T.spans(1031, 128) == [(0, 128), (128, 257), (257, 386), (386, 515), (515, 644), (644, 773), (773, 902),
                                (902, 1031)]
  assert T.spans(96, None) == [(0, 96)] and T.spans(200, 128) == [(0, 200)]
