"""The MotionMLP reference of tests/test_motion_stage_gpu.py (tests/motion_stage_ref.py) on the CPU: it
agrees with the oracle in exact mode, and every planted error exceeds the GPU test's tolerance at least 3x."""

import pytest
import torch

import motion_stage_ref as msr
from dynibar_b200 import synthetic
from oracle import dynibar_oracle as O

MARGIN = 3.0


@pytest.fixture(scope="module")
def case():
  model, _ = synthetic.make_model(16, 16, seed=3)
  w = model.motion_mlp.state_dict()
  pts = msr.make_points(16 * 64, seed=1, big=64).reshape(16, 64, 3)
  return w, pts, msr.motion_coeffs(w, pts, 0.3)


def test_exact_mode_matches_oracle(case):
  w, pts, _ = case
  want = O.motion_coefficients(w, pts, torch.tensor(0.3))  # fp32
  got = msr.motion_coeffs(w, pts, 0.3, mode="exact")["coeff"].reshape(want.shape)
  assert torch.allclose(got, want.double(), rtol=1e-4, atol=1e-6)
  assert (got[:, -6:] == 0).all() and (got[:, :-6] != 0).all()


def test_zeroed_samples():
  # int(round(0.1 S)) rounds half to even; 0 zeroes the whole axis (x[:, -0:])
  assert [msr.n_last(S) for S in (1, 3, 4, 5, 15, 25, 64, 128)] == [1, 3, 4, 5, 2, 2, 6, 13]


def test_kernel_mode_within_tolerance_of_itself_and_off_exact(case):
  w, pts, ref = case
  assert msr.errors(ref["coeff"], ref)[1] == 0.0
  # the bf16 roundings are visible: the kernel-mode reference is not the exact one
  assert msr.errors(msr.motion_coeffs(w, pts, 0.3, mode="exact")["coeff"], ref)[0] > 0.0


@pytest.mark.parametrize("plant", msr.PLANTS)
def test_planted_error_exceeds_tolerance(case, plant):
  w, pts, ref = case
  got = msr.motion_coeffs(w, pts, 0.3, plant=plant)["coeff"]
  err, ratio, _ = msr.errors(got, ref)
  print("%s: max err %.3e, err / tol %.1f" % (plant, err, ratio))
  assert ratio >= MARGIN, (plant, err, ratio)
