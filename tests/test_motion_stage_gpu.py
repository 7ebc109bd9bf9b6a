"""The bf16 MotionMLP kernel against a float64 reference that rounds to bf16 where the kernel does
(tests/motion_stage_ref.py, mode="kernel").

Both entry points of a render reach the kernel: dyn_motion_mlp (MotionMLP.forward on xyzt rows, time as a column)
and dyn_motion_coeffs (a constant time, then the last round(0.1 S) samples of each ray zeroed, the whole axis
when S < 5).  Row counts around the kernel's 64-row warpgroup and 128-row iteration edges, a ragged count that
gives every persistent CTA several iterations, and one benchmark chunk (8192 rays x 64 or 128 samples, compared
on sampled rays).  Every case has points with |x| in the tens, where PE's angle-addition recurrence runs from
large angles.  The reference is evaluated on the GPU in float64.
"""

import pytest
import torch

import motion_stage_ref as msr
from dynibar_b200 import render_ray as rr, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def motion():
  model, _ = synthetic.make_model(16, 16, seed=3)
  return synthetic.model_to(model, DEV).motion_mlp


@pytest.fixture
def bf16():
  rr.set_precision("bf16")
  yield
  rr.set_precision("fp32")


def _check(name, got, ref):
  err, ratio, per_mag = msr.errors(got, ref)
  print("%s: max err %.3e, err / tol %.3f, err / mag %.3e" % (name, err, ratio, per_mag))
  assert ratio <= 1.0, (name, err, ratio, per_mag)


@pytest.mark.parametrize("N", [1, 63, 64, 65, 127, 129, 3001])
@pytest.mark.parametrize("div", [1.0, 4.0])
def test_motion_mlp_rows(motion, bf16, N, div):
  g = torch.Generator().manual_seed(N)
  xyz = msr.make_points(N, seed=N, big=min(N, 16))
  xyzt = torch.cat([xyz, torch.rand(N, 1, generator=g) * 2 - 1], -1).to(DEV)
  motion.sf_mag_div = div
  try:
    got = rr.motion_mlp_forward(motion, xyzt)
  finally:
    motion.sf_mag_div = 1.0
  torch.cuda.synchronize()
  ref = msr.motion_mlp(motion.state_dict(), xyzt, div=div)
  _check("mlp N=%d div=%g" % (N, div), got, ref)


@pytest.mark.parametrize("R,S", [(7, 3), (5, 4), (37, 64), (21, 128), (1, 5), (3, 20)])
def test_motion_coeffs(motion, bf16, R, S):
  pts = msr.make_points(R * S, seed=R * 1000 + S, big=min(R * S, 32)).reshape(R, S, 3).to(DEV)
  got = rr.motion_coefficients(motion, pts, 0.37)
  torch.cuda.synchronize()
  ref = msr.motion_coeffs(motion.state_dict(), pts, 0.37)
  _check("coeffs R=%d S=%d" % (R, S), got, ref)


@pytest.mark.parametrize("S", [64, 128])
def test_motion_coeffs_bench_chunk(motion, bf16, S):
  """One benchmark chunk (8192 rays), compared on 512 sampled rays."""
  R = 8192
  pts = msr.make_points(R * S, seed=S, scale=2.0, big=4096).reshape(R, S, 3).to(DEV)
  motion.sf_mag_div = 2.0
  try:
    got = rr.motion_coefficients(motion, pts, -0.5)
  finally:
    motion.sf_mag_div = 1.0
  torch.cuda.synchronize()
  rays = torch.randperm(R, generator=torch.Generator().manual_seed(S))[:512].to(DEV)
  rays[0] = 0  # the big-|x| points
  ref = msr.motion_coeffs(motion.state_dict(), pts[rays], -0.5, div=2.0)
  _check("coeffs chunk S=%d" % S, got[rays], ref)
