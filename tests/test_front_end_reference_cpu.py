"""The float64 reference of the fp32 ray front end (tests/front_end_ref.py) without a GPU: in float64 it equals the
oracle's functions, evaluated in fp32 it stays within its own bars, and planted errors exceed those bars by 3x or
more."""

import pytest
import torch

import front_end_ref as FE
from geometry_stage_ref import d64, excess, float64, rig
from oracle import dynibar_oracle as O


def _inputs():
  g = torch.Generator().manual_seed(3)
  R, S, T, nb, V = 13, 70, 9, 8, 32
  o, d = torch.randn(R, 3, generator=g), torch.randn(R, 3, generator=g)
  jitter = torch.rand(R, S, generator=g)
  pts = torch.randn(R, S, 3, generator=g) * 3.0
  coeff, basis = torch.randn(R, S, 3 * nb, generator=g), torch.randn(T, nb, generator=g)
  wa, wb = torch.rand(R, S, generator=g) / S, torch.rand(R, S, generator=g) / S
  cams, query = rig(V, 40, 60, 5)
  xyz = torch.randn(V, R * S, 3, generator=g)
  xst = torch.randn(V, R * S, 3, generator=g)
  return dict(o=o, d=d, jitter=jitter, pts=pts, coeff=coeff, basis=basis, wa=wa, wb=wb, cams=cams, query=query,
              xyz=xyz, xst=xst, S=S)


X = _inputs()
NEAR, FAR = 0.5, 60.0
OFFS = [-3, -2, -1, 1, 2, 3]


def outputs(dt=torch.float64, plant=None):
  """name -> (bar name, value, mag) of every reference output on the shared inputs."""
  x = X
  z = FE.sample_z32(NEAR, FAR, x["S"], True, x["jitter"], plant=plant)
  ps = FE.points_s(x["o"], x["d"], z, NEAR, FAR, dt, plant)
  seq, smag = FE.traj_displace(x["pts"], x["coeff"], x["basis"], 1, [-4] + OFFS, 2, dt, plant)
  dl, dmag = FE.traj_delta(x["coeff"], x["basis"], [-9, -1, 3], [0, 8, -2], dt, plant)
  oc = FE.occlusion(x["wa"], x["wb"], dt, plant)
  pr = FE.plucker_ref(x["o"], x["d"], dt, plant)
  pss = FE.plucker_src(x["pts"], x["cams"], dt, plant)
  an = FE.compute_angle(x["xst"], x["xyz"], x["query"], x["cams"], dt, plant)
  return {"z": ("s_vals", z.double(), torch.zeros_like(z.double())),
          "pts": ("pts", ps["pts"], ps["pts_mag"]), "s": ("s_vals", ps["s"], ps["s_mag"]),
          "traj_displace": ("traj", seq, smag), "traj_delta": ("traj", dl, dmag),
          "occ": ("occ", oc["occ"], oc["occ_mag"]), "occ_map": ("occ", oc["map"], oc["map_mag"]),
          "plucker_ref": ("plucker_m", pr["out"], pr["mag"]), "plucker_src": ("plucker_m", pss["out"], pss["mag"]),
          "angle": ("angle", an["out"], an["mag"])}


def test_exact_mode_equals_the_oracle():
  x = X
  o64, d64_, c64 = d64(x["o"]), d64(x["d"]), d64(x["cams"])
  # sample_along_ray: z in fp32 bit for bit, pts and s_vals in float64
  for inv in (False, True):
    for jit in (None, x["jitter"]):
      _, z32, _ = O.sample_along_ray(x["o"], x["d"], torch.tensor([[NEAR, FAR]]), x["S"], inv, jit)
      assert torch.equal(FE.sample_z32(NEAR, FAR, x["S"], inv, jit).expand_as(z32), z32)
      with float64():
        p_o, z64, s_o = O.sample_along_ray(o64, d64_, torch.tensor([[NEAR, FAR]]), x["S"], inv,
                                           None if jit is None else d64(jit))
      assert z64.dtype == torch.float64
      ps = FE.points_s(o64, d64_, z64, NEAR, FAR)
      torch.testing.assert_close(ps["pts"], p_o, rtol=1e-14, atol=1e-14)
      torch.testing.assert_close(ps["s"], s_o, rtol=1e-12, atol=1e-12)
  torch.testing.assert_close(FE.plucker_ref(o64, d64_)["out"], O.plucker_ref(o64, d64_), rtol=1e-14, atol=1e-14)
  torch.testing.assert_close(FE.plucker_src(d64(x["pts"]), c64)["out"], O.plucker_src(d64(x["pts"]), c64[None]),
                             rtol=1e-13, atol=1e-13)
  q = d64(x["query"])
  torch.testing.assert_close(FE.compute_angle(d64(x["xst"][:1]), d64(x["xyz"]), q, c64)["out"],
                             O.ray_angle_diff(d64(x["xst"][0]), d64(x["xyz"]), q, c64), rtol=1e-13, atol=1e-13)
  seq, _ = FE.traj_displace(d64(x["pts"]), d64(x["coeff"]), d64(x["basis"]), 4, OFFS, 0)
  want, traj = O.displaced_points(d64(x["pts"]), d64(x["coeff"]), d64(x["basis"]), 4, OFFS)
  torch.testing.assert_close(seq, want, rtol=1e-14, atol=1e-14)
  dl, _ = FE.traj_delta(d64(x["coeff"]), d64(x["basis"]), [5, 6], [4, 3])
  torch.testing.assert_close(dl, torch.stack([traj[1] - traj[0], traj[2] - traj[-1]]), rtol=1e-14, atol=1e-14)
  oc = FE.occlusion(x["wa"], x["wb"])
  torch.testing.assert_close(oc["occ"], 1.0 - (d64(x["wa"]) - d64(x["wb"])).abs(), rtol=0, atol=0)


def test_fp32_evaluation_stays_within_the_bars():
  ref, f32 = outputs(), outputs(torch.float32)
  for k, (name, r, mag) in ref.items():
    x = excess(name, f32[k][1].double(), r, mag, 0.0, tol=FE.TOL)
    assert x.max() <= FE.TOL[name][1], (k, x.max().item())


@pytest.mark.parametrize("plant", FE.PLANTS)
def test_planted_errors_exceed_the_bars_threefold(plant):
  ref, bad = outputs(), outputs(plant=plant)
  worst = 0.0
  for k, (name, r, mag) in ref.items():
    b = bad[k][1]
    if b.shape != r.shape:
      worst = float("inf")
      continue
    x = excess(name, b, r, mag, 0.0, tol=FE.TOL) / FE.TOL[name][1]
    worst = max(worst, x.max().item())
  assert worst >= 3.0, (plant, worst)
