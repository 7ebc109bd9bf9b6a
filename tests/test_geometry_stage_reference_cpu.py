"""The float64 reference of the fp32 glue kernels (tests/geometry_stage_ref.py) on the CPU: its exact mode equals
float64 autograd through the oracle away from kinks, the gather and its backward are adjoint, central differences
confirm d xyz, the coordinate bound delta covers an fp32 evaluation of the projection, and every planted error
would fail the GPU comparison (tests/test_geometry_stage_gpu.py) on the inputs that test uses by a wide margin."""

import pytest
import torch

import geometry_stage_ref as G

MARGIN = 3.0  # a planted error must exceed its bar by this factor on some compared element

# the GPU test's "V5_tails" gather case and seeds (test_geometry_stage_gpu.py)
GATHER_V5 = dict(V=5, R=7, S=9, H=37, W=53, h=10, w=14, seed=5 * 31 + 7)


def _v5():
  a = GATHER_V5
  return G.gather_case(a["V"], a["R"], a["S"], a["H"], a["W"], a["h"], a["w"], seed=a["seed"])


def test_exact_gather_matches_oracle_autograd():
  case = _v5()
  ref = G.gather(case, exact=True)
  rf, mask, gm, gx = G.gather_oracle_autograd(case)
  N, V = case["R"] * case["S"], case["V"]
  assert (ref["rgb_feat"] - rf.reshape(N, V, 35)).abs().max() < 1e-12
  assert torch.equal(ref["mask"], mask.reshape(N, V))
  assert (ref["g_maps"] - gm).abs().max() < 1e-12
  clean = ~ref["xyz_kink"]
  assert clean.all()  # no sample of this case sits at a kink
  assert ((ref["g_xyz"] - gx.reshape(V, N, 3)).abs().amax(-1)[clean]).max() < 1e-9 * gx.abs().max()


@pytest.mark.parametrize("vanilla", [False, True])
def test_exact_composite_matches_oracle_autograd(vanilla):
  case = G.composite_case(7, 33, seed=33 + 100 * vanilla, special=True)
  for gs_on in (True, False):
    ref = G.composite(case, vanilla=vanilla, gs_on=gs_on)
    o, ga, gb = G.composite_oracle_autograd(case, vanilla=vanilla, gs_on=gs_on)
    assert (ref["samples"][0 if vanilla else 4] - o["weights"]).abs().max() < 1e-15
    assert (ref["rays"][:, 3 if vanilla else 9] - o["depth"]).abs().max() < 1e-12
    assert (ref["g_raw_a"] - ga).abs().max() < 1e-12 * (1 + ga.abs().max())
    if not vanilla:
      assert (ref["g_raw_b"] - gb).abs().max() < 1e-12 * (1 + gb.abs().max())
      want_mask = (((case["mask_a"].sum(-1) > case["min_a"]).sum(-1) > 8)
                   | ((case["mask_b"].sum(-1) > case["min_b"]).sum(-1) > 8)).double()
      assert torch.equal(ref["rays"][:, 10], want_mask)


def test_exact_flow_matches_oracle_autograd():
  case = G.flow_case(6, 5, 33, seed=6 * 7 + 33, close_to_camera=True, zero_weights=True)
  ref = G.flow(case, exact=True)
  fl, gw, gp = G.flow_oracle_autograd(case)
  rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
  assert rel(ref["flows"], fl) < 1e-12 and rel(ref["g_weights"], gw) < 1e-12 and rel(ref["g_pts"], gp) < 1e-12


@pytest.mark.parametrize("det", [True, False])
@pytest.mark.parametrize("inv_uniform", [0, 1])
def test_resample_matches_oracle(inv_uniform, det):
  case = G.resample_case(6, 64, 64, seed=64 * 3 + 64 + 7 * inv_uniform + det, det=det, inv_uniform=inv_uniform,
                         special=True)
  ref = G.resample(case)
  want = G.resample_oracle(case)
  # the reference adds the fp32 value of 1e-5 (relative difference 2e-9) to the weights
  assert (ref["merged"] - want).abs().max() < 1e-7
  assert (ref["lo"] <= ref["fine"]).all() and (ref["fine"] <= ref["hi"]).all()


def test_gather_backward_is_the_adjoint_of_the_gather():
  """<g, gather(F)> = <gather_bwd(g), F> for the feature-map part (the gather is linear in the maps)."""
  case = _v5()
  ref = G.gather(case, exact=True)
  g = G.d64(case["g_feat"]).reshape(-1, case["V"], 35)[..., 3:]
  lhs = (g * ref["rgb_feat"][..., 3:]).sum()
  rhs = (ref["g_maps"] * G.d64(case["featmaps"])).sum()
  assert abs(lhs - rhs) <= 1e-12 * abs(lhs)


def test_dxyz_matches_central_differences():
  case = _v5()
  ref = G.gather(case, exact=True)
  V, N = case["V"], case["R"] * case["S"]
  g = G.d64(case["g_feat"]).reshape(N, V, 35)
  h = 1e-7
  xyz = G.d64(case["xyz"])
  for k in range(3):
    fd = []
    for s in (1, -1):
      c = dict(case, xyz=(xyz + s * h * torch.nn.functional.one_hot(torch.tensor(k), 3)))
      r = G.gather(c, backward=False, exact=True)
      fd.append((g * r["rgb_feat"]).sum(-1))  # [N,V]: each (point, view) owns its own gradient
    num = (fd[0] - fd[1]).t() / (2 * h)
    ana = ref["g_xyz"][..., k]
    assert ((num - ana).abs() <= 1e-6 * (1 + ana.abs())).all(), (num - ana).abs().max()


def test_fp32_projection_stays_within_a_quarter_of_delta():
  """An fp32 evaluation of the kernel's chain (px, pz, u = px / max(pz, 1e-8), fx = (2u/(W-1) - 1 + 1) 0.5 (w-1))
  lands within delta / 4 of the float64 value on the GPU test's inputs."""
  for case in (_v5(), G.gather_case(8, 64, 64, 288, 512, 72, 128, seed=5), G.exact_case()):
    V, N = case["V"], case["R"] * case["S"]
    P = G.view_P(case["cams"])
    q = G.d64(case["xyz"]).reshape(V, N, 3)
    with G.float64():
      pr = G.project(P, q)
      h_img, w_img = float(case["cams"][0, 0]), float(case["cams"][0, 1])
      fx, dfx = G.grid_coord(pr["u"], pr["du"], w_img, case["featmaps"].shape[3])
    P32, q32 = P.float(), q.float()
    row = lambda i: ((P32[:, None, i, 0] * q32[..., 0] + P32[:, None, i, 1] * q32[..., 1]) + P32[:, None, i, 2] * q32[..., 2]) + P32[:, None, i, 3]
    px, pz = row(0), row(2)
    u32 = (px / torch.clamp(pz, min=torch.tensor(1e-8, dtype=torch.float32))).clamp(-1e6, 1e6)
    one = torch.tensor(1.0, dtype=torch.float32)
    gx = 2 * u32 / (torch.tensor(w_img, dtype=torch.float32) - one) - one
    fx32 = (gx + one) * 0.5 * float(case["featmaps"].shape[3] - 1)
    live = pr["u0"].abs() <= 1e6
    assert ((u32.double() - pr["u"]).abs() <= pr["du"] / 4)[live].all()
    assert ((fx32.double() - fx).abs() <= dfx / 4)[live].all()


def _ratio(name, planted, ref, mag, sens, clean=None):
  r = (planted - ref).abs() / G.bar(name, ref, mag, sens)
  if clean is not None:
    while clean.dim() < r.dim():
      clean = clean[..., None]
    r = r * clean.expand_as(r)
  return torch.nan_to_num(r, nan=0.0).max().item()


def _plant_ratio(plant):
  if plant in ("mask_right_exclusive", "pz_clamp_grad_kept", "feat_norm_by_map", "ax_bx_swap", "dxyz_no_p8"):
    case = G.exact_case() if plant in ("mask_right_exclusive", "pz_clamp_grad_kept") else _v5()
    ref, pl = G.gather(case), G.gather(case, plant=plant)
    if (pl["mask"] != ref["mask"]).any():
      return float("inf")
    return max(_ratio("rgb_feat", pl["rgb_feat"], ref["rgb_feat"], ref["rgb_feat_mag"], ref["rgb_feat_sens"]),
               _ratio("g_maps", pl["g_maps"], ref["g_maps"], ref["g_maps_mag"], ref["g_maps_sens"]),
               _ratio("g_xyz", pl["g_xyz"], ref["g_xyz"], ref["g_xyz_mag"], ref["g_xyz_sens"], ~ref["xyz_kink"]))
  if plant in ("composite_no_1e10", "last_delta_one", "T_inclusive", "suffix_off_by_one"):
    case = G.composite_case(7, 33, seed=33, special=True)  # the GPU test's S = 33 case
    ref, pl = G.composite(case), G.composite(case, plant=plant)
    return max(_ratio("comp_rays", pl["rays"], ref["rays"], ref["rays_mag"], ref["rays_sens"]),
               _ratio("comp_samples", pl["samples"], ref["samples"], ref["samples_mag"], ref["samples_sens"]),
               _ratio("comp_grad", pl["g_raw_a"], ref["g_raw_a"], ref["g_raw_a_mag"], ref["g_raw_a_sens"]),
               _ratio("comp_grad", pl["g_raw_b"], ref["g_raw_b"], ref["g_raw_b_mag"], ref["g_raw_b_sens"]))
  if plant == "flow_Rw_transposed":
    case = G.flow_case(6, 5, 33, seed=6 * 7 + 33, close_to_camera=True, zero_weights=True)
    ref, pl = G.flow(case), G.flow(case, plant=plant)
    return max(_ratio("flow_g_w", pl["g_weights"], ref["g_weights"], ref["g_weights_mag"], ref["g_weights_sens"]),
               _ratio("flow_g_pts", pl["g_pts"], ref["g_pts"], ref["g_pts_mag"], ref["g_pts_sens"]))
  det = plant == "cdf_M_plus_1"  # u = 1 (the last linspace point) reaches the last cdf entry
  case = G.resample_case(6, 64, 64, seed=64 * 3 + 64 + det, det=det, inv_uniform=0, special=True)
  ref, pl = G.resample(case), G.resample(case, plant=plant)
  b = G.bar("resample", ref["fine"], ref["fine"].abs(), ref["sens"])
  outside = torch.maximum(ref["lo"] - b - pl["fine"], pl["fine"] - ref["hi"] - b).clamp(min=0) / b
  return torch.nan_to_num(outside, nan=0.0).max().item() + 1.0


@pytest.mark.parametrize("plant", G.PLANTS)
def test_planted_error_exceeds_its_bar(plant):
  r = _plant_ratio(plant)
  assert r >= MARGIN, (plant, r)
