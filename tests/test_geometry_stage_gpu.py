"""The fp32 glue kernels against their float64 reference (tests/geometry_stage_ref.py), element by element: the
projection + bilinear gather and its backward, compositing forward and backward (both variants), optical flow
forward and backward, and hierarchical resampling.

Every compared element either meets its bar, or is flagged at a kink and matches one of its one-sided reference
values within the bar.  The number of kink-flagged elements is asserted per case, so the classifier cannot absorb
a bug.  With GEOMETRY_STAGE_REPORT=<path> the worst (err - atol - sens) / (ulp + 2^-24 mag) per bar is written
there as JSON: that is how the ulps of geometry_stage_ref.TOL were measured."""

import json
import os

import pytest
import torch

import geometry_stage_ref as G
from dynibar_b200 import autograd as ag
from dynibar_b200 import projection
from dynibar_b200._lib import lib, ptr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
  yield
  path = os.environ.get("GEOMETRY_STAGE_REPORT")
  if path:
    with open(path, "w") as f:
      json.dump(_WORST, f, indent=1, sort_keys=True)


def _check(tag, name, got, ref, mag, sens, kink=None, alts=None, max_kink=0):
  """got / ref / mag / sens: same shapes; kink: bool over the leading dims of ref that alts [..., k] extends."""
  got = G.d64(got)
  # every compared output is finite in the reference; a NaN or inf from the kernel fails here rather than slipping
  # through the comparisons below (NaN > bar is False)
  assert torch.isfinite(ref).all(), "%s %s: non-finite reference" % (tag, name)
  fin = torch.isfinite(got)
  assert fin.all(), "%s %s: %d non-finite elements, first at %s" % (tag, name, int((~fin).sum()),
                                                                    tuple((~fin).nonzero()[0].tolist()))
  b = G.bar(name, ref, mag, sens)
  err = (got - ref).abs()
  ex = G.excess(name, got, ref, mag, sens)
  if kink is None:
    kink = torch.zeros(ref.shape[:1], dtype=torch.bool)
  kk = kink
  while kk.dim() < ref.dim():
    kk = kk[..., None]
  kk = kk.expand_as(ref)
  clean = ~kk
  w = torch.nan_to_num(ex[clean], nan=float("inf")).max().item() if clean.any() else 0.0
  _WORST[name] = max(_WORST.get(name, -1e30), w)
  bad = ~(err <= b) & clean
  assert not bad.any(), "%s %s: %d elements over the bar, worst err %.3e bar %.3e at %s" % (
      tag, name, int(bad.sum()), err[bad].max().item(), b[bad][err[bad].argmax()].item(),
      tuple(bad.nonzero()[0].tolist()))
  n_kink = int(kink.sum())
  assert n_kink <= max_kink, "%s %s: %d elements at a kink (at most %d expected)" % (tag, name, n_kink, max_kink)
  if n_kink:
    if alts is None:  # both sides acceptable (a discontinuous 0 / 1 output)
      return
    ok = ((got[..., None] - alts).abs() <= b[..., None]).all(-2 if alts.dim() > ref.dim() else -1)
    ok = ok.any(-1)
    while ok.dim() > kink.dim():
      ok = ok.all(-1)
    assert ok[kink].all(), "%s %s: kink elements match no one-sided value" % (tag, name)


# ----------------------------------------------------------------------------------------------------------------
# gather
# ----------------------------------------------------------------------------------------------------------------
def _run_gather(case, need_xyz=True):
  d = lambda t: None if t is None else t.to(DEV)
  V, R, S = case["V"], case["R"], case["S"]
  cams = d(case["cams"])[None]
  imgs = d(case["rgbs"])[None]
  fm = d(case["featmaps"]).requires_grad_(True)
  xyz = None if case["xyz"] is None else d(case["xyz"]).requires_grad_(need_xyz)
  cam_idx = None if case["tgt_idx"] is None else d(case["tgt_idx"])
  rf, rd, mk = projection.project_gather(d(case["xyz_st"]), None if xyz is None else xyz.detach(),
                                         d(case["queries"]), imgs, cams, fm.detach(), camera_index=cam_idx)
  rf2, _, _ = ag.project_gather(d(case["xyz_st"]), xyz, d(case["queries"][:1]), imgs, cams, fm)
  (rf2 * d(case["g_feat"])).sum().backward()
  torch.cuda.synchronize()
  N = R * S
  return (rf.reshape(N, V, 35).cpu(), rd.reshape(N, V, 4).cpu(), mk.reshape(N, V).cpu(), fm.grad.cpu(),
          None if xyz is None else xyz.grad.reshape(V, N, 3).cpu())


def _compare_gather(tag, case, ref, got, max_kink, rows=None):
  rf, rd, mk, gm, gx = got
  if rows is not None:
    rf, rd, mk = rf[rows], rd[rows], mk[rows]
    gx = None if gx is None else gx[:, rows]
  _check(tag, "rgb_feat", rf, ref["rgb_feat"], ref["rgb_feat_mag"], ref["rgb_feat_sens"])
  _check(tag, "ray_diff", rd, ref["ray_diff"], ref["ray_diff_mag"], torch.zeros_like(ref["ray_diff"]))
  mk_bad = (G.d64(mk) != ref["mask"]) & ~ref["mask_kink"]
  assert not mk_bad.any(), (tag, "mask", mk_bad.nonzero()[:5].tolist())
  assert int(ref["mask_kink"].sum()) <= max_kink, (tag, "mask kinks", int(ref["mask_kink"].sum()))
  _check(tag, "g_maps", gm, ref["g_maps"], ref["g_maps_mag"], ref["g_maps_sens"])
  if gx is not None:
    _check(tag, "g_xyz", gx, ref["g_xyz"], ref["g_xyz_mag"], ref["g_xyz_sens"], kink=ref["xyz_kink"],
           alts=ref["g_xyz_alt"], max_kink=max_kink)


GATHER_CASES = {  # name: (V, R, S, H, W, h, w, static, K)
    "V1": (1, 3, 7, 37, 53, 10, 14, False, 1),
    "V5_tails": (5, 7, 9, 37, 53, 10, 14, False, 1),
    "V7_static": (7, 5, 11, 48, 64, 12, 16, True, 1),
    "V11_h2": (11, 3, 13, 30, 40, 2, 10, False, 1),
    "V32_w2": (32, 2, 5, 40, 30, 10, 2, False, 1),       # 320 pairs: a partial 256-pair block
    "V8_multicam": (8, 5, 11, 48, 64, 12, 16, False, 3),
}


@pytest.mark.parametrize("name", sorted(GATHER_CASES))
def test_gather_forward_backward(name):
  V, R, S, H, W, h, w, static, K = GATHER_CASES[name]
  assert (R * S * V) % 256 != 0 and (V == 32 or (R * S * V) % 32 != 0)  # both tail paths of the gather
  case = G.gather_case(V, R, S, H, W, h, w, seed=V * 31 + R, static=static, K=K)
  ref = G.gather(case)
  _compare_gather(name, case, ref, _run_gather(case), max_kink=4)


def test_gather_exact_rig():
  """Points exactly on u = 0, u = W-1, v = 0, v = H-1 and on pixel centres, just outside, behind the camera, at
  0 < pz < 1e-8 and beyond the 1e6 clamp: the mask must match exactly."""
  case = G.exact_case()
  ref = G.gather(case)
  got = _run_gather(case)
  assert torch.equal(G.d64(got[2]), ref["mask"]), (got[2].t(), ref["mask"].t())
  assert ref["mask"].sum() > 0 and (ref["mask"] == 0).sum() > 0
  # points on pixel centres (or clamped to +-1e6) sit on integer tap coordinates of the image grid: exactly those
  # are d-xyz kinks in every view; the points at fractional positions are compared against their bar alone
  on_grid = case["on_grid"][None].expand(case["V"], -1)
  assert torch.equal(ref["xyz_kink"], on_grid)
  _compare_gather("exact", case, dict(ref, mask_kink=torch.zeros_like(ref["mask_kink"])), got,
                  max_kink=int(on_grid.sum()))


def test_gather_training_shape():
  """1024 rays x 64 samples x 8 views, 288 x 512 images, 72 x 128 maps: g_featmaps compared in full, everything
  else on 512 sampled points."""
  case = G.gather_case(8, 1024, 64, 288, 512, 72, 128, seed=5)
  rows = torch.randperm(1024 * 64, generator=torch.Generator().manual_seed(0))[:512].sort().values
  ref = G.gather(case, rows=rows)
  # about 2 delta / 1 of each of the 4 tap coordinates of 4096 (point, view) pairs lies within delta of a grid line
  _compare_gather("train", case, ref, _run_gather(case), max_kink=24, rows=rows)


# ----------------------------------------------------------------------------------------------------------------
# compositing
# ----------------------------------------------------------------------------------------------------------------
def _run_composite(case, vanilla, gs_on):
  d = lambda t: t.to(DEV).contiguous()
  R, S = case["R"], case["S"]
  ra, rb, z = d(case["raw_a"]), d(case["raw_b"]), d(case["z"])
  ma, mb = d(case["mask_a"]), d(case["mask_b"])
  gr, gs = d(case["g_rays"]), d(case["g_samples"])
  if vanilla:
    rays, samp = torch.empty(R, 5, device=DEV), torch.empty(2, R, S, device=DEV)
    assert lib.dyn_composite_vanilla(ptr(ra), ptr(z), ptr(ma), ma.shape[2], case["min_a"], R, S, ptr(rays),
                                     ptr(samp), None) == 0
    grv = torch.cat([gr[:, 0:3], gr[:, 9:10], gr[:, 10:11]], -1).contiguous()
    gsv = gs[[4, 3]].contiguous()
    g_a = torch.empty_like(ra)
    assert lib.dyn_composite_vanilla_backward(ptr(ra), ptr(z), ptr(grv), ptr(gsv) if gs_on else None, R, S,
                                              ptr(g_a), None) == 0
    g_b = None
  else:
    rays, samp = torch.empty(R, 11, device=DEV), torch.empty(5, R, S, device=DEV)
    assert lib.dyn_composite(ptr(ra), ptr(rb), ptr(z), ptr(ma), ma.shape[2], case["min_a"], ptr(mb), mb.shape[2],
                             case["min_b"], R, S, ptr(rays), ptr(samp), None) == 0
    g_a, g_b = torch.empty_like(ra), torch.empty_like(rb)
    assert lib.dyn_composite_backward(ptr(ra), ptr(rb), ptr(z), ptr(gr), ptr(gs) if gs_on else None, R, S,
                                      ptr(g_a), ptr(g_b), None) == 0
  torch.cuda.synchronize()
  return rays.cpu(), samp.cpu(), g_a.cpu(), None if g_b is None else g_b.cpu()


COMPOSITE_S = (1, 2, 31, 32, 33, 128, 255, 256)


@pytest.mark.parametrize("vanilla", [False, True], ids=["composite", "vanilla"])
@pytest.mark.parametrize("S", COMPOSITE_S)
def test_composite_forward_backward(S, vanilla):
  case = G.composite_case(7, S, seed=S + 100 * vanilla, special=True)
  for gs_on in ((True, False) if S in (1, 33, 256) else (True,)):
    ref = G.composite(case, vanilla=vanilla, gs_on=gs_on)
    rays, samp, g_a, g_b = _run_composite(case, vanilla, gs_on)
    tag = "S%d%s%s" % (S, "v" if vanilla else "", "" if gs_on else "-nogs")
    nr = rays.shape[1] - 1
    _check(tag, "comp_rays", rays[:, :nr], ref["rays"][:, :nr], ref["rays_mag"][:, :nr], ref["rays_sens"][:, :nr])
    assert torch.equal(G.d64(rays[:, nr]), ref["rays"][:, nr]), (tag, "mask", rays[:, nr], ref["rays"][:, nr])
    _check(tag, "comp_samples", samp, ref["samples"], ref["samples_mag"], ref["samples_sens"])
    _check(tag, "comp_grad", g_a, ref["g_raw_a"], ref["g_raw_a_mag"], ref["g_raw_a_sens"])
    if not vanilla:
      _check(tag, "comp_grad", g_b, ref["g_raw_b"], ref["g_raw_b_mag"], ref["g_raw_b_sens"])
  if S >= 9:  # the > 8 rule of the ray mask: 8 samples seen by more than min_views views -> 0, 9 -> 1
    assert ref["rays"][4, -1] == 0 and ref["rays"][5, -1] == 1


@pytest.mark.parametrize("vanilla", [False, True], ids=["composite", "vanilla"])
def test_composite_autograd_wrappers(vanilla):
  """ag.composite / ag.composite_vanilla map each output key and each upstream gradient to the kernels' slots."""
  S = 33
  case = G.composite_case(7, S, seed=S + 100 * vanilla, special=True)
  ref = G.composite(case, vanilla=vanilla, gs_on=True)
  d = lambda t: t.float().to(DEV)
  ra, rb = d(case["raw_a"]).requires_grad_(True), d(case["raw_b"]).requires_grad_(True)
  gr, gs = d(ref["g_rays_used"]), d(ref["g_samples_used"])
  if vanilla:
    out = ag.composite_vanilla(ra, d(case["z"]), d(case["mask_a"]), case["min_a"])
    ray_keys = (("rgb", slice(0, 3)), ("depth", 3))
    samp_keys = ("weights", "alpha")
  else:
    out = ag.composite(ra, rb, d(case["z"]), d(case["mask_a"]), d(case["mask_b"]), case["min_a"], case["min_b"])
    ray_keys = (("rgb", slice(0, 3)), ("rgb_static", slice(3, 6)), ("rgb_dy", slice(6, 9)), ("depth", 9))
    samp_keys = ("alpha_dy", "weights_dy", "weights_st", "alpha", "weights")
  loss = sum((out[k] * gr[:, c]).sum() for k, c in ray_keys) + sum((out[k] * gs[i]).sum() for i, k in enumerate(samp_keys))
  loss.backward()
  torch.cuda.synchronize()
  tag = "ag-" + ("vanilla" if vanilla else "composite")
  for k, c in ray_keys:
    _check(tag, "comp_rays", out[k].detach().cpu(), ref["rays"][:, c], ref["rays_mag"][:, c], ref["rays_sens"][:, c])
  assert torch.equal(out["mask"].cpu().double(), ref["rays"][:, -1]), tag
  for i, k in enumerate(samp_keys):
    _check(tag, "comp_samples", out[k].detach().cpu(), ref["samples"][i], ref["samples_mag"][i], ref["samples_sens"][i])
  _check(tag, "comp_grad", ra.grad.cpu(), ref["g_raw_a"], ref["g_raw_a_mag"], ref["g_raw_a_sens"])
  if not vanilla:
    _check(tag, "comp_grad", rb.grad.cpu(), ref["g_raw_b"], ref["g_raw_b_mag"], ref["g_raw_b_sens"])


def test_composite_backward_refuses_more_than_256_samples():
  R, S = 3, 257
  x = torch.zeros(R, S, 4, device=DEV)
  z = torch.ones(R, S, device=DEV)
  g = torch.zeros(R, 11, device=DEV)
  assert lib.dyn_composite_backward(ptr(x), ptr(x), ptr(z), ptr(g), None, R, S, ptr(x), ptr(x), None) != 0
  assert lib.dyn_composite_vanilla_backward(ptr(x), ptr(z), ptr(g), None, R, S, ptr(x), None) != 0


# ----------------------------------------------------------------------------------------------------------------
# optical flow
# ----------------------------------------------------------------------------------------------------------------
def _run_flow(case):
  d = lambda t: t.to(DEV)
  w = d(case["weights"]).requires_grad_(True)
  p = d(case["pts_seq"]).requires_grad_(True)
  fl = ag.optical_flow(w, p, case["cams"][None], d(case["uv"]))
  (fl * d(case["g_flows"])).sum().backward()
  torch.cuda.synchronize()
  return fl.detach().cpu(), w.grad.cpu(), p.grad.cpu()


@pytest.mark.parametrize("n_flow,S", [(1, 1), (6, 33), (16, 128), (1, 256), (16, 256), (6, 128)])
def test_flow_forward_backward(n_flow, S):
  case = G.flow_case(n_flow, 5, S, seed=n_flow * 7 + S, close_to_camera=True, zero_weights=True)
  ref = G.flow(case)
  fl, gw, gp = _run_flow(case)
  tag = "n%d_S%d" % (n_flow, S)
  k = ref["flow_kink"]
  _check(tag, "flow", fl, ref["flows"], ref["flows_mag"], ref["flows_sens"], kink=k, max_kink=0)
  _check(tag, "flow_g_w", gw, ref["g_weights"], ref["g_weights_mag"], ref["g_weights_sens"])
  _check(tag, "flow_g_pts", gp, ref["g_pts"], ref["g_pts_mag"], ref["g_pts_sens"])


def test_flow_backward_refuses_more_than_256_samples():
  R, S = 2, 257
  case = G.flow_case(2, R, S, seed=1)
  d = lambda t: t.to(DEV).contiguous()
  gw, gp = torch.empty(R, S, device=DEV), torch.empty(2, R, S, 3, device=DEV)
  rc = lib.dyn_flow_backward(ptr(d(case["weights"])), ptr(d(case["pts_seq"])), case["cams"].contiguous().data_ptr(),
                             ptr(d(case["g_flows"])), 2, R, S, ptr(gw), ptr(gp), None)
  assert rc != 0


def test_flow_with_no_views_has_zero_gradients():
  """An empty view dimension: no flows, and the weights' gradient is zero, not uninitialised memory."""
  case = G.flow_case(1, 4, 20, seed=3)
  w = case["weights"].to(DEV).requires_grad_(True)
  p = torch.empty(0, 4, 20, 3, device=DEV).requires_grad_(True)
  fl = ag.optical_flow(w, p, case["cams"][None], case["uv"].to(DEV))
  assert fl.shape == (0, 4, 2)
  junk = torch.full((4, 20), float("nan"), device=DEV)  # a freed block the gradient's allocation may reuse
  del junk
  fl.sum().backward()
  assert torch.equal(w.grad.cpu(), torch.zeros(4, 20))


# ----------------------------------------------------------------------------------------------------------------
# resampling
# ----------------------------------------------------------------------------------------------------------------
RESAMPLE = [(3, 2), (32, 16), (64, 64), (128, 128), (128, 384), (64, 2), (3, 128)]


@pytest.mark.parametrize("det", [True, False], ids=["det", "u"])
@pytest.mark.parametrize("inv_uniform", [0, 1])
@pytest.mark.parametrize("S,Ni", RESAMPLE)
def test_resample(S, Ni, inv_uniform, det):
  from dynibar_b200 import render_ray as rr
  R = 6
  case = G.resample_case(R, S, Ni, seed=S * 3 + Ni + 7 * inv_uniform + det, det=det, inv_uniform=inv_uniform,
                         special=True)
  ref = G.resample(case)
  u = None if det else case["u"].to(DEV)
  out = rr.resample_depths(case["z"].to(DEV), case["weights"].to(DEV), Ni, inv_uniform, det, u).cpu()
  tag = "S%d_Ni%d_inv%d_%s" % (S, Ni, inv_uniform, "det" if det else "u")
  assert (out[:, 1:] >= out[:, :-1]).all(), tag
  n_kink = int(ref["kink"].sum())
  M = S - 2
  if det:
    # the all-zero ray's cdf is i / M, and the interior linspace point k / (Ni - 1) lies on it when M k is a
    # multiple of Ni - 1; the single-spike ray's empty bins put den within rounding of 1e-5, and u = 0 and u = 1
    # land in two of them
    allowed = sum(1 for k in range(1, Ni - 1) if (M * k) % (Ni - 1) == 0) + 2
  else:
    # one ray puts min(Ni - 2, M - 1) of its u on cdf entries; u = 0 and u = 1 of the single-spike ray as above
    allowed = min(Ni - 2, M - 1) + 2
  # plus chance coincidences in the random rays: each cdf entry is known to about (i + M / 32 + 8) 2^-24, so a u lands
  # within rounding of one with probability ~ 1e-3 at M = 126 (about one expected over 3 rays x 384 u)
  allowed += 3
  assert n_kink <= allowed, (tag, n_kink, allowed)
  bad, worst = G.resample_check(case, ref, out)
  assert not bad, (tag, bad)
  _WORST["resample"] = max(_WORST.get("resample", -1e30), worst)
