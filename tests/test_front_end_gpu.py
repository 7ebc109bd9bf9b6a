"""The fp32 ray front end (csrc/geometry.cu: sample_rays, points_from_depths, traj_displace, traj_delta,
occlusion_weights, plucker_ref, plucker_src, compute_angle, compute_projections) against the float64 reference of
tests/front_end_ref.py, at the edges where these kernels go wrong: V = 32 views, nb = 8 basis terms, 32 displaced
rows, wrapped frame indices, S > 32 in the warp-per-ray occlusion sum, zero-length directions, points at a camera
centre, on or behind a camera plane and beyond the 1e6 clamp.  Bars: front_end_ref.TOL; the worst excess per
output is printed (pytest -s)."""

import math

import pytest
import torch

import front_end_ref as FE
from geometry_stage_ref import bar, excess, rig

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WORST = {}


def _check(name, got, ref, mag, skip=None):
  got = got.detach().cpu().double()
  ref, mag = ref.double(), mag.double().expand_as(ref)
  fin = torch.isfinite(ref)
  assert torch.equal(torch.isfinite(got), fin), "%s: non-finite pattern differs" % name
  assert torch.equal(got[~fin], ref[~fin]), "%s: non-finite values differ" % name
  keep = fin if skip is None else fin & ~skip
  g, r, m = got[keep], ref[keep], mag[keep]
  if g.numel() == 0:
    return
  x = excess(name, g, r, m, 0.0, tol=FE.TOL)
  WORST[name] = max(WORST.get(name, -math.inf), x.max().item())
  bad = (g - r).abs() > bar(name, r, m, 0.0, tol=FE.TOL)
  assert not bad.any(), "%s: %d of %d over the bar, worst excess %.3g (bar %.3g): got %r want %r" % (
      name, int(bad.sum()), bad.numel(), x.max().item(), FE.TOL[name][1], g[bad][0].item(), r[bad][0].item())


@pytest.fixture(scope="module", autouse=True)
def report():
  yield
  print("\n[front end] worst excess (ulps): " + ", ".join("%s %.3g" % kv for kv in sorted(WORST.items())))


def rr():
  from dynibar_b200 import render_ray
  return render_ray


def rays(R, seed, scale=1.0):
  g = torch.Generator().manual_seed(seed)
  return torch.randn(R, 3, generator=g) * scale, torch.randn(R, 3, generator=g)


# ---- sample_rays / points_from_depths -----------------------------------------------------------------------------
@pytest.mark.parametrize("S", [2, 3, 64, 128, 384])
@pytest.mark.parametrize("inv_uniform", [False, True])
@pytest.mark.parametrize("jit", ["det", "rand", "edges"])
def test_sample_rays(S, inv_uniform, jit):
  R = 37
  o, d = rays(R, S)
  for near, far in ((0.7, 41.0), (1e-3, 1e4)):
    jitter = None
    if jit == "rand":
      jitter = torch.rand(R, S, generator=torch.Generator().manual_seed(S))
    elif jit == "edges":  # exactly 0 and the largest draw below 1
      jitter = torch.where(torch.arange(R * S).reshape(R, S) % 2 == 0, 0.0, 1.0 - 2.0 ** -24)
    pts, z, s = rr().sample_along_camera_ray(o.to(DEV), d.to(DEV), torch.tensor([[near, far]], device=DEV), S,
                                             inv_uniform, jit == "det", None if jitter is None else jitter.to(DEV))
    want_z = FE.sample_z32(near, far, S, inv_uniform, jitter).expand(R, S)
    assert torch.equal(z.cpu(), want_z), "z must equal the fp32 restatement bit for bit"
    ref = FE.points_s(o, d, z.cpu(), near, far)
    _check("pts", pts, ref["pts"], ref["pts_mag"])
    _check("s_vals", s, ref["s"], ref["s_mag"])


def test_sample_rays_refuses_one_sample_and_an_empty_range():
  o, d = (t.to(DEV) for t in rays(4, 0))
  with pytest.raises(RuntimeError, match="S >= 2"):
    rr().sample_along_camera_ray(o, d, torch.tensor([[1.0, 2.0]], device=DEV), 1, False, True)
  for near, far in ((2.0, 2.0), (3.0, 2.0)):
    with pytest.raises((AssertionError, RuntimeError)):
      rr().sample_along_camera_ray(o, d, torch.tensor([[near, far]], device=DEV), 8, False, True)


@pytest.mark.parametrize("S", [1, 5, 64])
def test_points_from_depths_with_zero_and_huge_depths(S):
  R = 29
  o, d = rays(R, 100 + S)
  z = torch.rand(R, S, generator=torch.Generator().manual_seed(S)) * 50.0
  z[0] = 0.0
  z[1] = 1e30
  z[2] = 1e-30
  pts, s = rr().points_from_depths(o.to(DEV), d.to(DEV), z.to(DEV), torch.tensor([[0.5, 60.0]], device=DEV))
  ref = FE.points_s(o, d, z, 0.5, 60.0)
  assert not torch.isfinite(ref["s"][0]).any()
  _check("pts", pts, ref["pts"], ref["pts_mag"])
  _check("s_vals", s, ref["s"], ref["s_mag"])


# ---- trajectories --------------------------------------------------------------------------------------------------
def _traj_inputs(R, S, T, nb, seed):
  g = torch.Generator().manual_seed(seed)
  return (torch.randn(R, S, 3, generator=g) * 3.0, torch.randn(R, S, 3 * nb, generator=g),
          torch.randn(T, nb, generator=g))


@pytest.mark.parametrize("nb", range(1, 9))
def test_traj_displace(nb):
  T, R, S = 12, 9, 33
  pts, coeff, basis = _traj_inputs(R, S, T, nb, nb)
  cases = [(0, [-3, -2, -1, 1, 2, 3], 2), (T - 1, [-T + 1 - T, -1, 0, -T], 0),  # frames -T, T-2, T-1, -1
           (-1, list(range(-T + 1, 1)) + list(range(0, T - 12 + 1)), 32 - T - 1), (5, [], 4)]
  for f, offs, vv in cases:
    n = len(offs) + vv
    assert n <= 32
    got = rr().displaced_points(pts.to(DEV), coeff.to(DEV), basis, f, offs, vv)
    want, mag = FE.traj_displace(pts, coeff, basis, f, offs, vv)
    _check("traj", got, want, mag)
    assert torch.equal(got[len(offs):].cpu(), pts[None].expand(vv, -1, -1, -1)), "virtual-view rows must be pts"


def test_traj_displace_refuses_bad_frames_and_sizes():
  T = 6
  pts, coeff, basis = _traj_inputs(2, 3, T, 4, 0)
  p, c = pts.to(DEV), coeff.to(DEV)
  for f, offs in ((0, [T]), (0, [-T - 1]), (T, [0]), (-T - 1, [])):
    with pytest.raises(RuntimeError):
      rr().displaced_points(p, c, basis, f, offs)
  _, c9, b9 = _traj_inputs(2, 3, T, 9, 0)
  with pytest.raises(RuntimeError):
    rr().displaced_points(p, c9.to(DEV), b9, 0, [1])
  with pytest.raises(RuntimeError):
    rr().displaced_points(p, c, basis, 0, [1] * 30, 3)


@pytest.mark.parametrize("n", range(1, 9))
def test_traj_delta(n):
  T, nb = 10, 8
  _, coeff, basis = _traj_inputs(7, 40, T, nb, 50 + n)
  fa = [-T + 2 * v for v in range(n)]
  fb = [(T - 1 - 2 * v) if v % 2 else -1 - v for v in range(n)]
  got = rr().traj_deltas(coeff.to(DEV), basis, fa, fb)
  want, mag = FE.traj_delta(coeff, basis, fa, fb)
  _check("traj", got, want, mag)


# ---- occlusion weights ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 31, 32, 33, 64, 256, 384])
def test_occlusion_weights(S):
  R = 8 * 5 + 3  # not a multiple of the 8 rays of a 256-thread block
  g = torch.Generator().manual_seed(S)
  a, b = torch.rand(R, S, generator=g) / S * 2, torch.rand(R, S, generator=g) / S * 2
  b[::4] = a[::4]  # w_ref == w_anchor: exactly 1
  occ, occ_map = rr().occlusion_weights(a.to(DEV), b.to(DEV))
  ref = FE.occlusion(a, b)
  _check("occ", occ, ref["occ"], ref["occ_mag"])
  _check("occ", occ_map, ref["map"], ref["map_mag"])
  assert (occ[::4] == 1).all() and (occ_map[::4] == 1).all()


# ---- Plucker coordinates -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [1.0, 1e3])
def test_plucker_ref(scale):
  o, d = rays(300, 7, scale)
  o = o + scale
  d[::7] = 0.0  # zero directions: F.normalize gives 0
  got = rr().compute_ref_plucker_coordinate(o.to(DEV), d.to(DEV))
  ref = FE.plucker_ref(o, d)
  _check("plucker_d", got[:, :3], ref["out"][:, :3], ref["mag"][:, :3])
  _check("plucker_m", got[:, 3:], ref["out"][:, 3:], ref["mag"][:, 3:])
  assert (got[::7] == 0).all()


@pytest.mark.parametrize("V", [1, 8, 32])
@pytest.mark.parametrize("scale", [1.0, 1e3])
def test_plucker_src(V, scale):
  cams, _ = rig(V, 40, 60, V, radius=4.0 * scale)
  R, S = 11, 37
  pts = torch.randn(R, S, 3, generator=torch.Generator().manual_seed(V)) * scale
  centres = FE.cam_centres(cams).float()
  pts[0, :V] = centres[:S][:min(V, S)]  # points at a source camera centre
  got = rr().compute_src_plucker_coordinate(pts.to(DEV), cams[None].to(DEV))
  ref = FE.plucker_src(pts, cams)
  _check("plucker_d", got[..., :3], ref["out"][..., :3], ref["mag"][..., :3])
  _check("plucker_m", got[..., 3:], ref["out"][..., 3:], ref["mag"][..., 3:])
  for v in range(min(V, S)):
    assert (got[0, v, v] == 0).all()


# ---- compute_angle / compute_projections ---------------------------------------------------------------------------
@pytest.mark.parametrize("st_views", ["one", "V"])
def test_compute_angle(st_views):
  from dynibar_b200.projection import Projector
  V, N = 32, 500
  cams, query = rig(V, 40, 60, 3)
  tgt = FE.cam_centres(query)[0].float()
  g = torch.Generator().manual_seed(9)
  xyz = torch.randn(V, N, 3, generator=g)
  xst = torch.randn(V if st_views == "V" else 1, N, 3, generator=g)
  src = FE.cam_centres(cams).float()
  xst[:, 0] = tgt               # a static point at the target centre
  xyz[:, 1] = src                # a point at its source centre
  xyz[:, 2:40] = xst[:, 2:40] + 1e-4 * torch.randn(xst[:, 2:40].shape, generator=g)  # a ~ b when centres coincide
  cams[5, 18 + 3], cams[5, 18 + 7], cams[5, 18 + 11] = tgt[0], tgt[1], tgt[2]  # view 5 sits at the target centre
  got = Projector(torch.device(DEV)).compute_angle(xst.to(DEV), xyz.to(DEV), query.to(DEV), cams.to(DEV))
  ref = FE.compute_angle(xst, xyz, query, cams)
  _check("angle", got, ref["out"], ref["mag"])


def test_compute_projections():
  from dynibar_b200.projection import Projector
  V, N = 32, 4000
  cams, _ = rig(V, 40, 60, 11)
  g = torch.Generator().manual_seed(11)
  xyz = torch.randn(V, N, 3, generator=g) * 6.0  # about half behind the cameras (radius 4)
  xyz[:, :50] *= 1e4                              # far off: beyond the 1e6 clamp
  # points on each camera's plane: pz = 0 up to the fp32 rounding of the point
  P = FE.view_P(cams)
  for v in range(V):
    q = xyz[v, 50:80].double()
    n = P[v, 2, :3]
    q = q - (((q @ n) + P[v, 2, 3]) / (n @ n))[:, None] * n
    xyz[v, 50:80] = q.float()
  pix, front = Projector(torch.device(DEV)).compute_projections(xyz.to(DEV), cams.to(DEV))
  ref = FE.compute_projections(xyz, cams)
  flag = ref["flag"]
  assert int(flag.sum()) <= 40 * V, int(flag.sum())
  _check("pix", pix, ref["pix"], ref["mag"], skip=flag[..., None].expand_as(ref["pix"]))
  assert torch.equal(front.cpu()[~flag], ref["front"][~flag])
  # flagged points: either one-sided value of the clamps
  pr = ref["pr"]
  got = pix.cpu().double()[flag]
  sides = [torch.stack([pr[c0] / dd for c0 in ("px", "py")], -1)[flag].clamp(-FE.CLAMP, FE.CLAMP)
           for dd in (pr["pz"].clamp(min=FE.C8), torch.full_like(pr["pz"], FE.C8))]
  sides += [torch.full_like(got, FE.CLAMP), torch.full_like(got, -FE.CLAMP)]
  ok = torch.zeros_like(got, dtype=torch.bool)
  for s in sides:
    ok |= (got - s).abs() <= bar("pix", s, ref["mag"][flag], 0.0, tol=FE.TOL) + 1e-3 * s.abs()
  assert ok.all()
