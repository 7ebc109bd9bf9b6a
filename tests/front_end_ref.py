"""Float64 reference of the fp32 ray front end (csrc/geometry.cu): dyn_sample_rays, dyn_points_from_depths,
dyn_traj_displace, dyn_traj_delta, dyn_occlusion_weights, dyn_plucker_ref, dyn_plucker_src, dyn_compute_angle and
dyn_compute_projections.

The formulas are the oracle's (oracle/dynibar_oracle.py: sample_along_ray, z_to_s, traj_offset, displaced_points,
plucker_ref, plucker_src, ray_angle_diff, project_points, and the occlusion weights of _cross_time), evaluated on the
fp32 values the kernels read.  They round where the kernels do and nowhere else: the projection matrix is K inv(c2w)
rounded to fp32 (build_view_cams, geometry_stage_ref.view_P), and the constants 1e-12 (the normalize floor) and 1e-8
(the pz clamp) are their fp32 values.  z of sample_rays is the exception: the kernel reproduces the reference's fp32
operation order with explicit roundings, so its z is compared bit for bit with the oracle evaluated in fp32.

Every function takes `dt`: torch.float64 is the reference, torch.float32 the same formulas in fp32 (which must stay
within the bars, test_front_end_reference_cpu.py).  Each output comes with `mag`, the sum of the absolute values of the
terms it is formed from, scaled by the conditioning of a normalization where there is one, so that the bar is
    |got - ref| <= atol + ulps (ulp(ref) + 2^-24 mag)                       (geometry_stage_ref.bar)
with ulps the measured constant of TOL.  Kinks (the normalize floor, pz = 0 and the 1e-8 clamp, the 1e6 clamp) are
flagged within delta and either one-sided value is accepted there; the tests bound how many points are flagged.

`plant` names a deliberate error (PLANTS) used to show that the bars would catch it.
"""

import torch

from geometry_stage_ref import C8, CLAMP, EPS, F32, d64, project, view_P

N12 = F32(1e-12)

PLANTS = (
    "jitter_wrong_neighbour",  # jittered interval: upper mid-point taken from i - 1
    "basis_drop_last",         # trajectory sums miss the basis term k = nb - 1
    "frame_no_wrap",           # a negative frame index clamped to 0 instead of wrapping
    "occ_first_32",            # occlusion map summed over the first 32 samples only
    "moment_swapped",          # Plucker moment d x o instead of o x d
    "st_stride",               # compute_angle: static point of view 0 for every view
    "s_vals_far_near",         # s_vals denominator 1/near - 1/far
    "angle_dot_unnormalized",  # compute_angle: a . b from the unnormalized vectors
    "pts_o_dropped",           # points_from_depths without ray_o
)

# output -> (atol, ulps).  atol is the smallest normal fp32 number.  ulps: 2x the worst
# (err - atol) / (ulp + 2^-24 mag) measured over every case of test_front_end_gpu.py on an NVIDIA H100 80GB HBM3
# (SXM) at its 700 W power limit, with the worst value beside each.
TOL = {
    "pts": (2.0 ** -126, 0.98),       # sample_rays / points_from_depths; worst 0.488
    "s_vals": (2.0 ** -126, 0.34),    # worst 0.168
    "traj": (2.0 ** -126, 1.7),       # traj_displace, traj_delta; worst 0.838
    "occ": (2.0 ** -126, 0.52),       # occ_weights, occ_weight_map; worst 0.258
    "plucker_d": (2.0 ** -126, 0.62), # worst 0.307
    "plucker_m": (2.0 ** -126, 0.22), # worst 0.108
    "angle": (2.0 ** -126, 0.32),     # compute_angle; worst 0.158
    "pix": (2.0 ** -126, 0.38),       # compute_projections outside the flagged kinks; worst 0.187
}


def _t(x, dt):
  return d64(x).to(dt)


def wrap(f, T):
  """Python indexing of the [T, nb] basis: -T <= f < T."""
  if f < -T or f >= T:
    raise IndexError(f)
  return f + T if f < 0 else f


# ---- sample_rays / points_from_depths ------------------------------------------------------------------------------
def sample_z32(near, far, S, inv_uniform, jitter=None, plant=None):
  """z of sample_along_ray in fp32 (the kernel's rounding order) -> [R or 1, S] fp32."""
  n, f = torch.tensor(near, dtype=torch.float32), torch.tensor(far, dtype=torch.float32)
  if inv_uniform:
    start = 1.0 / n
    step = (1.0 / f - start) / (S - 1)
    z = 1.0 / torch.stack([start + i * step for i in range(S)])[None]
  else:
    step = (f - n) / (S - 1)
    z = torch.stack([n + i * step for i in range(S)])[None]
  if jitter is not None:
    mids = 0.5 * (z[:, 1:] + z[:, :-1])
    upper = torch.cat([mids, z[:, -1:]], -1)
    if plant == "jitter_wrong_neighbour":
      upper = torch.cat([z[:, :1], mids], -1)
    lower = torch.cat([z[:, :1], mids], -1)
    z = lower + (upper - lower) * jitter
  return z


def points_s(ray_o, ray_d, z, near, far, dt=torch.float64, plant=None):
  """pts = z d + o and s = (1/z - 1/near) / (1/far - 1/near) on the fp32 z -> dict(pts, pts_mag, s, s_mag)."""
  o, d, z = _t(ray_o, dt), _t(ray_d, dt), _t(z, dt)
  zd = z[..., None] * d[:, None, :]
  pts = zd if plant == "pts_o_dropped" else zd + o[:, None, :]
  inv_n, inv_f = 1.0 / torch.tensor(F32(near), dtype=dt), 1.0 / torch.tensor(F32(far), dtype=dt)
  den = (inv_n - inv_f) if plant == "s_vals_far_near" else (inv_f - inv_n)
  iz = 1.0 / z  # z = 0 gives inf, as in the kernel
  s = (iz - inv_n) / den
  s_mag = 4.0 * ((iz.abs() + inv_n.abs()) / den.abs() + s.abs() * (inv_f.abs() + inv_n.abs()) / den.abs())
  return dict(pts=pts, pts_mag=2.0 * (zd.abs() + o[:, None, :].abs()), s=s, s_mag=s_mag)


# ---- trajectories ---------------------------------------------------------------------------------------------------
def _traj(c, row, nb, plant):
  """sum_k c[ax nb + k] row[k] per axis -> (value [..., 3], sum of |terms| [..., 3])."""
  cc = c.reshape(c.shape[:-1] + (3, nb))
  terms = cc * row
  if plant == "basis_drop_last":
    terms = terms[..., :nb - 1]
  return terms.sum(-1), terms.abs().sum(-1)


def traj_displace(pts, coeff, basis, frame_idx, offsets, num_vv, dt=torch.float64, plant=None):
  """pts_seq [n_off + num_vv, R, S, 3] = pts + (traj(f + o) - traj(f)), then num_vv copies of pts -> (seq, mag)."""
  T, nb = basis.shape
  p, c, b = _t(pts, dt), _t(coeff, dt), _t(basis, dt)
  fr = lambda f: (0 if f < 0 else f) if plant == "frame_no_wrap" else wrap(f, T)
  t0, a0 = _traj(c, b[fr(frame_idx)], nb, plant)
  seq, mag = [], []
  for o in offsets:
    t, a = _traj(c, b[fr(frame_idx + o)], nb, plant)
    seq.append(p + (t - t0))
    mag.append(nb * (a + a0) + p.abs())
  seq += [p] * num_vv
  mag += [torch.zeros_like(p)] * num_vv
  return torch.stack(seq), torch.stack(mag)


def traj_delta(coeff, basis, frames_a, frames_b, dt=torch.float64, plant=None):
  """traj(frames_a[v]) - traj(frames_b[v]) -> ([n, R, S, 3], mag)."""
  T, nb = basis.shape
  c, b = _t(coeff, dt), _t(basis, dt)
  fr = lambda f: (0 if f < 0 else f) if plant == "frame_no_wrap" else wrap(f, T)
  out, mag = [], []
  for fa, fb in zip(frames_a, frames_b):
    ta, aa = _traj(c, b[fr(fa)], nb, plant)
    tb, ab = _traj(c, b[fr(fb)], nb, plant)
    out.append(ta - tb)
    mag.append(nb * (aa + ab))
  return torch.stack(out), torch.stack(mag)


# ---- occlusion weights ----------------------------------------------------------------------------------------------
def occlusion(w_ref, w_anchor, dt=torch.float64, plant=None):
  """occ = 1 - |w_ref - w_anchor|, occ_map = 1 - |sum_s (w_ref - w_anchor)| -> dict(occ, occ_mag, map, map_mag)."""
  a, b = _t(w_ref, dt), _t(w_anchor, dt)
  d = a - b
  S = d.shape[-1]
  summed = d[:, :32] if plant == "occ_first_32" else d
  chain = -(-S // 32) + 5
  return dict(occ=1.0 - d.abs(), occ_mag=1.0 + a.abs() + b.abs(), map=1.0 - summed.sum(-1).abs(),
              map_mag=1.0 + chain * (a.abs() + b.abs()).sum(-1))


# ---- Plucker coordinates and ray angles ----------------------------------------------------------------------------
def normalize(v, mag_v):
  """v / max(|v|, 1e-12) with the relative conditioning of the result: mag_v / |v| (mag_v: the absolute error scale
  of v's components in units of 2^-24) -> (unit vector, its mag, |v|)."""
  n = v.norm(dim=-1, keepdim=True)
  u = v / n.clamp(min=N12)
  return u, 4.0 * (1.0 + mag_v / n.clamp(min=N12)), n[..., 0]


def _cross(a, b, plant):
  return torch.linalg.cross(b, a, dim=-1) if plant == "moment_swapped" else torch.linalg.cross(a, b, dim=-1)


def plucker_ref(ray_o, ray_d, dt=torch.float64, plant=None):
  """[normalize(d), o x normalize(d)] -> dict(out [R,6], mag [R,6], norm [R] (|d|, for the 1e-12 kink))."""
  o, d = _t(ray_o, dt), _t(ray_d, dt)
  dn, dmag, n = normalize(d, 0.0 * d.abs().sum(-1, keepdim=True))
  m = _cross(o, dn, plant)
  mmag = 4.0 * o.norm(dim=-1, keepdim=True) * (dn.norm(dim=-1, keepdim=True) * dmag)
  return dict(out=torch.cat([dn, m], -1), mag=torch.cat([dmag.expand_as(dn), mmag.expand_as(m)], -1), norm=n)


def cam_centres(cams):
  return d64(cams).reshape(-1, 34)[:, 18:34].reshape(-1, 4, 4)[:, :3, 3]


def plucker_src(pts, src_cams, dt=torch.float64, plant=None):
  """pts [R,S,3], src_cams [V,34] -> dict(out [R,S,V,6], mag, norm [R,S,V])."""
  o = cam_centres(src_cams).to(dt)[:, None, None, :]
  p = _t(pts, dt)[None]
  v = p - o
  dn, dmag, n = normalize(v, (p.abs() + o.abs()).sum(-1, keepdim=True))
  m = _cross(o.expand_as(dn), dn, plant)
  mmag = 4.0 * o.norm(dim=-1, keepdim=True) * dmag * (n[..., None] > 0)
  out = torch.cat([dn, m], -1).permute(1, 2, 0, 3)
  mag = torch.cat([dmag.expand_as(dn), mmag.expand_as(m)], -1).permute(1, 2, 0, 3)
  return dict(out=out, mag=mag, norm=n.permute(1, 2, 0))


def compute_angle(xyz_st, xyz, query_cam, src_cams, dt=torch.float64, plant=None):
  """xyz_st [st_views, N, 3], xyz [V, N, 3] -> dict(out [V,N,4], mag, kink norms na, nb, nd [V,N])."""
  tgt = d64(query_cam).reshape(-1)[18:34].reshape(4, 4)[:3, 3].to(dt)
  src = cam_centres(src_cams).to(dt)[:, None, :]
  s, q = _t(xyz_st, dt), _t(xyz, dt)
  if plant == "st_stride":
    s = s[:1]
  s = s.expand_as(q)
  va, vb = tgt - s, src - q
  a, amag, na = normalize(va, (tgt.abs() + s.abs()).sum(-1, keepdim=True))
  b, bmag, nb_ = normalize(vb, (src.abs() + q.abs()).sum(-1, keepdim=True))
  dot = ((va * vb).sum(-1, keepdim=True) if plant == "angle_dot_unnormalized" else (a * b).sum(-1, keepdim=True))
  d, dmag, nd = normalize(a - b, amag + bmag)
  out = torch.cat([d, dot], -1)
  mag = torch.cat([dmag.expand_as(d), amag + bmag + 3.0], -1)
  return dict(out=out, mag=mag, na=na, nb=nb_, nd=nd)


def compute_projections(xyz, src_cams, plant=None):
  """xyz [V, N, 3] -> dict(pix [V,N,2], front [V,N], mag [V,N,2], flag [V,N] (a kink within delta)), always float64:
  the bounds come from geometry_stage_ref.project."""
  P = view_P(src_cams)
  pr = project(P, d64(xyz))
  pix = torch.stack([pr["u"], pr["v"]], -1)
  # the bar's mag from project()'s first-order bound: du = DELTA (...) in absolute terms -> in units of 2^-24
  mag = torch.stack([pr["du"], pr["dv"]], -1) / EPS
  flag = (pr["pz"].abs() <= pr["dpz"]) | ((pr["pz"] - C8).abs() <= pr["dpz"])
  for c0, dc in ((pr["u0"], pr["du"]), (pr["v0"], pr["dv"])):
    flag |= (c0.abs() - CLAMP).abs() <= 4 * EPS * c0.abs() + dc
  return dict(pix=pix, front=pr["pz"] > 0, mag=mag, flag=flag, pr=pr)
