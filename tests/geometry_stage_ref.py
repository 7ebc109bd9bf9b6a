"""Float64 reference of the fp32 glue between the network stages: projection + bilinear gather (csrc/geometry.cu
project_gather_kernel) and its backward (csrc/backward.cu gather_backward_kernel), compositing forward and
backward (composite_kernel, composite_backward_kernel), optical flow forward and backward (flow_sf_kernel,
flow_backward_kernel) and hierarchical resampling (resample_kernel).

The formulas are the oracle's (oracle/dynibar_oracle.py: project_points, bilinear_gather, ray_angle_diff,
composite, composite_vanilla, optical_flow, sample_pdf, resample_depths), evaluated in float64 on the fp32
values the kernels read.  The reference rounds where the kernels do and nowhere else:
  - the projection matrix is K inv(c2w) formed in float64 and rounded to fp32 (build_view_cams);
  - the flow's Kc, Rw = inv(c2w)[:3,:3] and tw = inv(c2w)[:3,3] are rounded to fp32 (build_flow_cams);
  - the constants 1e-8, 1e-10 and 1e-5 are their fp32 values.
What remains between kernel and reference is the kernels' own fp32 arithmetic.

Each compared output carries a bar
    |got - ref| <= atol + ulps * (ulp(ref) + 2^-24 mag) + sens
  - mag: the sum of the absolute values of the terms the kernel adds (times the length of its longest addition
    chain for the warp scans and sums), so that ulps counts fp32 roundings per term;
  - sens: the first-order effect of the kernel's fp32 error in the quantities an output is sensitive to: the
    bilinear gradient times the coordinate bound delta for gathered values, |q| / q2^2 times the error of q for
    flows, the alpha error through the transmittance scan (a Jacobian computed in float64) for compositing.
ulps is the only measured constant per output: TOL gives it at 2x the worst (err - atol - sens) / (ulp + 2^-24
mag) observed on an H100 SXM (80 GB, 700 W power limit) over every case of tests/test_geometry_stage_gpu.py.

Kinks.  Where an output is discontinuous in a quantity the kernel computes in fp32, an element whose reference
value of that quantity lies within its error bound of the discontinuity is flagged, and the GPU test accepts
either one-sided reference value there:
  1. mask: u in {0, W-1}, v in {0, H-1}, pz = 0 (bound delta_u, delta_v, delta_pz);
  2. d xyz: integer tap coordinates of the feature-map grid and of the image grid (bound delta_fx, delta_fy),
     the 1e-8 clamp of pz and the 1e6 clamp of u, v;
  3. resampling: u at a cdf entry (the inverse-CDF count) and den at 1e-5 (the den < 1e-5 switch);
  4. flow: q2 = 0.
delta is twice the first-order bound of the fp32 evaluation, in which a dot product of n terms errs by at most
n 2^-24 sum|terms| and each further operation by 2^-24 of its result (test_geometry_stage_reference_cpu.py checks
that an fp32 emulation of the projection stays within delta / 4).

`plant` names a deliberate error (PLANTS) used to show that the bars would catch it.
"""

import contextlib
import math

import torch
import torch.nn.functional as F

from oracle import dynibar_oracle as O

EPS = 2.0 ** -24
F32 = lambda x: float(torch.tensor(x, dtype=torch.float32))
C8, C10, C5 = F32(1e-8), F32(1e-10), F32(1e-5)
CLAMP = 1e6  # exact in fp32
DELTA = 2.0  # delta is twice the first-order worst-case bound: room for second-order terms and FMA contraction

PLANTS = (
    "mask_right_exclusive",   # mask: u < W-1 instead of u <= W-1
    "feat_norm_by_map",       # feature coordinates normalised by the feature-map size, not the image size
    "ax_bx_swap",             # bilinear weights ax and bx swapped
    "dxyz_no_p8",             # d xyz: the -u P[8+k] term dropped
    "pz_clamp_grad_kept",     # d xyz: gradient through pz kept where the 1e-8 clamp is active
    "composite_no_1e10",      # compositing: the + 1e-10 of 1 - alpha + 1e-10 dropped
    "last_delta_one",         # compositing: last sample's delta = 1 instead of 1e10
    "T_inclusive",            # compositing: inclusive instead of exclusive transmittance
    "suffix_off_by_one",      # compositing backward: the suffix sum includes the sample itself
    "flow_Rw_transposed",     # flow backward: Rw instead of Rw^T
    "cdf_M_plus_1",           # inverse CDF counts all M+1 cdf entries
    "den_threshold_dropped",  # inverse CDF: den < 1e-5 -> 1 rule dropped
)

# Bars of the GPU test: output -> (atol, ulps).  atol is the smallest normal fp32 number, so an exact zero
# passes against a reference that is zero; everything else is in ulps (see the module docstring).  ulps is 2x
# the worst (err - atol - sens) / (ulp + 2^-24 mag) measured over every case of test_geometry_stage_gpu.py on an
# NVIDIA H100 80GB HBM3 (SXM) at its 700 W power limit, and 1 where that worst value was <= 0 (the sens term
# alone covered every error).
TOL = {
    "rgb_feat": (2.0 ** -126, 1.0),      # gathered colours + features; worst -4.3
    "ray_diff": (2.0 ** -126, 1.7),      # normalize(a - b), a . b; worst 0.82
    "g_maps": (2.0 ** -126, 1.0),        # atomic scatter into the feature maps; worst -39
    "g_xyz": (2.0 ** -126, 1.0),         # d displaced points; worst -4.6
    "comp_rays": (2.0 ** -126, 0.17),    # rgb, rgb_static, rgb_dy, depth; worst 0.084
    "comp_samples": (2.0 ** -126, 0.15), # alphas and weights; worst 0.072
    "comp_grad": (2.0 ** -126, 26.0),    # d raw (colours and densities); worst 12.7
    "flow": (2.0 ** -126, 1.0),          # worst -3.1
    "flow_g_w": (2.0 ** -126, 1.0),      # worst -0.43
    "flow_g_pts": (2.0 ** -126, 1.0),    # worst -1.7
    "resample": (2.0 ** -126, 1.0),      # fine depths; worst -0.19
}


@contextlib.contextmanager
def float64():
  old = torch.get_default_dtype()
  torch.set_default_dtype(torch.float64)
  try:
    yield
  finally:
    torch.set_default_dtype(old)


def d64(t):
  return t.detach().to("cpu", torch.float64)


def ulp32(x):
  """Spacing of fp32 numbers at |x| (the smallest subnormal at 0)."""
  _, e = torch.frexp(x.abs().float().double())
  return torch.where(x == 0, torch.full_like(x, 2.0 ** -149), torch.ldexp(torch.ones_like(x), (e - 24).clamp(min=-149)))


def bar(name, ref, mag, sens, ulps=None, tol=TOL):
  """atol + ulps (ulp(ref) + 2^-24 mag) + sens, with (atol, ulps) = tol[name]."""
  atol, u = tol[name]
  u = u if ulps is None else ulps
  return atol + u * (ulp32(ref) + EPS * mag) + sens


def excess(name, got, ref, mag, sens, tol=TOL):
  """(err - atol - sens) / (ulp + 2^-24 mag): the measured quantity behind tol[name]'s ulps."""
  atol, _ = tol[name]
  return ((d64(got) - ref).abs() - atol - sens) / (ulp32(ref) + EPS * mag)


# ----------------------------------------------------------------------------------------------------------------
# cameras
# ----------------------------------------------------------------------------------------------------------------
def rig(V, H, W, seed, radius=4.0):
  """V source cameras on an arc around the origin looking at it (small random roll / jitter) and one target
  camera; cameras are [34] fp32 vectors [h, w, K, c2w]."""
  g = torch.Generator().manual_seed(seed)
  with float64():
    f = 0.8 * W
    K = torch.tensor([[f, 0, W / 2.0 + 0.3, 0], [0, f * 1.03, H / 2.0 - 0.2, 0], [0, 0, 1, 0], [0, 0, 0, 1]])

    def cam(yaw, pitch, roll, dist):
      c = torch.tensor([math.sin(yaw) * math.cos(pitch), math.sin(pitch), -math.cos(yaw) * math.cos(pitch)]) * dist
      fwd = -c / c.norm()
      up = torch.tensor([math.sin(roll), math.cos(roll), 0.0])
      right = torch.linalg.cross(up, fwd)
      right = right / right.norm()
      up2 = torch.linalg.cross(fwd, right)
      c2w = torch.eye(4)
      c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, -up2, fwd, c
      return torch.cat([torch.tensor([float(H), float(W)]), K.reshape(-1), c2w.reshape(-1)])

    r = lambda: float(torch.rand(1, generator=g)) - 0.5
    cams = torch.stack([cam(0.5 * (i / max(V - 1, 1) - 0.5) + 0.02 * r(), 0.1 * r(), 0.1 * r(),
                            radius * (1 + 0.05 * r())) for i in range(V)])
    query = cam(0.03, 0.02, 0.0, radius)
  return cams.float(), query.float()


def exact_rig(V, H, W):
  """K with integer entries and c2w = I: P = K[:3] is exact in fp32 and so is u = px / pz for pz a power of 2."""
  K = torch.tensor([[8.0, 0, 20, 0], [0, 8, 12, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
  c = torch.cat([torch.tensor([float(H), float(W)]), K.reshape(-1), torch.eye(4).reshape(-1)])
  return c[None].repeat(V, 1), c.clone()


def view_P(cams, exact=False):
  """build_view_cams: rows 0..2 of K inv(c2w), float64, rounded to fp32 (unless exact) -> [V,3,4] float64."""
  c = d64(cams).reshape(-1, 34)
  K = c[:, 2:18].reshape(-1, 4, 4)
  w2c = torch.linalg.inv(c[:, 18:34].reshape(-1, 4, 4))
  P = (K @ w2c)[:, :3, :]
  return P if exact else P.float().double()


def flow_cams(cams, exact=False):
  """build_flow_cams: Kc = K[:3,:3] (fp32 already), Rw, tw from inv(c2w) in float64 rounded to fp32 (unless
  exact)."""
  c = d64(cams).reshape(-1, 34)
  w2c = torch.linalg.inv(c[:, 18:34].reshape(-1, 4, 4))
  w2c = w2c if exact else w2c.float().double()
  return c[:, 2:18].reshape(-1, 4, 4)[:, :3, :3], w2c[:, :3, :3], w2c[:, :3, 3]


# ----------------------------------------------------------------------------------------------------------------
# projection + bilinear gather
# ----------------------------------------------------------------------------------------------------------------
def project(P, q):
  """P [V,3,4], q [V,N,3] -> dict of px, py, pz, u0, v0 (unclamped), u, v, d = max(pz, 1e-8) and the first-order
  fp32 error bounds du, dv, dpz."""
  terms = P[:, None, :, :3] * q[:, :, None, :]
  p = terms.sum(-1) + P[:, None, :, 3]
  A = terms.abs().sum(-1) + P[:, None, :, 3].abs()
  px, py, pz = p.unbind(-1)
  d = pz.clamp(min=C8)
  u0, v0 = px / d, py / d
  live = pz > C8
  dpz = DELTA * 4 * EPS * A[..., 2]
  out = dict(px=px, py=py, pz=pz, d=d, u0=u0, v0=v0, live=live, dpz=dpz,
             u=u0.clamp(-CLAMP, CLAMP), v=v0.clamp(-CLAMP, CLAMP))
  for c, c0, Ai in (("u", u0, A[..., 0]), ("v", v0, A[..., 1])):
    e = DELTA * ((4 * EPS * (Ai + torch.where(live, c0.abs() * A[..., 2], torch.zeros_like(c0)))) / d + EPS * c0.abs())
    out["d" + c] = torch.where(c0.abs() > CLAMP, torch.zeros_like(e), e)
  return out


def grid_coord(u, du, n_img, n_map):
  """The kernel's chain gx = 2u/(n_img-1) - 1, fx = (gx+1) 0.5 (n_map-1) -> fx and its first-order error bound."""
  t = 2 * u / (n_img - 1.0)
  gx = t - 1
  fx = u * (n_map - 1.0) / (n_img - 1.0)
  dfx = (0.5 * (n_map - 1) * (2 * du / (n_img - 1.0) + DELTA * EPS * (t.abs() + gx.abs() + (gx + 1).abs()))
         + DELTA * EPS * fx.abs())
  return fx, dfx


def _taps(img, fx, fy, x0, y0, plant=None):
  """Bilinear taps of img [V,C,hh,ww] at (fx, fy) [V,N] with cell corners (x0, y0): value, d/dfx, d/dfy,
  cross = d2/dfx dfy, mag = sum |tap * weight|, and the per-tap (index, weight, in-bounds) for the scatter."""
  V, C, hh, ww = img.shape
  ax, ay = fx - x0, fy - y0
  bx, by = x0 + 1 - fx, y0 + 1 - fy
  if plant == "ax_bx_swap":
    ax, bx = bx, ax
  flat = img.reshape(V, C, hh * ww)
  m, taps = [], []
  for dy in (0, 1):
    for dx in (0, 1):
      xi, yi = x0 + dx, y0 + dy
      ok = (xi >= 0) & (xi <= ww - 1) & (yi >= 0) & (yi <= hh - 1)
      idx = (yi.clamp(0, hh - 1) * ww + xi.clamp(0, ww - 1)).long()
      t = torch.gather(flat, 2, idx[:, None, :].expand(V, C, -1)).permute(0, 2, 1) * ok[..., None]
      wgt = (ax if dx else bx) * (ay if dy else by)
      m.append(t)
      taps.append((idx, wgt, ok, (ay if dy else by), (ax if dx else bx)))
  m00, m01, m10, m11 = m
  ax_, ay_, bx_, by_ = (a[..., None] for a in (ax, ay, bx, by))
  val = m00 * bx_ * by_ + m01 * ax_ * by_ + m10 * bx_ * ay_ + m11 * ax_ * ay_
  dfx = (m01 - m00) * by_ + (m11 - m10) * ay_
  dfy = (m10 - m00) * bx_ + (m11 - m01) * ax_
  cross = m11 - m10 - m01 + m00
  mag = (m00 * bx_ * by_).abs() + (m01 * ax_ * by_).abs() + (m10 * bx_ * ay_).abs() + (m11 * ax_ * ay_).abs()
  sumabs = m00.abs() + m01.abs() + m10.abs() + m11.abs()
  return dict(val=val, dfx=dfx, dfy=dfy, cross=cross, mag=mag, sumabs=sumabs, taps=taps)


def _near_int(x, dx):
  return (x - torch.round(x)).abs() <= dx


def gather_case(V, R, S, H, W, h, w, seed, static=False, K=1, spread=1.0):
  """Random points around the origin, displaced per view unless static; K > 1 gives the multi-camera variant with
  a per-ray target camera.  Every third sample is spread 3x wider in x and every fifth 3x wider in y, so that many
  points project beyond the left / right and top / bottom image borders (partial and out-of-image taps)."""
  g = torch.Generator().manual_seed(seed)
  cams, query = rig(V, H, W, seed)
  if K > 1:
    queries = torch.stack([rig(V, H, W, seed + 17 * k)[1] for k in range(K)])
    tgt_idx = torch.randint(0, K, (R,), generator=g, dtype=torch.int32)
  else:
    queries, tgt_idx = query[None], None
  xyz_st = (torch.rand(R, S, 3, generator=g) - 0.5) * 2.4 * spread
  xyz_st[:, 0::3, 0] *= 3.0
  xyz_st[:, 1::5, 1] *= 3.0
  xyz = None if static else xyz_st[None] + 0.05 * torch.randn(V, R, S, 3, generator=g)
  rgbs = torch.rand(V, H, W, 3, generator=g)
  fm = torch.randn(V, 32, h, w, generator=g)
  gfeat = torch.randn(R, S, V, 35, generator=g)
  return dict(cams=cams, queries=queries, tgt_idx=tgt_idx, xyz_st=xyz_st, xyz=xyz, rgbs=rgbs, featmaps=fm,
              g_feat=gfeat, R=R, S=S, V=V)


def exact_case(V=3, H=26, W=42, h=7, w=11):
  """Exact rig (exact_rig) with points on the mask edges and pixel centres, just outside, at fractional pixel
  positions inside, behind the camera, at 0 < pz < 1e-8 and beyond the 1e6 clamp.  u = (8 x + 20 z) / z,
  v = (8 y + 12 z) / z, exact in fp32 for these points.  `on_grid` [S] says which points have an integer image
  coordinate u or v by construction (True: every view must flag them as a d-xyz kink) and which have only
  fractional tap coordinates in both grids (False: no view may flag them)."""
  cams, query = exact_rig(V, H, W)
  pts, on_grid = [], []
  for z in (1.0, 2.0, 0.5):
    for (u, v) in ((0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1), (W - 1, 7), (13, H - 1), (5, 9), (17, 3),
                   (-1, 5), (W, 5), (4, -1), (4, H), (W - 1 + 0.0625, 3), (-0.0625, 3), (3, H - 1 + 0.125)):
      pts.append(((u - 20) * z / 8, (v - 12) * z / 8, z))
      on_grid.append(True)
    # fractional positions inside the image; their feature-map coordinates u (w-1)/(W-1), v (h-1)/(H-1) are not
    # integers either
    for (u, v) in ((5.3125, 9.4375), (0.25, 0.75), (W - 1 - 0.125, H - 1 - 0.375), (19.375, 12.625)):
      pts.append(((u - 20) * z / 8, (v - 12) * z / 8, z))
      on_grid.append(False)
  pts += [(0.1, 0.2, -1.0), (0.0, 0.0, 0.0), (-0.5, 0.3, -1e-3)]          # behind / on the camera plane
  pts += [(0.0, 0.0, 5e-9), (1e-8, 2e-9, 4e-9), (2e-9, -1e-9, 7e-9)]      # 0 < pz < 1e-8: u = (8x + 20z)/1e-8
  pts += [(1e3, 0.0, 1e-3), (-1e3, 0.0, 1e-3), (0.0, 1e3, 1e-4)]          # |u| or |v| > 1e6
  # u, v of these: clamped to -1e6 (both); 0, 0; clamped; 10, 6; 16, 6.4; 15.6, 7.6; 1e6; -1e6; v = 1e6
  on_grid += [True, True, True, True, True, False, True, True, True]
  xyz_st = torch.tensor(pts, dtype=torch.float32)[None]                  # R = 1 ray of all points
  g = torch.Generator().manual_seed(11)
  R, S = 1, xyz_st.shape[1]
  return dict(cams=cams, queries=query[None], tgt_idx=None, xyz_st=xyz_st, xyz=xyz_st[None].repeat(V, 1, 1, 1),
              rgbs=torch.rand(V, H, W, 3, generator=g), featmaps=torch.randn(V, 32, h, w, generator=g),
              g_feat=torch.randn(R, S, V, 35, generator=g), R=R, S=S, V=V, on_grid=torch.tensor(on_grid))


def gather(case, backward=True, rows=None, plant=None, chunk=4096, exact=False):
  """Reference of project_gather_kernel and gather_backward_kernel.  rows: indices of the (ray * S + sample)
  points compared (all when None); g_maps is always formed over all points.

  Returns float64 tensors in the kernels' layouts restricted to `rows` ([n] points): rgb_feat [n,V,35],
  ray_diff [n,V,4], mask [n,V] with rgb_feat_mag / rgb_feat_sens, ray_diff_mag, mask_kink; and with backward:
  g_maps [V,32,h,w] (+ g_maps_mag, g_maps_sens), g_xyz [V,n,3] (+ g_xyz_mag, g_xyz_sens, xyz_kink) and
  g_xyz_alt [V,n,3,k]: the d xyz of every combination of one-sided cell choices at the kinks.  exact=True keeps
  the projection matrix in float64 (the oracle's)."""
  with float64():
    return _gather(case, backward, rows, plant, chunk, exact)


def _gather(case, backward, rows, plant, chunk, exact):
  cams, V, R, S = case["cams"], case["V"], case["R"], case["S"]
  N = R * S
  P = view_P(cams, exact)
  h_img, w_img = float(cams[0, 0]), float(cams[0, 1])
  rgbs = d64(case["rgbs"]).permute(0, 3, 1, 2)
  fm = d64(case["featmaps"])
  _, C, h, w = fm.shape
  H, W = rgbs.shape[2], rgbs.shape[3]
  xst = d64(case["xyz_st"]).reshape(N, 3)
  xyz = xst[None].expand(V, N, 3) if case["xyz"] is None else d64(case["xyz"]).reshape(V, N, 3)
  gfeat = d64(case["g_feat"]).reshape(N, V, 35)
  tgt = d64(case["queries"]).reshape(-1, 34)[:, 18:34].reshape(-1, 4, 4)[:, :3, 3]
  centers = d64(cams)[:, 18:34].reshape(-1, 4, 4)[:, :3, 3]
  tgt_idx = case["tgt_idx"]
  g_maps = torch.zeros(V * C * h * w)
  g_maps_mag, g_maps_sens = torch.zeros_like(g_maps), torch.zeros_like(g_maps)
  rows = torch.arange(N) if rows is None else torch.as_tensor(rows)
  keep = torch.zeros(N, dtype=torch.bool)
  keep[rows] = True
  res = {}

  def push(k, t):
    res.setdefault(k, []).append(t)

  for n0 in range(0, N, chunk):
    sl = slice(n0, min(N, n0 + chunk))
    kp = keep[sl]
    if not backward and not kp.any():
      continue
    pr = project(P, xyz[:, sl])
    u, v = pr["u"], pr["v"]
    fmap = lambda n_img, n_map, c, dc: grid_coord(c, dc, n_img, n_map)
    if plant == "feat_norm_by_map":
      ffx, dffx = fmap(w, w, u, pr["du"])
      ffy, dffy = fmap(h, h, v, pr["dv"])
    else:
      ffx, dffx = fmap(w_img, w, u, pr["du"])
      ffy, dffy = fmap(h_img, h, v, pr["dv"])
    ifx, difx = fmap(w_img, W, u, pr["du"])
    ify, dify = fmap(h_img, H, v, pr["dv"])
    tf = _taps(fm, ffx, ffy, torch.floor(ffx), torch.floor(ffy), plant)
    ti = _taps(rgbs, ifx, ify, torch.floor(ifx), torch.floor(ify), plant)
    # ---- forward (compared rows only)
    if kp.any():
      def sens(t, dfx_, dfy_):
        # the slope on either side of the nearest grid line bounds the slope within delta of it
        return t["dfx"].abs() * dfx_[..., None] + t["dfy"].abs() * dfy_[..., None] + t["cross"].abs() * (
            dfx_ * dfy_)[..., None]
      altx = lambda img, fx_, fy_: _taps(img, fx_, fy_, torch.floor(fx_) - 1, torch.floor(fy_) - 1)
      sf = torch.maximum(sens(tf, dffx, dffy), sens(altx(fm, ffx, ffy), dffx, dffy))
      si = torch.maximum(sens(ti, difx, dify), sens(altx(rgbs, ifx, ify), difx, dify))
      push("rgb_feat", torch.cat([ti["val"], tf["val"]], -1).permute(1, 0, 2)[kp])
      push("rgb_feat_mag", torch.cat([ti["mag"], tf["mag"]], -1).permute(1, 0, 2)[kp])
      push("rgb_feat_sens", torch.cat([si, sf], -1).permute(1, 0, 2)[kp])
      right = (u < w_img - 1) if plant == "mask_right_exclusive" else (u <= w_img - 1)
      inb = right & (u >= 0) & (v <= h_img - 1) & (v >= 0)
      push("mask", (inb & (pr["pz"] > 0)).double().t()[kp])
      du, dv = pr["du"], pr["dv"]
      kink = ((u.abs() <= du) | ((u - (w_img - 1)).abs() <= du) | (v.abs() <= dv) | ((v - (h_img - 1)).abs() <= dv)
              | (pr["pz"].abs() <= pr["dpz"]))
      push("mask_kink", kink.t()[kp])
      # ray_diff (oracle ray_angle_diff with the per-ray target of the multi-camera variant)
      pts_st = xst[sl]
      if tgt_idx is None:
        tg = tgt[0][None].expand(pts_st.shape[0], 3)
      else:
        tg = tgt[tgt_idx.long().repeat_interleave(S)[sl]]
      a = F.normalize(tg - pts_st, dim=-1)[None]
      b = F.normalize(centers[:, None, :] - xyz[:, sl], dim=-1)
      dd = a - b
      rd = torch.cat([F.normalize(dd, dim=-1), (a * b).sum(-1, keepdim=True)], -1)
      push("ray_diff", rd.permute(1, 0, 2)[kp])
      cond = 1.0 / dd.norm(dim=-1, keepdim=True).clamp(min=1e-30)
      push("ray_diff_mag", torch.cat([cond.expand(-1, -1, 3) * 4, torch.full_like(cond, 4.0)], -1).permute(1, 0, 2)[kp])
    if not backward:
      continue
    # ---- backward
    g = gfeat[sl].permute(1, 0, 2)  # [V,n,35]
    gi, gf = g[..., :3], g[..., 3:]
    for (idx, wgt, ok, wy_, wx_) in tf["taps"]:
      flat_idx = (torch.arange(V)[:, None, None] * C + torch.arange(C)[None, None, :]) * (h * w) + idx[..., None]
      okc = ok[..., None].double()
      g_maps.index_add_(0, flat_idx.reshape(-1), (gf * wgt[..., None] * okc).reshape(-1))
      g_maps_mag.index_add_(0, flat_idx.reshape(-1), (gf * wgt[..., None] * okc).abs().reshape(-1))
      s_ = gf.abs() * (wy_ * dffx + wx_ * dffy + dffx * dffy)[..., None] * okc
      g_maps_sens.index_add_(0, flat_idx.reshape(-1), s_.reshape(-1))
    if not kp.any():
      continue
    sl_kp = lambda t: t[:, kp]
    prk = {k: sl_kp(t) for k, t in pr.items()}
    co = dict(ffx=(ffx, dffx), ffy=(ffy, dffy), ifx=(ifx, difx), ify=(ify, dify))
    co = {k: (sl_kp(a_), sl_kp(b_)) for k, (a_, b_) in co.items()}
    gk = sl_kp(g)
    fm_taps = lambda x0, y0: _taps(fm, co["ffx"][0], co["ffy"][0], x0, y0, plant)
    im_taps = lambda x0, y0: _taps(rgbs, co["ifx"][0], co["ify"][0], x0, y0, plant)

    def dxyz(cells):
      tf_, ti_ = fm_taps(*cells[:2]), im_taps(*cells[2:])
      sx_f, sy_f = (w - 1.0) / (w_img - 1.0), (h - 1.0) / (h_img - 1.0)
      if plant == "feat_norm_by_map":
        sx_f = sy_f = 1.0
      sx_i, sy_i = (W - 1.0) / (w_img - 1.0), (H - 1.0) / (h_img - 1.0)
      du = (gk[..., 3:] * tf_["dfx"]).sum(-1) * sx_f + (gk[..., :3] * ti_["dfx"]).sum(-1) * sx_i
      dv = (gk[..., 3:] * tf_["dfy"]).sum(-1) * sy_f + (gk[..., :3] * ti_["dfy"]).sum(-1) * sy_i
      live = torch.ones_like(du) if plant == "pz_clamp_grad_kept" else prk["live"].double()
      su = torch.where(prk["u0"].abs() <= CLAMP, du / prk["d"], torch.zeros_like(du))
      sv = torch.where(prk["v0"].abs() <= CLAMP, dv / prk["d"], torch.zeros_like(dv))
      P8 = P[:, None, 2, :3]
      p8 = torch.zeros_like(P8) if plant == "dxyz_no_p8" else P8
      ju = P[:, None, 0, :3] - (live * prk["u0"])[..., None] * p8
      jv = P[:, None, 1, :3] - (live * prk["v0"])[..., None] * p8
      out = su[..., None] * ju + sv[..., None] * jv
      # magnitude of the terms and the first-order effect of the coordinate errors
      mag_du = (gk[..., 3:].abs() * tf_["sumabs"]).sum(-1) * sx_f + (gk[..., :3].abs() * ti_["sumabs"]).sum(-1) * sx_i
      mag_dv = (gk[..., 3:].abs() * tf_["sumabs"]).sum(-1) * sy_f + (gk[..., :3].abs() * ti_["sumabs"]).sum(-1) * sy_i
      s_du = (gk[..., 3:] * tf_["cross"]).abs().sum(-1) * sx_f * co["ffy"][1] + (
          gk[..., :3] * ti_["cross"]).abs().sum(-1) * sx_i * co["ify"][1]
      s_dv = (gk[..., 3:] * tf_["cross"]).abs().sum(-1) * sy_f * co["ffx"][1] + (
          gk[..., :3] * ti_["cross"]).abs().sum(-1) * sy_i * co["ifx"][1]
      okd = lambda c0, x: torch.where(c0.abs() <= CLAMP, x, torch.zeros_like(x))
      rel_d = prk["dpz"] / prk["d"] * prk["live"].double()
      mag = (okd(prk["u0"], mag_du / prk["d"])[..., None] * ju.abs()
             + okd(prk["v0"], mag_dv / prk["d"])[..., None] * jv.abs()
             + (su.abs() * prk["u0"].abs() + sv.abs() * prk["v0"].abs())[..., None] * p8.abs())
      sens = (okd(prk["u0"], s_du / prk["d"])[..., None] * ju.abs() + okd(prk["v0"], s_dv / prk["d"])[..., None] * jv.abs()
              + (su.abs() * prk["du"] + sv.abs() * prk["dv"])[..., None] * p8.abs()
              + (su.abs()[..., None] * ju.abs() + sv.abs()[..., None] * jv.abs()) * rel_d[..., None])
      return out, mag, sens

    cells = tuple(torch.floor(co[k][0]) for k in ("ffx", "ffy", "ifx", "ify"))
    gx, gmag, gsens = dxyz(cells)
    near = {k: _near_int(*co[k]) for k in co}
    kink = near["ffx"] | near["ffy"] | near["ifx"] | near["ify"]
    kink |= ((prk["u0"].abs() - CLAMP).abs() <= prk["du"] + EPS * CLAMP) | (
        (prk["v0"].abs() - CLAMP).abs() <= prk["dv"] + EPS * CLAMP)
    kink |= (prk["pz"] - C8).abs() <= prk["dpz"]
    alts = []
    for combo in range(16):
      cc = []
      for bit, k in enumerate(("ffx", "ffy", "ifx", "ify")):
        r_ = torch.round(co[k][0])
        side = r_ - 1 if (combo >> bit) & 1 == 0 else r_
        cc.append(torch.where(near[k], side, torch.floor(co[k][0])))
      alts.append(dxyz(tuple(cc))[0])
    push("g_xyz", gx)
    push("g_xyz_mag", gmag)
    push("g_xyz_sens", gsens)
    push("xyz_kink", kink)
    push("g_xyz_alt", torch.stack(alts, -1))
  out = {}
  for k, t in res.items():
    out[k] = torch.cat(t, 1 if k.startswith("g_xyz") or k == "xyz_kink" else 0)
  if backward:
    out["g_maps"] = g_maps.reshape(V, C, h, w)
    out["g_maps_mag"] = g_maps_mag.reshape(V, C, h, w)
    out["g_maps_sens"] = g_maps_sens.reshape(V, C, h, w)
  return out


def gather_oracle_autograd(case):
  """float64 torch autograd through the oracle's project_gather: (rgb_feat, mask, d featmaps, d xyz)."""
  with float64():
    cams, V, R, S = case["cams"], case["V"], case["R"], case["S"]
    fm = d64(case["featmaps"]).requires_grad_(True)
    xyz = (d64(case["xyz_st"])[None].repeat(V, 1, 1, 1) if case["xyz"] is None else d64(case["xyz"]))
    xyz.requires_grad_(True)
    rf, _, mask = O.project_gather(d64(case["xyz_st"]), xyz, d64(case["queries"][:1]), d64(case["rgbs"])[None],
                                   d64(cams)[None], fm)
    (rf * d64(case["g_feat"])).sum().backward()
  return rf.detach(), mask.detach(), fm.grad, xyz.grad


# ----------------------------------------------------------------------------------------------------------------
# compositing
# ----------------------------------------------------------------------------------------------------------------
def composite_case(R, S, seed, special=False, V=(8, 5), min_views=(1, 2)):
  """Random raws; special=True adds: densities above the softplus threshold, the -1e9 sentinel, a fully opaque ray
  whose transmittance underflows, a transparent ray and rays where exactly 8 / 9 samples are seen by more than
  min_views views."""
  g = torch.Generator().manual_seed(seed)
  raw_a, raw_b = torch.randn(R, S, 4, generator=g), torch.randn(R, S, 4, generator=g)
  raw_a[..., :3].sigmoid_()
  raw_b[..., :3].sigmoid_()
  raw_a[..., 3] = raw_a[..., 3] * 2 - 2.0
  raw_b[..., 3] = raw_b[..., 3] * 2 - 2.5
  z = torch.sort(torch.rand(R, S, generator=g) * 20 + 1, dim=1).values
  mask_a = (torch.rand(R, S, V[0], generator=g) > 0.5).float()
  mask_b = (torch.rand(R, S, V[1], generator=g) > 0.5).float()
  if special and R >= 6:
    raw_a[0, :, 3] = 50.0                                # opaque everywhere: T underflows
    raw_b[0, :, 3] = -1e9
    raw_a[1, :, 3] = -30.0                               # transparent
    raw_b[1, :, 3] = -1e9
    raw_a[2, S // 3, 3] = 25.0                           # one saturated sample (softplus(x) = x above 20)
    raw_b[2, S // 2, 3] = 40.0
    raw_a[3, ::3, 3] = -1e9                              # invalid samples
    raw_b[3, 1::3, 3] = -1e9
    raw_a[4, 0, 3] = 50.0                                # first sample opaque, later ones behind it
    for r_, n_ in ((4, 8), (5, 9)):                      # exactly n_ samples seen by more than min_views views
      mask_a[r_] = 0.0
      mask_b[r_] = 0.0
      mask_a[r_, :min(n_, S), :min_views[0] + 1] = 1.0
      mask_b[r_, :, :min_views[1]] = 1.0                 # exactly min_views: not more
  g_rays = torch.randn(R, 11, generator=g)
  g_samples = torch.randn(5, R, S, generator=g)
  return dict(raw_a=raw_a, raw_b=raw_b, z=z, mask_a=mask_a, mask_b=mask_b, min_a=min_views[0], min_b=min_views[1],
              g_rays=g_rays, g_samples=g_samples, R=R, S=S)


def _excl_cumprod(f):
  T = torch.cumprod(f, -1)
  return torch.cat([torch.ones_like(f[:, :1]), T[:, :-1]], -1)


def _rev_excl_cumsum(x):
  c = torch.flip(torch.cumsum(torch.flip(x, [1]), 1), [1])
  return c - x


def _alpha_parts(sigma, S, plant):
  delta = torch.ones_like(sigma)
  if plant != "last_delta_one":
    delta[:, -1] = 1e10
  y = F.softplus(sigma) * delta
  a = 1 - torch.exp(-y)
  # fp32 error of the kernel's alpha = 1 - expf(-y): the rounding of 1 - e (none below 0.5, at most 2^-25 and at
  # most e itself above) plus expf's and y's relative errors on e, doubled
  e = torch.exp(-y)
  err = 2 * (torch.where(a >= 0.5, torch.minimum(e, torch.full_like(e, 2.0 ** -25)), torch.zeros_like(e))
             + 4 * EPS * e * (1 + y))
  return a, delta, err


def _composite_fn(aA, aB, c, vanilla, gs_on, plant):
  """Kernel-order compositing forward and backward as a function of the alphas (so that their error can be
  propagated by a Jacobian).  Returns dict of outputs."""
  ra, rb, z, gr, gsamp, delta = c["ra"], c["rb"], c["z"], c["gr"], c["gs"], c["delta"]
  al = aA if vanilla else 1 - (1 - aB) * (1 - aA)
  f = 1 - al + (0.0 if plant == "composite_no_1e10" else C10)
  T = torch.cumprod(f, -1) if plant == "T_inclusive" else _excl_cumprod(f)
  wA, wB, wt = aA * T, aB * T, al * T
  o = {}
  o["rgb_dy"] = (wA[..., None] * ra[..., :3]).sum(1)
  o["rgb_static"] = (wB[..., None] * rb[..., :3]).sum(1)
  o["depth"] = (wt * z).sum(-1)
  o["alpha_dy"], o["weights_dy"], o["weights_st"], o["alpha"], o["weights"] = aA, wA, wB, al, wt
  if vanilla:
    gA, gB, gdepth = gr[:, 0:3], torch.zeros_like(gr[:, 0:3]), gr[:, 3]
  else:
    gA, gB, gdepth = gr[:, 0:3] + gr[:, 6:9], gr[:, 0:3] + gr[:, 3:6], gr[:, 9]
  z0 = torch.zeros_like(aA)
  if gs_on:
    gs_aA, gs_wA, gs_wB = (z0, z0, z0) if vanilla else (gsamp[0], gsamp[1], gsamp[2])
    gs_al, gs_w = (gsamp[1], gsamp[0]) if vanilla else (gsamp[3], gsamp[4])
  else:
    gs_aA = gs_wA = gs_wB = gs_al = gs_w = z0
  dwA = gs_wA + (gA[:, None, :] * ra[..., :3]).sum(-1)
  dwB = gs_wB + (gB[:, None, :] * rb[..., :3]).sum(-1)
  dw = gs_w + gdepth[:, None] * z
  G = dwA * aA + dwB * aB + dw * al
  gt = G * T
  suf = (_rev_excl_cumsum(gt) + gt) if plant == "suffix_off_by_one" else _rev_excl_cumsum(gt)
  dal = gs_al + dw * T - suf / f
  daA = gs_aA + dwA * T + dal * (1 - aB)
  daB = dwB * T + dal * (1 - aA)
  ea, eb = 1 - aA, 1 - aB
  dsa = torch.where(ea > 0, daA * ea * delta * torch.sigmoid(c["sa"]), z0)
  dsb = torch.where(eb > 0, daB * eb * delta * torch.sigmoid(c["sb"]), z0)
  o["g_a"] = torch.cat([gA[:, None, :] * wA[..., None], dsa[..., None]], -1)
  o["g_b"] = torch.cat([gB[:, None, :] * wB[..., None], dsb[..., None]], -1)
  # magnitudes (sum |terms| of the kernel's sums)
  Gabs = ((gs_wA.abs() + (gA[:, None, :] * ra[..., :3]).abs().sum(-1)) * aA
          + (gs_wB.abs() + (gB[:, None, :] * rb[..., :3]).abs().sum(-1)) * aB + (gs_w.abs() + (gdepth[:, None] * z).abs()) * al)
  sufabs = _rev_excl_cumsum(Gabs * T)
  dal_abs = gs_al.abs() + dw.abs() * T + sufabs / f
  o["g_a_mag"] = torch.cat([(gA[:, None, :] * wA[..., None]).abs(),
                            ((gs_aA.abs() + dwA.abs() * T + dal_abs * (1 - aB)) * ea * delta * torch.sigmoid(c["sa"]))[..., None]], -1)
  o["g_b_mag"] = torch.cat([(gB[:, None, :] * wB[..., None]).abs(),
                            ((dwB.abs() * T + dal_abs * (1 - aA)) * eb * delta * torch.sigmoid(c["sb"]))[..., None]], -1)
  o["rgb_dy_mag"] = (wA[..., None] * ra[..., :3]).abs().sum(1)
  o["rgb_static_mag"] = (wB[..., None] * rb[..., :3]).abs().sum(1)
  o["depth_mag"] = (wt * z).abs().sum(-1)
  return o


SENS_KEYS = ("rgb_dy", "rgb_static", "depth", "alpha_dy", "weights_dy", "weights_st", "alpha", "weights", "g_a", "g_b")


def composite(case, vanilla=False, gs_on=True, plant=None):
  """Reference of composite_kernel<!vanilla> and composite_backward_kernel on `case` (composite_case).
  Returns dict: rays [R,11] (vanilla [R,5]) and samples [5,R,S] (vanilla [2,R,S]) with *_mag and *_sens of the
  same shapes, g_raw_a / g_raw_b [R,S,4] with their mag and sens."""
  with float64():
    R, S = case["R"], case["S"]
    ra, rb, z = d64(case["raw_a"]), d64(case["raw_b"]), d64(case["z"])
    aA, delta, errA = _alpha_parts(ra[..., 3], S, plant)
    aB, _, errB = _alpha_parts(rb[..., 3], S, plant)
    if vanilla:
      aB, errB = torch.zeros_like(aA), torch.zeros_like(aA)
    gr = d64(case["g_rays"])
    if vanilla:
      gr = torch.cat([gr[:, 0:3], gr[:, 9:10], gr[:, 10:11]], -1)
    gs = d64(case["g_samples"])
    if vanilla:
      gs = gs[[4, 3]]  # d/d(weights, alpha)
    c = dict(ra=ra, rb=rb, z=z, gr=gr, gs=gs, delta=delta, sa=ra[..., 3], sb=rb[..., 3])
    o = _composite_fn(aA, aB, c, vanilla, gs_on, plant)
    # Jacobian of every output with respect to the alphas, weighted by their fp32 error
    sens = {k: torch.zeros_like(o[k]) for k in SENS_KEYS}
    for k in range(S):
      for which, err in (("A", errA), ("B", errB)):
        if vanilla and which == "B":
          continue
        tan = torch.zeros_like(aA)
        tan[:, k] = err[:, k]
        if not bool((tan != 0).any()):
          continue
        fn = ((lambda x: _composite_fn(x, aB, c, vanilla, gs_on, plant)) if which == "A"
              else (lambda y: _composite_fn(aA, y, c, vanilla, gs_on, plant)))
        _, t = torch.func.jvp(fn, ((aA if which == "A" else aB),), (tan,))
        for key in SENS_KEYS:
          sens[key] += t[key].abs()
    nseg = (S + 31) // 32
    chain = nseg + 8  # longest chain of roundings: lane scan (5) + segment carries + the product / sum
    mask_a = d64(case["mask_a"])
    cnt_a = (mask_a.sum(-1) > case["min_a"]).sum(-1)
    out = {}
    per_sample = lambda k: (o[k], chain * o[k].abs(), sens[k])
    if vanilla:
      rays = [o["rgb_dy"], o["depth"][:, None], (cnt_a > 8).double()[:, None]]
      rmag = [o["rgb_dy_mag"], o["depth_mag"][:, None], torch.zeros(R, 1)]
      rsens = [sens["rgb_dy"], sens["depth"][:, None], torch.zeros(R, 1)]
      keys = ("weights", "alpha")
    else:
      cnt_b = (d64(case["mask_b"]).sum(-1) > case["min_b"]).sum(-1)
      rays = [o["rgb_dy"] + o["rgb_static"], o["rgb_static"], o["rgb_dy"], o["depth"][:, None],
              ((cnt_a > 8) | (cnt_b > 8)).double()[:, None]]
      rmag = [o["rgb_dy_mag"] + o["rgb_static_mag"], o["rgb_static_mag"], o["rgb_dy_mag"], o["depth_mag"][:, None],
              torch.zeros(R, 1)]
      rsens = [sens["rgb_dy"] + sens["rgb_static"], sens["rgb_static"], sens["rgb_dy"], sens["depth"][:, None],
               torch.zeros(R, 1)]
      keys = ("alpha_dy", "weights_dy", "weights_st", "alpha", "weights")
    out["rays"], out["rays_mag"], out["rays_sens"] = torch.cat(rays, -1), chain * torch.cat(rmag, -1), torch.cat(rsens, -1)
    out["samples"] = torch.stack([o[k] for k in keys])
    out["samples_mag"] = torch.stack([per_sample(k)[1] for k in keys])
    out["samples_sens"] = torch.stack([sens[k] for k in keys])
    out["g_raw_a"], out["g_raw_a_mag"], out["g_raw_a_sens"] = o["g_a"], chain * o["g_a_mag"], sens["g_a"]
    out["g_raw_b"], out["g_raw_b_mag"], out["g_raw_b_sens"] = o["g_b"], chain * o["g_b_mag"], sens["g_b"]
    out["g_rays_used"], out["g_samples_used"] = gr, gs
  return out


def composite_oracle_autograd(case, vanilla=False, gs_on=True):
  """float64 autograd through oracle.composite / composite_vanilla with the upstream gradients of `case`."""
  with float64():
    ra = d64(case["raw_a"]).requires_grad_(True)
    rb = d64(case["raw_b"]).requires_grad_(True)
    z = d64(case["z"])
    gr, gs = d64(case["g_rays"]), d64(case["g_samples"])
    ones = torch.ones(z.shape, dtype=torch.bool)
    if vanilla:
      o = O.composite_vanilla(ra, z, ones)
      L = (o["rgb"] * gr[:, 0:3]).sum() + (o["depth"] * gr[:, 9]).sum()
      if gs_on:
        L = L + (o["weights"] * gs[4]).sum() + (o["alpha"] * gs[3]).sum()
      L.backward()
      return o, ra.grad, None
    o = O.composite(ra, rb, z, ones, ones)
    L = sum((o[k] * gr[:, i:i + 3]).sum() for k, i in (("rgb", 0), ("rgb_static", 3), ("rgb_dy", 6)))
    L = L + (o["depth"] * gr[:, 9]).sum()
    if gs_on:
      L = L + sum((o[k] * gs[i]).sum() for i, k in enumerate(("alpha_dy", "weights_dy", "weights_st", "alpha", "weights")))
    L.backward()
    return o, ra.grad, rb.grad


# ----------------------------------------------------------------------------------------------------------------
# optical flow
# ----------------------------------------------------------------------------------------------------------------
def flow_case(n_flow, R, S, seed, close_to_camera=False, zero_weights=False):
  """close_to_camera: the expected point of ray R-1 sits 0.02 in front of source camera 0, so q2 is small and the
  flow large and ill-conditioned (yet well away from the q2 = 0 kink, which no case reaches)."""
  g = torch.Generator().manual_seed(seed)
  cams, _ = rig(max(n_flow, 1), 48, 64, seed, radius=4.0)
  w = torch.softmax(torch.randn(R, S, generator=g) * 2, 1) * 0.9
  if zero_weights:
    w[0] = 0.0
    w[1, ::2] = 0.0
  pts = (torch.rand(n_flow, R, S, 3, generator=g) - 0.5) * 1.5
  if close_to_camera and n_flow >= 1:
    c = d64(cams[0])[18:34].reshape(4, 4)
    fwd, ctr = c[:3, 2], c[:3, 3]
    pts[0, R - 1] = (ctr + 0.02 * fwd + 0.3 * c[:3, 0]).float()[None] + 1e-3 * torch.randn(S, 3, generator=g)
    w[R - 1] = 1.0 / S
  uv = torch.rand(R, 2, generator=g) * torch.tensor([64.0, 48.0])
  g_flows = torch.randn(n_flow, R, 2, generator=g)
  return dict(weights=w, pts_seq=pts, cams=cams[:n_flow] if n_flow else cams[:1], uv=uv, g_flows=g_flows,
              n_flow=n_flow, R=R, S=S)


def flow(case, plant=None, exact=False):
  """Reference of flow_sf_kernel (flows only) and flow_backward_kernel: flows [n,R,2], g_weights [R,S],
  g_pts [n,R,S,3], each with mag and sens, and flow_kink [n,R] (q2 within its bound of 0)."""
  with float64():
    w, p = d64(case["weights"]), d64(case["pts_seq"])
    Kc, Rw, tw = flow_cams(case["cams"], exact)
    n, R, S = case["n_flow"], case["R"], case["S"]
    nseg = (S + 31) // 32
    e = (w[None, ..., None] * p).sum(2)                        # [n,R,3]
    de = (nseg + 6) * EPS * (w[None, ..., None] * p).abs().sum(2)
    c = torch.einsum("vij,vrj->vri", Rw, e) + tw[:, None]
    dc = torch.einsum("vij,vrj->vri", Rw.abs(), de) + 4 * EPS * (torch.einsum("vij,vrj->vri", Rw.abs(), e.abs()) + tw[:, None].abs())
    q = torch.einsum("vij,vrj->vri", Kc, c)
    dq = torch.einsum("vij,vrj->vri", Kc.abs(), dc) + 3 * EPS * torch.einsum("vij,vrj->vri", Kc.abs(), c.abs())
    q2 = q[..., 2]
    uv = d64(case["uv"])
    fl = q[..., :2] / q2[..., None] - uv[None]
    out = dict(flows=fl)
    out["flows_mag"] = (q[..., :2] / q2[..., None]).abs() + uv[None].abs()
    out["flows_sens"] = dq[..., :2] / q2[..., None].abs() + q[..., :2].abs() * dq[..., 2:3] / q2[..., None] ** 2
    out["flow_kink"] = q2.abs() <= dq[..., 2]
    gfl = d64(case["g_flows"])
    g0, g1 = gfl[..., 0], gfl[..., 1]
    gq = torch.stack([g0 / q2, g1 / q2, -(g0 * q[..., 0] + g1 * q[..., 1]) / q2 ** 2], -1)
    dgq = torch.stack([g0.abs() * dq[..., 2] / q2 ** 2, g1.abs() * dq[..., 2] / q2 ** 2,
                       (g0.abs() * dq[..., 0] + g1.abs() * dq[..., 1]) / q2 ** 2
                       + 2 * (g0 * q[..., 0] + g1 * q[..., 1]).abs() * dq[..., 2] / q2.abs() ** 3], -1)
    mgq = torch.stack([(g0 / q2).abs(), (g1 / q2).abs(), ((g0 * q[..., 0]).abs() + (g1 * q[..., 1]).abs()) / q2 ** 2], -1)
    KT = Kc.transpose(1, 2)
    RT = Rw if plant == "flow_Rw_transposed" else Rw.transpose(1, 2)
    gc = torch.einsum("vij,vrj->vri", KT, gq)
    ge = torch.einsum("vij,vrj->vri", RT, gc)
    abs_chain = lambda x: torch.einsum("vij,vrj->vri", Rw.abs().transpose(1, 2), torch.einsum("vij,vrj->vri", Kc.abs().transpose(1, 2), x))
    dge = abs_chain(dgq)
    mge = abs_chain(mgq)                                       # sum |terms| through both products
    gw = (ge[:, :, None, :] * p).sum(-1).sum(0)                # [R,S]
    out["g_weights"] = gw
    out["g_weights_mag"] = (mge[:, :, None, :] * p.abs()).sum(-1).sum(0) * (n + 3)
    out["g_weights_sens"] = (dge[:, :, None, :] * p.abs()).sum(-1).sum(0)
    out["g_pts"] = w[None, ..., None] * ge[:, :, None, :]
    out["g_pts_mag"] = w[None, ..., None].abs() * mge[:, :, None, :]
    out["g_pts_sens"] = w[None, ..., None].abs() * dge[:, :, None, :]
  return out


def flow_oracle_autograd(case):
  with float64():
    w = d64(case["weights"]).requires_grad_(True)
    p = d64(case["pts_seq"]).requires_grad_(True)
    fl = O.optical_flow(w, p, d64(case["cams"])[None], d64(case["uv"]))
    (fl * d64(case["g_flows"])).sum().backward()
  return fl.detach(), w.grad, p.grad


# ----------------------------------------------------------------------------------------------------------------
# resampling
# ----------------------------------------------------------------------------------------------------------------
def kernel_cdf32(weights, inv_uniform):
  """The kernel's fp32 cdf, emulated bit for bit: lane-strided partial sums of w + 1e-5, the xor-shuffle tree,
  then the sequential cumsum of (w + 1e-5) / tot (additions and divisions only, so no FMA contraction)."""
  w = weights.float()
  R, S = w.shape
  M = S - 2
  inner = w[:, 1:S - 1]
  if inv_uniform:
    inner = torch.flip(inner, [1])
  c5 = torch.tensor(1e-5, dtype=torch.float32)
  part = torch.zeros(R, 32, dtype=torch.float32)
  for i in range(M):
    part[:, i % 32] = part[:, i % 32] + (inner[:, i] + c5)
  for o in (16, 8, 4, 2, 1):
    part = part + part[:, torch.arange(32) ^ o]
  tot = part[:, 0]
  cdf = torch.zeros(R, M + 1, dtype=torch.float32)
  c = torch.zeros(R, dtype=torch.float32)
  for i in range(M):
    c = c + (inner[:, i] + c5) / tot
    cdf[:, i + 1] = c
  return cdf


def resample_case(R, S, Ni, seed, det, inv_uniform, special=False):
  """z [R,S] sorted in (near 1, far 20); weights; u [R,Ni] (None when det).  special=True adds an all-zero ray, a
  single spike, a spike with empty end bins (den < 1e-5 at both ends, the last one reached by u = 1) and, with
  given u, u = 0, u = 1, u equal to the kernel's cdf entries and u inside bins with den < 1e-5."""
  g = torch.Generator().manual_seed(seed)
  near, far = 1.0, 20.0
  if inv_uniform:
    t = torch.sort(torch.rand(R, S, generator=g), dim=1).values
    z = 1.0 / (1.0 / near + t * (1.0 / far - 1.0 / near))
  else:
    z = torch.sort(torch.rand(R, S, generator=g) * (far - near) + near, dim=1).values
  w = torch.rand(R, S, generator=g) ** 3
  if special and R >= 4:
    w[0] = 0.0
    w[1] = 0.0
    w[1, S // 2] = 1.0
    w[2] = 1e-7
    w[2, S // 2] = 100.0
    w[2, S // 2 + 1] = 3e-4
  u = None
  if not det:
    u = torch.rand(R, Ni, generator=g)
    if special and R >= 4:
      cdf = kernel_cdf32(w, inv_uniform)
      M = S - 2
      u[3, 0], u[3, 1] = 0.0, 1.0
      k = min(Ni - 2, M - 1)
      u[3, 2:2 + k] = cdf[3, 1:1 + k]                          # exactly at cdf entries
      u[2, 0], u[2, 1] = 0.0, 1.0
      j = min(Ni - 2, max(1, S // 4))
      u[2, 2:2 + j] = 0.5 * (cdf[2, :j] + cdf[2, 1:j + 1])     # inside bins of den < 1e-5 (before the spike)
  return dict(z=z.float(), weights=w.float(), u=u, R=R, S=S, Ni=Ni, inv_uniform=inv_uniform, det=det)


def resample(case, plant=None):
  """Reference of resample_kernel: fine samples (unsorted) as [R,Ni] intervals lo / hi (one-sided values at the
  kinks) with sens, the kink flags, and the merged sorted output of the coarse and the reference fine samples."""
  with float64():
    z, w = d64(case["z"]), d64(case["weights"])
    R, S, Ni, inv = case["R"], case["S"], case["Ni"], case["inv_uniform"]
    M = S - 2
    if case["u"] is None:
      u = torch.linspace(0.0, 1.0, Ni)[None].repeat(R, 1)
      du = 2 * EPS * u
    else:
      u = d64(case["u"])
      du = torch.zeros_like(u)
    if inv:
      iz = 1.0 / z
      bins = torch.flip(0.5 * (iz[:, 1:] + iz[:, :-1]), [1])
      wm = torch.flip(w[:, 1:-1], [1])
      dbins = 3 * EPS * bins.abs()
    else:
      bins = 0.5 * (z[:, 1:] + z[:, :-1])
      wm = w[:, 1:-1]
      dbins = EPS * bins.abs()
    wts = wm + C5
    pdf = wts / wts.sum(-1, keepdim=True)
    cdf = torch.cat([torch.zeros(R, 1), torch.cumsum(pdf, -1)], -1)
    dcdf = EPS * (torch.arange(M + 1)[None] + M / 32 + 8) * cdf
    n_count = M + 1 if plant == "cdf_M_plus_1" else M
    cnt = lambda off: (u[..., None] >= (cdf[:, None, :n_count] + off[:, None, :n_count])).long().sum(-1)
    above0 = cnt(torch.zeros_like(cdf))
    a_lo = (u[..., None] >= (cdf[:, None, :n_count] + dcdf[:, None, :n_count] + du[..., None])).long().sum(-1)
    a_hi = (u[..., None] >= (cdf[:, None, :n_count] - dcdf[:, None, :n_count] - du[..., None])).long().sum(-1)
    vals, senses = [], []
    kink = (a_lo != a_hi)
    # candidates: the reference count first, then every count within the cdf bound, each with the den rule at
    # the reference den and (at a den kink) the other side of it
    cands = [(above0, torch.ones_like(kink))] + [(a_lo + off, (a_lo + off) <= a_hi) for off in range(3)]
    for ci, (acount, valid_a) in enumerate(cands):
      above = acount.clamp(max=M)
      below = (acount - 1).clamp(min=0, max=M)
      c0, c1 = cdf.gather(1, below), cdf.gather(1, above)
      b0, b1 = bins.gather(1, below), bins.gather(1, above)
      dc0, dc1 = dcdf.gather(1, below), dcdf.gather(1, above)
      db0, db1 = dbins.gather(1, below), dbins.gather(1, above)
      den = c1 - c0
      dden = dc0 + dc1
      kden = (den - C5).abs() <= dden
      kink |= kden & valid_a
      for branch in (0, 1):
        use_one = den < C5
        if plant == "den_threshold_dropped":
          use_one = torch.zeros_like(use_one)
        if branch:
          use_one = ~use_one
        ok = valid_a & (kden if branch else torch.ones_like(kden))
        dn = torch.where(use_one, torch.ones_like(den), den)
        t = (u - c0) / dn
        dt = (du + dc0 + torch.where(use_one, torch.zeros_like(t), t.abs() * dden)) / dn
        smp = b0 + t * (b1 - b0)
        ds = (b1 - b0).abs() * dt + db0 + t.abs() * (db0 + db1) + EPS * (b0.abs() + 2 * (t * (b1 - b0)).abs())
        if inv:
          val, dv = 1.0 / smp, ds / smp ** 2 + EPS / smp.abs()
        else:
          val, dv = smp, ds
        vals.append(torch.where(ok, val, torch.full_like(val, float("nan"))))
        senses.append(torch.where(ok, dv, torch.zeros_like(dv)))
    V_ = torch.stack(vals, -1)
    ref = V_[..., 0]
    lo = torch.where(torch.isnan(V_), torch.full_like(V_, float("inf")), V_).min(-1).values
    hi = torch.where(torch.isnan(V_), torch.full_like(V_, -float("inf")), V_).max(-1).values
    sens = torch.stack(senses, -1).max(-1).values
    merged = torch.sort(torch.cat([z, ref], -1), -1).values
  return dict(fine=ref, lo=lo, hi=hi, sens=sens, kink=kink, merged=merged, above=above0)


def resample_check(case, ref, out):
  """The kernel's merged depths `out` [R, S + Ni] against `resample(case)`: -> (rows whose coarse depths are not all
  present bit for bit or whose fine samples leave the [lo - bar, hi + bar] intervals, the worst excess over the rays'
  kink-free samples)."""
  b_lo = bar("resample", ref["lo"], ref["lo"].abs(), ref["sens"])
  b_hi = bar("resample", ref["hi"], ref["hi"].abs(), ref["sens"])
  bad, worst = [], -1e30
  for r in range(case["R"]):
    row = out[r].tolist()
    try:
      for v in case["z"][r].tolist():  # every coarse depth appears bit for bit
        row.remove(v)
    except ValueError:
      bad.append(r)
      continue
    fine = d64(torch.tensor(row, dtype=torch.float32))
    if not (torch.isfinite(fine).all() and torch.isfinite(ref["lo"][r]).all() and torch.isfinite(ref["hi"][r]).all()):
      bad.append(r)
      continue
    lo = torch.sort(ref["lo"][r] - b_lo[r]).values
    hi = torch.sort(ref["hi"][r] + b_hi[r]).values
    if not ((fine >= lo) & (fine <= hi)).all():
      bad.append(r)
    clean = ~ref["kink"][r]
    if clean.any():
      srt, m = torch.sort(ref["fine"][r])
      ex = excess("resample", fine, srt, srt.abs(), ref["sens"][r][m])
      worst = max(worst, torch.nan_to_num(ex[clean[m]], nan=float("inf")).max().item())
  return bad, worst


def resample_oracle(case):
  with float64():
    return O.resample_depths(d64(case["z"]), d64(case["weights"]), case["Ni"], case["inv_uniform"],
                             None if case["u"] is None else d64(case["u"]))
