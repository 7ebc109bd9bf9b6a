"""CPU oracle for the DynIBaR per-ray volumetric IBR hot path.

TEST INFRASTRUCTURE ONLY.  This module is a torch-fp32 CPU restatement of the
reference algorithm (google/dynibar @ 5412b55); every function follows the dtype and
device of its inputs, so tests/train_step_ref.py evaluates it in float64 on the GPU.  It is imported only by
`tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / reference
arm.  The product (`dynibar_b200/`) never imports it and has no CPU fallback.

Pinning: `tests/golden/make_golden.py` runs the UNMODIFIED reference from
/root/reference on seeded inputs and commits the tensors under tests/golden/;
`tests/test_oracle_golden.py` checks this restatement against those fixtures
(and against a further stored run, tests/golden/live_reference.pt).

Everything is functional: network weights arrive as plain `state_dict`s whose
key names are the reference's (`base_fc.0.weight`, `ray_attention.w_qs.weight`
...), so the same dict feeds the reference modules, this oracle and the CUDA
weight packer.

Every function cites the reference file:line (relative to /root/reference) it
follows.
"""

from collections import OrderedDict
import math

import torch
import torch.nn.functional as F

# -----------------------------------------------------------------------------
# GEMM operand rounding emulation (used to *predict* the tensor-core path's
# error on CPU; "fp32" is the oracle proper).
# -----------------------------------------------------------------------------
_GEMM_MODE = "fp32"


def set_gemm_mode(mode):
  """'fp32' (oracle proper) or 'bf16' (bf16 operands, fp32 accumulate)."""
  global _GEMM_MODE
  assert mode in ("fp32", "bf16")
  _GEMM_MODE = mode


def _lin(x, w, b=None):
  if _GEMM_MODE == "bf16":
    x = x.to(torch.bfloat16).to(torch.float32)
    w = w.to(torch.bfloat16).to(torch.float32)
  y = x @ w.t()
  if b is not None:
    y = y + b
  return y


def _elu(x):
  return F.elu(x)


# -----------------------------------------------------------------------------
# a8  PeriodicEmbed  (ibrnet/mlp_network.py:530-555)
# -----------------------------------------------------------------------------
def periodic_embed(x, n_freq, linspace=False):
  """[x, cos(f_0 x) .. cos(f_{n-1} x), sin(f_0 x) .. sin(f_{n-1} x)].

  linspace=False: f_k = 2^k (mlp_network.py:546-547); linspace=True:
  f = linspace(1, max_freq+1, n) with max_freq == n (mlp_network.py:544, :589).
  """
  if linspace:
    freqs = torch.linspace(1, n_freq + 1, steps=n_freq)
  else:
    freqs = 2 ** torch.linspace(0, n_freq - 1, steps=n_freq)
  parts = [x]
  for fn in (torch.cos, torch.sin):
    for f in freqs:
      parts.append(fn(f * x))
  return torch.cat(parts, -1)


# -----------------------------------------------------------------------------
# a1  pixel rays  (ibrnet/sample_ray.py:143-163)
# -----------------------------------------------------------------------------
def pixel_rays(H, W, K, c2w, stride=1):
  """ray_d = R_c2w K^-1 [u, v, 1]^T at integer pixel centres, ray_o = t_c2w."""
  us = torch.arange(W, dtype=torch.float32)[::stride]
  vs = torch.arange(H, dtype=torch.float32)[::stride]
  v, u = torch.meshgrid(vs, us, indexing="ij")
  pix = torch.stack([u.reshape(-1), v.reshape(-1), torch.ones(u.numel())], 0)
  d = (c2w[:3, :3] @ torch.inverse(K[:3, :3]) @ pix).t().contiguous()
  o = c2w[:3, 3][None].repeat(d.shape[0], 1)
  uv = torch.stack([u.reshape(-1), v.reshape(-1)], -1)
  return o, d, uv


# -----------------------------------------------------------------------------
# a2  sample_along_camera_ray  (ibrnet/render_ray.py:67-131)
# -----------------------------------------------------------------------------
def sample_along_ray(ray_o, ray_d, depth_range, S, inv_uniform, jitter=None):
  """jitter: None (det=True) or a [R,S] tensor of U[0,1) (det=False;
  reference draws torch.rand_like at render_ray.py:119)."""
  near = depth_range[0, 0]
  far = depth_range[0, 1]
  R = ray_d.shape[0]
  ones = torch.ones(R, dtype=ray_d.dtype, device=ray_d.device)
  near_v = near * ones
  far_v = far * ones
  if inv_uniform:
    start = 1.0 / near_v
    step = (1.0 / far_v - start) / (S - 1)
    z = 1.0 / torch.stack([start + i * step for i in range(S)], 1)
  else:
    start = near_v
    step = (far_v - near_v) / (S - 1)
    z = torch.stack([start + i * step for i in range(S)], 1)
  if jitter is not None:
    mids = 0.5 * (z[:, 1:] + z[:, :-1])
    upper = torch.cat([mids, z[:, -1:]], -1)
    lower = torch.cat([z[:, :1], mids], -1)
    z = lower + (upper - lower) * jitter
  pts = z[..., None] * ray_d[:, None, :] + ray_o[:, None, :]
  s = z_to_s(z, near, far)
  return pts, z, s


def z_to_s(z, near, far):
  """ibrnet/render_ray.py:399-404."""
  return ((1.0 / z) - (1.0 / near)) / (1.0 / far - 1.0 / near)


# -----------------------------------------------------------------------------
# a3  MotionMLP + trajectory displacement
#     (ibrnet/mlp_network.py:605-618, ibrnet/render_ray.py:361-369, :462-500)
# -----------------------------------------------------------------------------
def motion_mlp(w, xyzt):
  x0 = periodic_embed(xyzt, 16, linspace=True)  # 4 -> 132
  h = x0
  for i in range(8):
    h = torch.relu(_lin(h, w["pts_linears.%d.weight" % i],
                        w["pts_linears.%d.bias" % i]))
    if i == 4:  # skips=[4], mlp_network.py:612-613
      h = torch.cat([x0, h], -1)
  return _lin(h, w["coeff_linear.weight"], w["coeff_linear.bias"])


def motion_coefficients(w, pts, t):
  """coeffs [R,S,3*nb] with the last round(0.1 S) samples zeroed
  (render_ray.py:459, :471-472)."""
  R, S = pts.shape[:2]
  xyzt = torch.cat([pts, t.to(pts).reshape(1, 1, 1).expand(R, S, 1)], -1)
  c = motion_mlp(w, xyzt)
  n_last = int(round(S * 0.1))
  c = c.clone()
  c[:, -n_last:, :] = c[:, -n_last:, :] * 0.0
  return c


def traj_offset(coeff, basis_row):
  """Sum_k coeff_axis[k] * basis[f, k] per axis (render_ray.py:361-369)."""
  nb = basis_row.shape[-1]
  return torch.stack(
      [(coeff[..., a * nb:(a + 1) * nb] * basis_row).sum(-1) for a in range(3)],
      -1)


def displaced_points(pts, coeff, basis, frame_idx, offsets):
  """pts_o = pts + (traj_o - traj_0), stacked over `offsets`
  (render_ray.py:479-497)."""
  traj = {o: traj_offset(coeff, basis[frame_idx + o]) for o in range(-3, 4)}
  seq = [pts + (traj[o] - traj[0]) for o in offsets]
  return torch.stack(seq, 0), traj


# -----------------------------------------------------------------------------
# a4-a6  Projector  (ibrnet/projection.py:13-176)
# -----------------------------------------------------------------------------
def project_points(xyz, cams):
  """xyz [V,N,3], cams [V,34] -> pix [V,N,2], in_front [V,N]
  (projection.py:32-59)."""
  Kmat = cams[:, 2:18].reshape(-1, 4, 4)
  c2w = cams[:, 18:34].reshape(-1, 4, 4)
  P = Kmat.bmm(torch.inverse(c2w))
  xyz_h = torch.cat([xyz, torch.ones_like(xyz[..., :1])], -1)
  proj = P.bmm(xyz_h.permute(0, 2, 1)).permute(0, 2, 1)
  pix = proj[..., :2] / torch.clamp(proj[..., 2:3], min=1e-8)
  pix = torch.clamp(pix, min=-1e6, max=1e6)
  return pix, proj[..., 2] > 0


def bilinear_gather(img, pix, h_img, w_img):
  """grid_sample(bilinear, zeros, align_corners=True) of img [V,C,h,w] at
  pixel coords `pix` [V,N,2] that are expressed in the SOURCE IMAGE frame
  (h_img, w_img) -- the reference normalises by the image size for both the
  image and the 1/4-res feature map (projection.py:22-30, :136-158).
  Returns [V,N,C]."""
  V, C, h, w = img.shape
  gx = 2 * pix[..., 0] / (w_img - 1.0) - 1.0
  gy = 2 * pix[..., 1] / (h_img - 1.0) - 1.0
  # align_corners=True un-normalisation
  x = (gx + 1) * 0.5 * (w - 1)
  y = (gy + 1) * 0.5 * (h - 1)
  x0 = torch.floor(x)
  y0 = torch.floor(y)
  out = torch.zeros(V, pix.shape[1], C, dtype=img.dtype, device=img.device)
  flat = img.reshape(V, C, h * w)
  for dy in (0, 1):
    for dx in (0, 1):
      xi = x0 + dx
      yi = y0 + dy
      wx = (x - x0) if dx else (x0 + 1 - x)
      wy = (y - y0) if dy else (y0 + 1 - y)
      ok = (xi >= 0) & (xi <= w - 1) & (yi >= 0) & (yi <= h - 1)
      idx = (yi.clamp(0, h - 1) * w + xi.clamp(0, w - 1)).long()
      tap = torch.gather(flat, 2, idx[:, None, :].expand(V, C, -1))
      out += (tap * (wx * wy * ok)[:, None, :]).permute(0, 2, 1)
  return out


def ray_angle_diff(xyz_st, xyz, query_cam, cams):
  """[normalize(a-b), a.b] with a = dir(point_st -> target cam),
  b = dir(point_v -> source cam v)  (projection.py:61-101).
  xyz_st [N,3], xyz [V,N,3] -> [V,N,4]."""
  tgt = query_cam[18:34].reshape(4, 4)[:3, 3]
  src = cams[:, 18:34].reshape(-1, 4, 4)[:, :3, 3]
  a = F.normalize(tgt[None, None, :] - xyz_st[None], dim=-1)
  b = F.normalize(src[:, None, :] - xyz, dim=-1)
  d = a - b
  dot = (a * b).sum(-1, keepdim=True)
  a = a.expand_as(b)
  return torch.cat([F.normalize(d, dim=-1), dot], -1)


def project_gather(xyz_st, xyz, query_cam, src_rgbs, src_cams, featmaps):
  """Projector.compute_with_motions (projection.py:103-176).

  xyz_st [R,S,3]; xyz [V,R,S,3]; query_cam [1,34]; src_rgbs [1,V,H,W,3];
  src_cams [1,V,34]; featmaps [V,C,h,w].
  Returns rgb_feat [R,S,V,3+C], ray_diff [R,S,V,4], mask [R,S,V,1] float.
  """
  V, R, S = xyz.shape[:3]
  cams = src_cams[0]
  h_img, w_img = float(cams[0, 0]), float(cams[0, 1])
  imgs = src_rgbs[0].permute(0, 3, 1, 2)
  pts = xyz.reshape(V, R * S, 3)
  pix, front = project_points(pts, cams)
  rgb = bilinear_gather(imgs, pix, h_img, w_img)
  feat = bilinear_gather(featmaps, pix, h_img, w_img)
  rgb_feat = torch.cat([rgb, feat], -1).reshape(V, R, S, -1).permute(1, 2, 0, 3)
  inb = ((pix[..., 0] <= w_img - 1.0) & (pix[..., 0] >= 0)
         & (pix[..., 1] <= h_img - 1.0) & (pix[..., 1] >= 0))
  rd = ray_angle_diff(xyz_st.reshape(R * S, 3), pts, query_cam[0], cams)
  rd = rd.reshape(V, R, S, 4).permute(1, 2, 0, 3)
  mask = (inb & front).to(xyz.dtype).reshape(V, R, S).permute(1, 2, 0)[..., None]
  return rgb_feat.contiguous(), rd.contiguous(), mask.contiguous()


# -----------------------------------------------------------------------------
# a7  Plucker coordinates  (ibrnet/render_ray.py:372-396)
#     (cross product over the LAST dim; the reference's dim-less torch.cross
#      agrees whenever no leading dim equals 3 -- SURVEY App. B quirk 2)
# -----------------------------------------------------------------------------
def plucker_ref(ray_o, ray_d):
  d = F.normalize(ray_d, dim=-1)
  return torch.cat([d, torch.linalg.cross(ray_o, d, dim=-1)], -1)


def plucker_src(pts, src_cams):
  """pts [R,S,3], src_cams [1,V,34] -> [R,S,V,6]."""
  o = src_cams[0, :, 18:34].reshape(-1, 4, 4)[:, :3, 3][:, None, None, :]
  d = F.normalize(pts[None] - o, dim=-1)
  m = torch.linalg.cross(o.expand_as(d), d, dim=-1)
  return torch.cat([d, m], -1).permute(1, 2, 0, 3)


# -----------------------------------------------------------------------------
# a11 ray transformer  (ibrnet/mlp_network.py:13-31, :56-104)
# -----------------------------------------------------------------------------
def ray_attention(w, x, row_valid, prefix="ray_attention."):
  """x [R,S,128]; row_valid [R,S] float (1 = keep).  NOTE the reference masks
  QUERY ROWS (mask [R,1,S,1] broadcast over keys, mlp_network.py:23-24,91-94):
  an invalid query attends uniformly, invalid keys are still attended."""
  R, S, D = x.shape
  H, dk = 4, 32
  q = _lin(x, w[prefix + "w_qs.weight"]).view(R, S, H, dk).transpose(1, 2)
  k = _lin(x, w[prefix + "w_ks.weight"]).view(R, S, H, dk).transpose(1, 2)
  v = _lin(x, w[prefix + "w_vs.weight"]).view(R, S, H, dk).transpose(1, 2)
  att = torch.matmul(q / (dk ** 0.5), k.transpose(2, 3))
  att = att.masked_fill(row_valid[:, None, :, None] == 0, -1e9)
  att = torch.softmax(att, -1)
  o = torch.matmul(att, v).transpose(1, 2).reshape(R, S, H * dk)
  o = _lin(o, w[prefix + "fc.weight"]) + x
  return F.layer_norm(o, (D,), w[prefix + "layer_norm.weight"],
                      w[prefix + "layer_norm.bias"], eps=1e-6)


def sinusoid_table(n_samples, d_hid=128):
  """mlp_network.py:220-234 (computed in float64, cast to float32: the reference's
  buffer holds these values whatever dtype the net is evaluated in)."""
  pos = torch.arange(n_samples, dtype=torch.float64)[:, None]
  j = torch.arange(d_hid)
  ang = pos / torch.pow(torch.tensor(10000.0, dtype=torch.float64),
                        2 * (j // 2).double() / d_hid)[None]
  tab = ang.clone()
  tab[:, 0::2] = torch.sin(ang[:, 0::2])
  tab[:, 1::2] = torch.cos(ang[:, 1::2])
  return tab.float()


def _weighted_mean_var(x, wgt):
  """fused_mean_variance (mlp_network.py:115-119); reduce over dim 2."""
  mean = (x * wgt).sum(2, keepdim=True)
  var = (wgt * (x - mean) ** 2).sum(2, keepdim=True)
  return mean, var


def _visibility_block(w, x, weight, mask):
  """Shared tail of both nets' per-view stage
  (mlp_network.py:272-281 / :485-495)."""
  xv = _elu(_lin(_elu(_lin(x * weight, w["vis_fc.0.weight"], w["vis_fc.0.bias"])),
                 w["vis_fc.2.weight"], w["vis_fc.2.bias"]))
  x_res, vis = xv[..., :-1], xv[..., -1:]
  vis = torch.sigmoid(vis) * mask
  x = x + x_res
  h = _elu(_lin(x * vis, w["vis_fc2.0.weight"], w["vis_fc2.0.bias"]))
  vis = torch.sigmoid(_lin(h, w["vis_fc2.2.weight"], w["vis_fc2.2.bias"])) * mask
  weight = vis / (vis.sum(2, keepdim=True) + 1e-8)
  mean, var = _weighted_mean_var(x, weight)
  glob = torch.cat([mean.squeeze(2), var.squeeze(2), weight.mean(2)], -1)
  return x, vis, glob


# -----------------------------------------------------------------------------
# a9  DynibarDynamic.forward  (ibrnet/mlp_network.py:236-316)
# -----------------------------------------------------------------------------
def net_dynamic(w, pts, rgb_feat, ray_dir, mask, t, shift=0.0):
  """pts [R,S,3]; rgb_feat [R,S,V,35]; ray_dir [R,3] (normalised);
  mask [R,S,V,1]; t scalar tensor -> raw [R,S,4].
  (ray_diff / time_diff are accepted by the reference but unused: SURVEY B.3)"""
  R, S, V, _ = rgb_feat.shape
  t_pe = periodic_embed(t.to(rgb_feat).reshape(1, 1), 10)  # [1,21]
  dfeat = _elu(_lin(_elu(_lin(t_pe, w["ray_dir_fc.0.weight"], w["ray_dir_fc.0.bias"])),
                    w["ray_dir_fc.2.weight"], w["ray_dir_fc.2.bias"]))
  feat = rgb_feat + dfeat.reshape(1, 1, 1, -1)
  weight = mask / (mask.sum(2, keepdim=True) + 1e-8)
  mean, var = _weighted_mean_var(feat, weight)
  x = torch.cat([mean.expand(-1, -1, V, -1), var.expand(-1, -1, V, -1), feat], -1)
  x = _elu(_lin(_elu(_lin(x, w["base_fc.0.weight"], w["base_fc.0.bias"])),
                w["base_fc.2.weight"], w["base_fc.2.bias"]))
  x, vis, glob = _visibility_block(w, x, weight, mask)
  g = _elu(_lin(_elu(_lin(glob, w["geometry_fc.0.weight"], w["geometry_fc.0.bias"])),
                w["geometry_fc.2.weight"], w["geometry_fc.2.bias"]))
  n_valid = mask.sum(2)  # [R,S,1]
  g = g + sinusoid_table(S).to(g)[None]
  g = ray_attention(w, g, (n_valid[..., 0] > 1).float())
  g = torch.cat([g, periodic_embed(pts, 5)], -1)
  g = _elu(_lin(_elu(_lin(g, w["ref_pts_fc.0.weight"], w["ref_pts_fc.0.bias"])),
                w["ref_pts_fc.2.weight"], w["ref_pts_fc.2.bias"]))
  sigma = _lin(_elu(_lin(g, w["out_geometry_fc.0.weight"], w["out_geometry_fc.0.bias"])),
               w["out_geometry_fc.2.weight"], w["out_geometry_fc.2.bias"]) - shift
  sigma = sigma.masked_fill(n_valid < 1, -1e9)
  d_pe = periodic_embed(ray_dir, 4)  # [R,27]
  h = torch.cat([g, d_pe[:, None, :].expand(-1, S, -1)], -1)
  h = _elu(_lin(h, w["rgb_fc.0.weight"], w["rgb_fc.0.bias"]))
  h = _elu(_lin(h, w["rgb_fc.2.weight"], w["rgb_fc.2.bias"]))
  rgb = torch.sigmoid(_lin(h, w["rgb_fc.4.weight"], w["rgb_fc.4.bias"]))
  rgb = rgb.masked_fill(n_valid == 0, 0)
  return torch.cat([rgb, sigma], -1)


# -----------------------------------------------------------------------------
# a10 DynibarStatic.forward  (ibrnet/mlp_network.py:423-527)
# -----------------------------------------------------------------------------
def net_static(w, pts, ref_rays, src_rays, rgb_feat, ray_diff, mask,
               anti_alias_pooling=True, mask_rgb=False):
  """pts [R,S,3]; ref_rays [R,6]; src_rays [R,S,V,6]; rgb_feat [R,S,V,35];
  ray_diff [R,S,V,4]; mask [R,S,V,1] -> raw [R,S,4]."""
  R, S, V, _ = rgb_feat.shape
  ref_pe = periodic_embed(ref_rays, 5)  # [R,66]
  src_pe = periodic_embed(src_rays, 5)  # [R,S,V,66]
  pts_pe = periodic_embed(pts, 5)  # [R,S,33]
  src_in = torch.cat([pts_pe[:, :, None, :].expand(-1, -1, V, -1), src_pe, ray_diff], -1)
  src_feat = _lin(_elu(_lin(src_in, w["ray_dir_fc.0.weight"], w["ray_dir_fc.0.bias"])),
                  w["ray_dir_fc.2.weight"], w["ray_dir_fc.2.bias"])
  ref_feat = _lin(ref_pe, w["ref_feature_fc.0.weight"], w["ref_feature_fc.0.bias"])
  rgb_in = rgb_feat[..., :3]
  if mask_rgb:
    mask = mask * (rgb_in.sum(-1, keepdim=True) > 1e-3).to(mask.dtype)
  feat = torch.cat([rgb_feat, src_feat * ref_feat[:, None, None, :]], -1)  # 70
  if anti_alias_pooling:
    e = torch.exp(torch.abs(w["s"]) * (ray_diff[..., 3:4] - 1))
    weight = (e - e.min(2, keepdim=True)[0]) * mask
    weight = weight / (weight.sum(2, keepdim=True) + 1e-8)
  else:
    weight = mask / (mask.sum(2, keepdim=True) + 1e-8)
  mean, var = _weighted_mean_var(feat, weight)
  x = torch.cat([mean.expand(-1, -1, V, -1), var.expand(-1, -1, V, -1), feat], -1)
  x = _elu(_lin(_elu(_lin(x, w["base_fc.0.weight"], w["base_fc.0.bias"])),
                w["base_fc.2.weight"], w["base_fc.2.bias"]))
  x, vis, glob = _visibility_block(w, x, weight, mask)
  g = _elu(_lin(_elu(_lin(glob, w["geometry_fc.0.weight"], w["geometry_fc.0.bias"])),
                w["geometry_fc.2.weight"], w["geometry_fc.2.bias"]))
  n_valid = mask.sum(2)
  g = ray_attention(w, g, (n_valid[..., 0] > 1).float())
  sigma = _lin(_elu(_lin(g, w["out_geometry_fc.0.weight"], w["out_geometry_fc.0.bias"])),
               w["out_geometry_fc.2.weight"], w["out_geometry_fc.2.bias"])
  sigma = sigma.masked_fill(n_valid < 1, -1e9)
  h = torch.cat([g[:, :, None, :].expand(-1, -1, V, -1), x, vis, ray_diff], -1)  # 261
  h = _elu(_lin(h, w["rgb_fc.0.weight"], w["rgb_fc.0.bias"]))
  h = _elu(_lin(h, w["rgb_fc.2.weight"], w["rgb_fc.2.bias"]))
  logit = _lin(h, w["rgb_fc.4.weight"], w["rgb_fc.4.bias"])
  logit = logit.masked_fill(mask == 0, -1e9)
  blend = torch.softmax(logit, 2)
  rgb = (rgb_in * blend).sum(2)
  return torch.cat([rgb, sigma], -1)


# -----------------------------------------------------------------------------
# a12 compositing  (ibrnet/render_ray.py:134-211, :214-330)
# -----------------------------------------------------------------------------
def _alpha(sigma):
  """1 - exp(-softplus(sigma) * delta), delta = 1 except last = 1e10
  (render_ray.py:154-184; USE_SOFTPLUS=True, USE_DISTANCE=False)."""
  d = torch.ones_like(sigma)
  d[..., -1] = 1e10
  return 1.0 - torch.exp(-F.softplus(sigma) * d)


def _transmittance(alpha):
  T = torch.cumprod(1.0 - alpha + 1e-10, -1)[:, :-1]
  return torch.cat([torch.ones_like(T[:, :1]), T], -1)


def composite_vanilla(raw, z, pix_mask):
  rgb, sigma = raw[..., :3], raw[..., 3]
  a = _alpha(sigma)
  wgt = a * _transmittance(a)
  return OrderedDict([
      ("rgb", (wgt[..., None] * rgb).sum(1)),
      ("depth", (wgt * z).sum(-1)),
      ("weights", wgt),
      ("mask", pix_mask.sum(1) > 8),
      ("alpha", a),
      ("z_vals", z),
  ])


def composite(raw_dy, raw_st, z, mask_dy, mask_st):
  a_dy = _alpha(raw_dy[..., 3])
  a_st = _alpha(raw_st[..., 3])
  a = 1 - (1 - a_st) * (1 - a_dy)
  T = _transmittance(a)
  w_dy = a_dy * T
  w_st = a_st * T
  rgb_dy = (w_dy[..., None] * raw_dy[..., :3]).sum(1)
  rgb_st = (w_st[..., None] * raw_st[..., :3]).sum(1)
  wgt = a * T
  return OrderedDict([
      ("rgb", rgb_dy + rgb_st),
      ("rgb_static", rgb_st),
      ("rgb_dy", rgb_dy),
      ("depth", (wgt * z).sum(-1)),
      ("alpha_dy", a_dy),
      ("weights_dy", w_dy),
      ("weights_st", w_st),
      ("alpha", a),
      ("weights", wgt),
      ("mask", (mask_dy.sum(1) > 8) | (mask_st.sum(1) > 8)),
      ("z_vals", z),
  ])


# -----------------------------------------------------------------------------
# a13 hierarchical resampling  (ibrnet/render_ray.py:19-64, :790-831)
# -----------------------------------------------------------------------------
def sample_pdf(bins, weights, n, u=None):
  """bins [R,M+1], weights [R,M]; u: None (det linspace) or [R,n] uniforms.
  The index is the count of the FIRST M cdf entries <= u (render_ray.py:38-39)."""
  M = weights.shape[1]
  wts = weights + 1e-5
  pdf = wts / wts.sum(-1, keepdim=True)
  cdf = torch.cat([torch.zeros_like(pdf[:, :1]), torch.cumsum(pdf, -1)], -1)
  if u is None:
    u = torch.linspace(0.0, 1.0, n)[None].repeat(bins.shape[0], 1)
  above = torch.zeros_like(u, dtype=torch.long)
  for i in range(M):
    above += (u >= cdf[:, i:i + 1]).long()
  below = torch.clamp(above - 1, min=0)
  c0 = torch.gather(cdf, 1, below)
  c1 = torch.gather(cdf, 1, above)
  b0 = torch.gather(bins, 1, below)
  b1 = torch.gather(bins, 1, above)
  den = c1 - c0
  den = torch.where(den < 1e-5, torch.ones_like(den), den)
  return b0 + (u - c0) / den * (b1 - b0)


def resample_depths(z, weights, n_importance, inv_uniform, u=None):
  """Coarse depths + coarse weights -> sorted [R, S+Ni] fine depths
  (render_ray.py:790-819)."""
  wmid = weights[:, 1:-1]
  if inv_uniform:
    iz = 1.0 / z
    mid = 0.5 * (iz[:, 1:] + iz[:, :-1])
    zs = 1.0 / sample_pdf(torch.flip(mid, [1]), torch.flip(wmid, [1]),
                          n_importance, u)
  else:
    mid = 0.5 * (z[:, 1:] + z[:, :-1])
    zs = sample_pdf(mid, wmid, n_importance, u)
  return torch.sort(torch.cat([z, zs], -1), -1)[0]


# -----------------------------------------------------------------------------
# a14 optical flow / expected scene flow
#     (ibrnet/render_ray.py:333-358, :585-595, :1086-1096)
# -----------------------------------------------------------------------------
def optical_flow(weights, pts_seq, src_cams, uv):
  """weights [R,S]; pts_seq [V,R,S,3]; src_cams [1,V,34]; uv [R,2] -> [V,R,2]."""
  cams = src_cams[0]
  Kmat = cams[:, 2:18].reshape(-1, 4, 4)[:, :3, :3]
  w2c = torch.inverse(cams[:, 18:34].reshape(-1, 4, 4))
  p = (weights[None, ..., None] * pts_seq).sum(-2)  # [V,R,3]
  pc = torch.einsum("vij,vrj->vri", w2c[:, :3, :3], p) + w2c[:, None, :3, 3]
  px = torch.einsum("vij,vrj->vri", Kmat, pc)
  px = px / px[..., 2:3]
  return px[..., :2] - uv[None]


def expected_scene_flow(weights, traj, k):
  p = (weights[..., None] * (traj[k] - traj[0])).sum(-2)
  m = (weights[..., None] * (traj[-k] - traj[0])).sum(-2)
  return torch.max(p, m)


# -----------------------------------------------------------------------------
# a15 orchestrators
# -----------------------------------------------------------------------------
def _sd(module_or_dict):
  if hasattr(module_or_dict, "state_dict"):
    m = module_or_dict.module if hasattr(module_or_dict, "module") else module_or_dict
    return {k: v.detach() for k, v in m.state_dict().items()}
  return module_or_dict


def _pass(ray_batch, feat_dy, feat_st, pts, z, s, t, frame_idx, offsets, num_vv,
          w_dy, w_st, w_mo, basis, args, shift, flow_views=None, sf_k=2):
  """One coarse-or-fine evaluation at the reference time
  (render_ray.py:455-597 == :672-782 == :951-1096)."""
  ray_dir = F.normalize(ray_batch["ray_d"], dim=-1)
  coeff = motion_coefficients(w_mo, pts, t)
  seq, traj = displaced_points(pts, coeff, basis, frame_idx, offsets)
  if num_vv:
    seq = torch.cat([seq, pts[None].repeat(num_vv, 1, 1, 1)], 0)
  V_st = ray_batch["static_src_rgbs"].shape[1]
  f_dy, rd_dy, m_dy = project_gather(pts, seq, ray_batch["camera"],
                                     ray_batch["src_rgbs"],
                                     ray_batch["src_cameras"], feat_dy)
  f_st, rd_st, m_st = project_gather(pts, pts[None].repeat(V_st, 1, 1, 1),
                                     ray_batch["camera"],
                                     ray_batch["static_src_rgbs"],
                                     ray_batch["static_src_cameras"], feat_st)
  pm_dy = m_dy[..., 0].sum(2) > 1
  pm_st = m_st[..., 0].sum(2) > 1
  raw_dy = net_dynamic(w_dy, pts, f_dy, ray_dir, m_dy, t, shift)
  raw_st = net_static(w_st, pts, plucker_ref(ray_batch["ray_o"], ray_batch["ray_d"]),
                      plucker_src(pts, ray_batch["static_src_cameras"]),
                      f_st, rd_st, m_st,
                      anti_alias_pooling=bool(args.anti_alias_pooling),
                      mask_rgb=bool(args.mask_rgb))
  out = composite(raw_dy, raw_st, z, pm_dy, pm_st)
  out_dy = composite_vanilla(raw_dy, z, pm_dy)
  out_st = composite_vanilla(raw_st, z, pm_st)
  nflow = seq.shape[0] if flow_views is None else flow_views
  out["render_flows"] = optical_flow(out["weights"], seq[:nflow],
                                     ray_batch["src_cameras"][:, :nflow],
                                     ray_batch["uv_grid"])
  out["s_vals"] = s
  out["exp_sf"] = expected_scene_flow(out["weights"], traj, sf_k)
  aux = dict(raw_dy=raw_dy, raw_st=raw_st, coeff=coeff, traj=traj, seq=seq,
             rgb_feat_dy=f_dy, rgb_feat_st=f_st, ray_diff_st=rd_st,
             mask_dy=m_dy, mask_st=m_st)
  return out, out_dy, out_st, aux


def render_rays_mv(frame_idx, time_embedding, time_offset, ray_batch, model,
                   projector, coarse_featmaps, fine_featmaps, N_samples, args,
                   inv_uniform=False, N_importance=0, raw_noise_std=0.0,
                   det=False, white_bkgd=False, is_train=True,
                   jitter=None, u=None, return_aux=False):
  """ibrnet/render_ray.py:600-867.  `jitter` / `u` carry the random draws the
  reference makes at :119 / :34 when det=False."""
  assert N_importance > 0
  t = time_embedding[0]
  offs = list(time_offset[0])
  pts, z, _ = sample_along_ray(ray_batch["ray_o"], ray_batch["ray_d"],
                               ray_batch["depth_range"], N_samples, inv_uniform,
                               None if det else jitter)
  ret = {"outputs_coarse": None, "outputs_fine": None}
  with torch.no_grad():
    out_c, _, _, aux_c = _pass(
        ray_batch, coarse_featmaps[0], coarse_featmaps[2], pts, z, None, t,
        frame_idx[0], offs, 0, _sd(model.net_coarse_dy), _sd(model.net_coarse_st),
        _sd(model.motion_mlp), model.trajectory_basis, args,
        getattr(model.net_coarse_dy, "shift", 0.0))
    # the reference's coarse dict has no flow/s_vals/exp_sf (render_ray.py:776-784)
    for k in ("render_flows", "s_vals", "exp_sf"):
      out_c.pop(k)
    ret["outputs_coarse_ref"] = out_c
    zf = resample_depths(z, out_c["weights"].clone(), N_importance, inv_uniform,
                         None if det else u)
  s = z_to_s(zf, ray_batch["depth_range"][0, 0], ray_batch["depth_range"][0, 1])
  pts_f = zf[..., None] * ray_batch["ray_d"][:, None, :] + ray_batch["ray_o"][:, None, :]
  out_f, out_f_dy, _, aux_f = _pass(
      ray_batch, fine_featmaps[0], fine_featmaps[2], pts_f, zf, s, t,
      frame_idx[0], offs, 0, _sd(model.net_fine_dy), _sd(model.net_fine_st),
      _sd(model.motion_mlp_fine), model.trajectory_basis_fine, args,
      getattr(model.net_fine_dy, "shift", 0.0))
  ret["outputs_fine_ref"] = out_f
  ret["outputs_fine_ref_dy"] = out_f_dy
  ret["outputs_fine_anchor"] = None
  ret["outputs_fine_anchor_dy"] = None
  if return_aux:
    ret["_aux_coarse"] = aux_c
    ret["_aux_fine"] = aux_f
  return ret


def render_rays_mono(frame_idx, time_embedding, time_offset, ray_batch, model,
                     featmaps, projector, N_samples, args, inv_uniform=False,
                     N_importance=0, raw_noise_std=0.0, det=False,
                     white_bkgd=False, is_train=True, num_vv=2, jitter=None,
                     return_aux=False):
  """ibrnet/render_ray.py:870-1277, including the training-only cross-time
  branch :1099-1270 (SURVEY row a16) when is_train=True."""
  t = time_embedding[0]
  pts, z, s = sample_along_ray(ray_batch["ray_o"], ray_batch["ray_d"],
                               ray_batch["depth_range"], N_samples, inv_uniform,
                               None if det else jitter)
  w_dy, w_st, w_mo = _sd(model.net_coarse_dy), _sd(model.net_coarse_st), _sd(model.motion_mlp)
  shift = getattr(model.net_coarse_dy, "shift", 0.0)
  out, out_dy, out_st, aux = _pass(
      ray_batch, featmaps[0], featmaps[2], pts, z, s, t, frame_idx[0],
      list(time_offset[0]), num_vv, w_dy, w_st, w_mo, model.trajectory_basis,
      args, shift, flow_views=6, sf_k=1)
  ret = {"outputs_coarse": None, "outputs_fine": None,
         "outputs_coarse_ref": out, "outputs_coarse_ref_dy": out_dy,
         "outputs_coarse_st": out_st}
  if is_train:
    ret.update(_cross_time(ray_batch, featmaps[1], pts, z, aux, frame_idx, time_embedding,
                           time_offset, num_vv, w_dy, w_mo, model.trajectory_basis, shift,
                           args.occ_weights_mode, out, out_dy))
  if return_aux:
    ret["_aux"] = aux
  return ret


def _cross_time(ray_batch, feat_anchor, pts, z, aux, frame_idx, time_embedding, time_offset,
                num_vv, w_dy, w_mo, basis, shift, occ_mode, out_ref, out_ref_dy):
  """Cross-time rendering for temporal consistency (render_ray.py:1099-1270)."""
  ref_idx, anc_idx = frame_idx
  t_anc = time_embedding[1]
  traj = aux["traj"]
  sf_seq = torch.stack([traj[o] - traj[o - 1] for o in (-2, -1, 0, 1, 2, 3)], 0)  # :1101-1105
  pts_anchor = pts + (traj[anc_idx - ref_idx] - traj[0])  # :1109-1112
  coeff_a = motion_coefficients(w_mo, pts_anchor, t_anc)  # :1126-1127
  traj_a0 = traj_offset(coeff_a, basis[anc_idx])
  seq_a, traj_ref_list, traj_anc_list = [], [], []
  for off in time_offset[1]:  # :1149-1168
    ref_off = anc_idx + off - ref_idx
    tmp = pts_anchor + (traj_offset(coeff_a, basis[anc_idx + off]) - traj_a0)
    seq_a.append(tmp)
    if ref_off not in traj:
      continue
    traj_anc_list.append(tmp)
    traj_ref_list.append(pts + traj[ref_off] - traj[0])
  seq_a += [pts_anchor] * num_vv  # :1171-1172
  seq_a = torch.stack(seq_a, 0)
  f_a, _, m_a = project_gather(pts, seq_a, ray_batch["camera"], ray_batch["anchor_src_rgbs"],
                               ray_batch["anchor_src_cameras"], feat_anchor)
  pm_a = m_a[..., 0].sum(2) > 0  # :1198-1200
  ray_dir = F.normalize(ray_batch["ray_d"], dim=-1)
  raw_a = net_dynamic(w_dy, pts_anchor, f_a, ray_dir, m_a, t_anc, shift)
  pm_st = aux["mask_st"][..., 0].sum(2) > 1
  out_a = composite(raw_a, aux["raw_st"], z, pm_a, pm_st)
  out_a_dy = composite_vanilla(raw_a, z, pm_a)
  occ_dy = (out_ref_dy["weights"] - out_a_dy["weights"]).detach()  # :1226
  if occ_mode == 0:  # :1232-1242
    key = "weights_dy" if abs(ref_idx - anc_idx) > 1 else "weights"
  elif occ_mode == 1:
    key = "weights_dy"
  elif occ_mode == 2:
    key = "weights"
  else:
    raise NotImplementedError
  occ = (out_ref[key] - out_a[key]).detach()  # :1254
  out_a["occ_weights"] = 1.0 - occ.abs()
  out_a["occ_weight_map"] = 1.0 - occ.sum(1).abs()
  out_a["pts_traj_ref"] = torch.stack(traj_ref_list, 0)
  out_a["pts_traj_anchor"] = torch.stack(traj_anc_list, 0)
  out_a["sf_seq"] = sf_seq
  out_a_dy["occ_weights"] = 1.0 - occ_dy.abs()
  out_a_dy["occ_weight_map"] = 1.0 - occ_dy.sum(1).abs()
  return {"outputs_coarse_anchor": out_a, "outputs_coarse_anchor_dy": out_a_dy}


# -----------------------------------------------------------------------------
# f1 2-D encoder  (ibrnet/feature_network.py:302-311 with BasicBlock.forward :68-84)
# -----------------------------------------------------------------------------
def _conv_reflect(x, w, stride, pad, bias=None):
  """nn.Conv2d(padding_mode='reflect') (feature_network.py:16-38, :224-232)."""
  if pad:
    x = F.pad(x, (pad, pad, pad, pad), mode="reflect")
  return F.conv2d(x, w, bias, stride=stride)


def _inst_norm(x, w, b):
  """nn.InstanceNorm2d(track_running_stats=False, affine=True), eps 1e-5 (:60-64)."""
  return F.instance_norm(x, weight=w, bias=b, eps=1e-5)


def encoder_forward(w, x):
  """The executed part of ResNet.forward (feature_network.py:302-311): `w` = state_dict (or a dict of leaf
  tensors), x [N,3,H,W] -> (coarse [N,32,H/4,W/4], fine [N,32,H/4,W/4])."""
  w = _sd(w)
  x = torch.relu(_inst_norm(_conv_reflect(x, w["conv1.weight"], 2, 3), w["bn1.weight"], w["bn1.bias"]))
  for b in range(3):
    p = "layer1.%d." % b
    ident = x
    out = _conv_reflect(x, w[p + "conv1.weight"], 2 if b == 0 else 1, 1)
    out = torch.relu(_inst_norm(out, w[p + "bn1.weight"], w[p + "bn1.bias"]))
    out = _inst_norm(_conv_reflect(out, w[p + "conv2.weight"], 1, 1), w[p + "bn2.weight"], w[p + "bn2.bias"])
    if b == 0:  # downsample = conv1x1 stride 2 + InstanceNorm (:243-252)
      ident = _inst_norm(_conv_reflect(x, w[p + "downsample.0.weight"], 2, 0), w[p + "downsample.1.weight"],
                         w[p + "downsample.1.bias"])
    x = torch.relu(out + ident)
  out = _conv_reflect(x, w["out_conv.weight"], 1, 0, w["out_conv.bias"])
  return out[:, :32], out[:, -32:]


# -----------------------------------------------------------------------------
# parity metric (eval_nvidia.py:201-225, full-image branch)
# -----------------------------------------------------------------------------
def psnr(a, b):
  mse = torch.mean((a - b) ** 2).item()
  return float("inf") if mse == 0 else -10.0 * math.log10(mse)
