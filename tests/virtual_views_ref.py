"""Restatement of render_source_vv.py's device work (tests/test_virtual_views_*.py, tests/golden/make_golden_vv.py).

The external `splatting` extension, kornia and skimage cannot run here, so their parts are restated from their
published definitions and pinned by these restatements only:
  splat64          splatting_function('softmax', frame, flow, metric, eps=1e-7): sum-splat of [frame e, e],
                   e = exp(metric), bilinear corners of (x + flow_x, y + flow_y) with NW = floor, each corner outside
                   the image dropped on its own, then sum[:-1] / (sum[-1] + eps);
  sobel_alpha64    kornia.filters.spatial_gradient(mode='sobel', normalized=False) (replicate border), then
                   exp(-beta sqrt(gx^2 + gy^2));
  erode_cross      skimage.morphology.erosion(mask, disk(1)) of skimage 0.19.3 = scipy.ndimage.grey_erosion with the
                   3x3 cross, mode 'reflect' (the edge is repeated at radius 1);
  quantise         render_source_vv.py:313-329 in fp32, as numpy evaluates it.
All sums are float64.  project32 is render_forward_splat's fp32 projection with the operation order of the CUDA
kernel (the reference's matmuls may sum in another order: a tap whose floor flips is the one expected difference).

`plant` selects a deliberate error (PLANTS) so the tests can show the comparison bars would catch it.
"""

import numpy as np
import torch

EPS = 1e-7
PLANTS = ("trunc_for_floor", "no_eps", "batch_minmax", "zero_pad", "square_erosion", "swap_ne_sw")


def splat64(frame, flow, metric, plant=None):
  """frame [B, C, H, W], flow [B, 2, H, W], metric [B, 1, H, W] (any float type) -> float64 [B, C, H, W]."""
  frame, flow, metric = (np.asarray(torch.as_tensor(a).detach().cpu().double()) for a in (frame, flow, metric))
  B, C, H, W = frame.shape
  e = np.exp(metric[:, 0])
  vals = np.concatenate([frame * e[:, None], e[:, None]], 1).reshape(B, C + 1, -1)  # [B, C+1, HW]
  # the extension adds the fp32 flow to the fp32 pixel coordinate
  ys, xs = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
  ox = (xs[None] + np.asarray(flow[:, 0], np.float32)).astype(np.float64).reshape(B, -1)
  oy = (ys[None] + np.asarray(flow[:, 1], np.float32)).astype(np.float64).reshape(B, -1)
  rnd = np.trunc if plant == "trunc_for_floor" else np.floor
  with np.errstate(invalid="ignore"):
    nx, ny = rnd(ox), rnd(oy)
  acc = np.zeros((B, C + 1, H * W))
  corners = [(0, 0, (nx + 1 - ox) * (ny + 1 - oy)), (1, 0, (ox - nx) * (ny + 1 - oy)),
             (0, 1, (nx + 1 - ox) * (oy - ny)), (1, 1, (ox - nx) * (oy - ny))]
  if plant == "swap_ne_sw":
    corners[1], corners[2] = (1, 0, corners[2][2]), (0, 1, corners[1][2])
  for dx, dy, w in corners:
    cx, cy = nx + dx, ny + dy
    ok = np.isfinite(cx) & np.isfinite(cy) & (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
    for b in range(B):
      k = ok[b]
      tgt = (cy[b, k] * W + cx[b, k]).astype(np.int64)
      for c in range(C + 1):
        np.add.at(acc[b, c], tgt, vals[b, c, k] * w[b, k])
  den = acc[:, -1:] + (0.0 if plant == "no_eps" else EPS)
  with np.errstate(invalid="ignore", divide="ignore"):
    return (acc[:, :-1] / den).reshape(B, C, H, W)


def project32(src_depths, r_cam, t_cam, k_src, k_dst):
  """render_forward_splat:21-53 in fp32: returns (flow [B, 2, H, W], 1 / new_z [B, 1, H, W]) as fp32 tensors."""
  d = torch.as_tensor(src_depths).float().cpu()
  B, H, W = d.shape
  f = lambda a: torch.as_tensor(a).detach().float().cpu()
  ki, r, t, kd = f(k_src).inverse(), f(r_cam), f(t_cam), f(k_dst)
  ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
  def mv(m, v, add=None):
    out = [(m[:, i, 0, None, None] * v[0] + m[:, i, 1, None, None] * v[1]) + m[:, i, 2, None, None] * v[2]
           for i in range(3)]
    return out if add is None else [out[i] + add[:, i, None, None] for i in range(3)]
  q = [(d * ki[:, i, 0, None, None]) * xs + (d * ki[:, i, 1, None, None]) * ys + d * ki[:, i, 2, None, None]
       for i in range(3)]
  p = mv(kd, mv(r, q, t))
  z = p[2]
  zc = torch.clamp(z, 1e-8, None)
  flow = torch.stack([p[0] / zc - xs, p[1] / zc - ys], 1)
  return flow, (1.0 / z)[:, None]


def weights32(inv_z, plant=None):
  """(imp - min) / (max - min + 1e-6) * 20 - 10 in fp32, min / max per batch item (plant: over the whole batch)."""
  dims = (0, 1, 2, 3) if plant == "batch_minmax" else (1, 2, 3)
  lo, hi = inv_z.amin(dims, keepdim=True), inv_z.amax(dims, keepdim=True)
  return (inv_z - lo) / (hi - lo + 1e-6) * 20 - 10


def render_forward_splat64(src_imgs, src_depths, r_cam, t_cam, k_src, k_dst, plant=None):
  """render_forward_splat: fp32 projection and weights, float64 splat.  Returns float64 ([B, C, H, W], [B, 1, H, W])."""
  flow, inv_z = project32(src_depths, r_cam, t_cam, k_src, k_dst)
  w = weights32(inv_z, plant)
  imgs = torch.as_tensor(src_imgs).float().cpu().permute(0, 3, 1, 2)
  C = imgs.shape[1]
  out = splat64(torch.cat([imgs, inv_z], 1), flow, w, plant)
  return out[:, :C], out[:, C:C + 1]


def sobel_alpha64(x, beta, plant=None):
  """x [N, H, W] -> float64 alpha [N, H, W]."""
  x = np.asarray(torch.as_tensor(x).detach().cpu().double())
  if plant == "zero_pad":
    p = np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="constant")
  else:
    p = np.pad(x, ((0, 0), (1, 1), (1, 1)), mode="edge")
  H, W = x.shape[1:]
  a = lambda j, i: p[:, j:j + H, i:i + W]
  gx = (a(0, 2) - a(0, 0)) + 2 * (a(1, 2) - a(1, 0)) + (a(2, 2) - a(2, 0))
  gy = (a(2, 0) - a(0, 0)) + 2 * (a(2, 1) - a(0, 1)) + (a(2, 2) - a(0, 2))
  return np.exp(-beta * np.sqrt(gx * gx + gy * gy))


def erode_cross(mask, plant=None):
  """Binary erosion of mask [..., H, W] by the 3x3 cross (plant: the 3x3 square), edge repeated."""
  m = np.pad(np.asarray(mask, bool), [(0, 0)] * (mask.ndim - 2) + [(1, 1), (1, 1)], mode="edge")
  H, W = mask.shape[-2:]
  out = np.ones(mask.shape, bool)
  for j in range(3):
    for i in range(3):
      if plant == "square_erosion" or j == 1 or i == 1:
        out &= m[..., j:j + H, i:i + W]
  return out


def quantise(F, plant=None):
  """Splatted rgba F [V, 4, H, W] -> uint8 [V, H, W, 3], render_source_vv.py:313-329 in fp32."""
  F = np.asarray(torch.as_tensor(F).detach().cpu().float())
  rgb = np.clip(F[:, :3].transpose(0, 2, 3, 1) / np.float32(255.0), 0.0, 1.0).astype(np.float32)
  mask = erode_cross(np.clip(F[:, 3], 0.0, 1.0) > 0.5, plant)
  return np.uint8(np.float32(255) * np.clip(rgb * mask[..., None], 0.0, 1.0))


def views_from_splat_inputs(rgba, flow, weights, plant=None):
  """The per-frame product from the splat's inputs: rgba [H, W, 4] shared by V views, flow [V, 2, H, W],
  weights [V, 1, H, W] -> uint8 [V, H, W, 3].  (The splat's 1 / z and ones channels are summed independently and
  unused.)"""
  V = flow.shape[0]
  frame = torch.as_tensor(rgba).float().permute(2, 0, 1)[None].expand(V, -1, -1, -1)
  F = splat64(frame, flow, weights, plant)
  return quantise(torch.from_numpy(F).float(), plant)


def rgba_of_frame(img, disp, plant=None):
  """rgba [H, W, 4] fp32 = [img * 255, alpha((1 / disp) / 10, beta 0.5)] (render_source_vv.py:283-297)."""
  img = np.asarray(img, np.float32)
  depth10 = (np.float32(1.0) / np.asarray(disp, np.float32)) / np.float32(10.0)
  alpha = sobel_alpha64(depth10[None], 0.5, plant)[0].astype(np.float32)
  return np.concatenate([img * np.float32(255.0), alpha[..., None]], -1).astype(np.float32)


# ---- cases shared by the CPU and GPU tests ------------------------------------------------------------------------
# Bars: max abs error of the GPU against the restatement, per tensor, at 2x the worst measured on an H100 SXM (80 GB
# HBM3, 700 W power limit): splat 1.78e-6 (the 12 000-source pile-up), forward-splat image 3.49e-7 and 1 / z 3.31e-7,
# Sobel alpha 1.12e-7 (DESIGN §3.5).
BARS = {"splat": 3.6e-6, "forward_image": 7e-7, "forward_disp": 7e-7, "sobel": 2.3e-7}
# render_virtual_views: share of bytes more than 1 LSB off, against the restatement on the synthetic 288 x 512 frame
# and against the reference's own PNGs.  Both measured 0 on the H100 (the kernels are deterministic, so a repeat
# cannot differ): no byte may be more than 1 LSB off.
PNG_FRAC_BAR = 0.0
PNG_FRAC_FIXTURE_BAR = 0.0


def ratio(err, bar):
  """err in units of bar (a zero bar: any error is infinitely far over it)."""
  return err / bar if bar > 0 else (float("inf") if err > 0 else 0.0)


def max_err(got, want):
  """max |got - want| over finite pairs; inf when one side is NaN / inf where the other is not."""
  got, want = (np.asarray(torch.as_tensor(a).detach().cpu().double()) for a in (got, want))
  fg, fw = np.isfinite(got), np.isfinite(want)
  if (fg != fw).any():
    return float("inf")
  return float(np.abs(got[fg] - want[fw]).max(initial=0.0))


def splat_case(name):
  """(frame [B, C, H, W], flow [B, 2, H, W], metric [B, 1, H, W]) fp32, seeded.
  odd: odd H and W; edges: taps off every edge and into (-1, 0); pileup: 12 000 sources in one cell;
  batch: B = 3."""
  g = torch.Generator().manual_seed({"odd": 1, "edges": 2, "pileup": 3, "batch": 4}[name])
  B, C, H, W = {"odd": (1, 3, 37, 53), "edges": (1, 2, 24, 31), "pileup": (1, 4, 128, 128), "batch": (3, 2, 29, 40)}[name]
  frame = torch.rand(B, C, H, W, generator=g)
  metric = torch.rand(B, 1, H, W, generator=g) * 20 - 10
  flow = torch.randn(B, 2, H, W, generator=g) * 2.5
  if name == "edges":
    flow = (torch.rand(B, 2, H, W, generator=g) - 0.5) * 1.6 * torch.tensor([W, H]).view(1, 2, 1, 1).float()
    xs = torch.arange(W).float().view(1, 1, W)
    ys = torch.arange(H).float().view(1, H, 1)
    flow[:, 0, ::3] = -xs - torch.rand(B, H // 3 + (H % 3 > 0), W, generator=g)  # x + flow in (-1, 0]
    flow[:, 1, :, ::4] = -ys - torch.rand(B, H, W // 4 + (W % 4 > 0), generator=g)
  if name == "pileup":
    n = 12000
    sel = torch.randperm(H * W, generator=g)[:n]
    tx = 37.0 + 0.98 * torch.rand(n, generator=g) + 0.01
    ty = 60.0 + 0.98 * torch.rand(n, generator=g) + 0.01
    fx, fy = flow[0, 0].flatten(), flow[0, 1].flatten()
    fx[sel] = tx - (sel % W).float()
    fy[sel] = ty - (sel // W).float()
  return frame, flow, metric


def forward_case(name):
  """(src_imgs [B, H, W, C], src_depths [B, H, W], r [B, 3, 3], t [B, 3], k [B, 3, 3]) fp32, seeded.
  batch: 288 x 512, B = 2 with depth ranges 1-5 and 20-60; const: constant depth (max = min)."""
  g = torch.Generator().manual_seed({"batch": 5, "const": 6}[name])
  B, H, W = {"batch": (2, 288, 512), "const": (1, 33, 47)}[name]
  imgs = torch.rand(B, H, W, 4, generator=g)
  if name == "const":
    depths = torch.full((B, H, W), 3.0)
  else:
    u = torch.rand(B, H, W, generator=g)
    depths = torch.stack([1.0 + 4.0 * u[0], 20.0 + 40.0 * u[1]])
  a = (torch.rand(B, 3, generator=g) - 0.5) * 0.1
  Kx = torch.zeros(B, 3, 3)
  Kx[:, 0, 1], Kx[:, 0, 2], Kx[:, 1, 2] = -a[:, 2], a[:, 1], -a[:, 0]
  Kx = Kx - Kx.transpose(1, 2)
  r = torch.linalg.matrix_exp(Kx.double()).float()
  t = (torch.rand(B, 3, generator=g) - 0.5) * 0.4
  f = 0.9 * W
  k = torch.tensor([[f, 0.0, W / 2.0], [0.0, f, H / 2.0], [0.0, 0.0, 1.0]]).expand(B, 3, 3).contiguous()
  return imgs, depths, r, t, k


def sobel_case():
  """a [2, 288, 512] plane with smooth structure, steps and noise."""
  g = torch.Generator().manual_seed(8)
  ys, xs = torch.meshgrid(torch.arange(288).float(), torch.arange(512).float(), indexing="ij")
  base = 0.3 + 0.1 * torch.sin(xs / 17.0) * torch.cos(ys / 11.0) + 0.2 * (xs > 300).float()
  return torch.stack([base, base.flip(1)]) + 0.01 * torch.rand(2, 288, 512, generator=g)


def fixture_frame_inputs(fx, i, views=None):
  """From the fixture: frame i's resized img, disp, its scaled K, ref2w and the virtual cameras (tgt c2w [8, 3, 4],
  float64) as the reference computes them."""
  from dynibar_b200 import virtual_views as vv
  npz = fx["npz"]
  H, W = fx["final_hw"]
  Ks = [vv.scaled_intrinsics(z["K"], z["img_1"].shape[2:], (H, W)) for z in npz]
  _, c2w = vv.virtual_view_poses(np.stack([z["cam_c2w"][0] for z in npz]), [z["depth"][0, 0] for z in npz], Ks[-1],
                                 (H, W))
  f = fx["frames"][i]
  return f["img"], f["disp"], Ks[i], npz[i]["cam_c2w"][0], c2w[i]


def ref2tgt(ref2w, tgt_c2w):
  """R [V, 3, 3], t [V, 3] fp32 of T_ref2tgt = inv(tgt2w) ref2w computed in float64 (render_source_vv.py:301-306)."""
  R, t = [], []
  for c in tgt_c2w:
    tgt2w = np.eye(4)
    tgt2w[:3, :4] = c
    T = np.dot(np.linalg.inv(tgt2w), ref2w)
    R.append(torch.from_numpy(T[:3, :3]).float())
    t.append(torch.from_numpy(T[:3, 3]).float())
  return torch.stack(R), torch.stack(t)


def decode_pngs(blobs):
  import io
  from PIL import Image
  return np.stack([np.asarray(Image.open(io.BytesIO(b))) for b in blobs])


def frame_case():
  """One synthetic 288 x 512 frame with near objects in front of a slanted background: (img [H, W, 3], disp [H, W],
  K [3, 3], ref2w [4, 4], tgt_c2w [8, 3, 4] float64 from virtual_view_poses)."""
  from dynibar_b200 import virtual_views as vv
  g = np.random.default_rng(9)
  H, W = 288, 512
  ys, xs = np.mgrid[0:H, 0:W].astype(np.float32)
  depth = 8.0 + 6.0 * ys / H + g.uniform(0, 0.05, (H, W))
  depth[(xs - 150) ** 2 + (ys - 140) ** 2 < 70 ** 2] = 1.5
  depth[60:230, 330:420] = 2.5 + 0.3 * g.random()
  disp = (1.0 / depth).astype(np.float32)
  img = (0.5 + 0.3 * np.sin(xs / 9.0)[..., None] * np.cos(ys / 13.0)[..., None] * np.array([1.0, -0.6, 0.8])
         + g.uniform(0, 0.15, (H, W, 3))).astype(np.float32)
  K = np.array([[400.0, 0.0, W / 2.0], [0.0, 401.0, H / 2.0], [0.0, 0.0, 1.0]], np.float32)
  ref2w = np.eye(4, dtype=np.float32)
  ref2w[:3, 3] = [0.1, -0.2, 0.05]
  _, c2w = vv.virtual_view_poses(ref2w[None], [depth], K, (H, W))
  return img, disp, K, ref2w, c2w[0]


def views64(img, disp, K, ref2w, tgt_c2w, plant=None):
  """render_virtual_views restated: uint8 [V, H, W, 3]."""
  rgba = torch.from_numpy(rgba_of_frame(img, disp, plant))
  R, t = ref2tgt(np.asarray(ref2w), tgt_c2w)
  V = R.shape[0]
  k = torch.from_numpy(np.array(K)).float()[None].expand(V, 3, 3)
  depth = (1.0 / torch.as_tensor(disp).float())[None].expand(V, -1, -1)
  flow, inv_z = project32(depth, R, t, k, k)
  return views_from_splat_inputs(rgba, flow, weights32(inv_z, plant), plant)


def png_mismatch(got, want):
  """Share of bytes more than 1 LSB apart."""
  return float((np.abs(np.asarray(got).astype(int) - np.asarray(want).astype(int)) > 1).mean())
