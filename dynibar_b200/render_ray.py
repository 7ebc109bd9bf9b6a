"""Per-ray renderer: drop-in for ibrnet/render_ray.py on the CUDA library.

Public surface (same names / signatures / returned dict keys as the
reference): `render_rays_mv` (render_ray.py:600), `render_rays_mono` (:870),
`sample_along_camera_ray` (:67), `raw2outputs` (:214), `raw2outputs_vanilla`
(:134), `compute_optical_flow` (:333), `compute_ref_plucker_coordinate` (:372),
`compute_src_plucker_coordinate` (:380), `z_to_s` (:399).

All math runs in `csrc/` kernels through the C ABI (include/dynibar_b200.h);
this file only allocates tensors and sequences calls.  `render_rays_mono` is
differentiable (training, SURVEY 8(f) f2): when gradients are enabled and the
model's parameters, its trajectory basis or the feature maps require grad it runs
the training path (`_render_mono_train`, autograd Functions of
dynibar_b200/autograd.py over the backward kernels).  `render_rays_mv` trains its
fine stage the same way (`_render_mv_train`) when a fine-stage tensor requires
grad; its coarse pass always runs under no_grad, as in the reference.
"""

from collections import OrderedDict
import contextlib
import ctypes as C
import os
import threading
import weakref

import torch

from dynibar_b200 import _lib
from dynibar_b200 import weights as _weights
from dynibar_b200._lib import lib, ptr, f32c, check, stream, dev_of, Args
from dynibar_b200.projection import project_gather

# GEMM precision of the network kernels: "bf16" = tensor cores (bf16 operands / fp32 accumulate and statistics; the
# production mode and the default), "fp32" = SIMT everywhere (parity mode).  Three ways to choose, innermost wins:
# the `precision=` argument of render_rays_mv / render_rays_mono (per call), `precision_scope(name)` (per
# thread, a context manager), `set_precision(name)` / the DYNIBAR_B200_PRECISION environment variable (process
# default).
_PREC = {"fp32": _lib.PREC_FP32, "bf16": _lib.PREC_BF16}
PRECISION = _PREC[os.environ.get("DYNIBAR_B200_PRECISION", "bf16")]
_tls = threading.local()
# DYN_PREC_BF16: use the fused per-view kernels (False = staged tensor-core layers)
USE_FUSED = True


def set_precision(name):
  """Process-wide default ("fp32" | "bf16")."""
  global PRECISION
  PRECISION = _PREC[name]


@contextlib.contextmanager
def precision_scope(name):
  """Precision of every library call made by this thread inside the block (None = leave unchanged)."""
  if name is None:
    yield
    return
  prev = getattr(_tls, "override", None)
  _tls.override = _PREC[name]
  try:
    yield
  finally:
    _tls.override = prev


def _prec():
  o = getattr(_tls, "override", None)
  return PRECISION if o is None else o


def _no_grad_only(*tensors):
  if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
    raise NotImplementedError(
        "dynibar_b200 kernels are forward-only (training backward = SURVEY 8(f) f2); "
        "call under torch.no_grad() with detached inputs")


def _wants_grad(model, *featmaps):
  """True when gradients are enabled and a parameter of the model, a tensor of the model (the trajectory basis) or a
  feature map requires grad."""
  if not torch.is_grad_enabled():
    return False
  mods = [m for m in vars(model).values() if isinstance(m, torch.nn.Module)]
  live = any(p.requires_grad for m in mods for p in m.parameters())
  live = live or any(torch.is_tensor(v) and v.requires_grad for v in vars(model).values())
  return live or any(torch.is_tensor(f) and f.requires_grad for fm in featmaps if fm is not None
                     for f in fm if f is not None)


_FINE_MODULES = ("net_fine_dy", "net_fine_st", "motion_mlp_fine")


def _fine_stage_wants_grad(model, fine_featmaps):
  """True when gradients are enabled and a tensor of render_rays_mv's fine stage requires grad: a parameter of
  net_fine_dy / net_fine_st / motion_mlp_fine, trajectory_basis_fine, or the fine feature maps [0] / [2] (what
  DynibarFF's optimiser updates, ibrnet/model.py:94-118).  The coarse stage never trains here: the reference runs
  it under no_grad (render_ray.py:672)."""
  if not torch.is_grad_enabled():
    return False
  mods = [getattr(model, k, None) for k in _FINE_MODULES]
  if any(p.requires_grad for m in mods if m is not None for p in m.parameters()):
    return True
  basis = getattr(model, "trajectory_basis_fine", None)
  if torch.is_tensor(basis) and basis.requires_grad:
    return True
  fm = fine_featmaps if fine_featmaps is not None else ()
  return any(torch.is_tensor(f) and f.requires_grad for f in (fm[0], fm[2]) if f is not None)


def _scalar(x):
  return float(x.reshape(-1)[0]) if torch.is_tensor(x) else float(x)


# ---------------------------------------------------------------------------
# a2
# ---------------------------------------------------------------------------
def sample_along_camera_ray(ray_o, ray_d, depth_range, N_samples, inv_uniform=False, det=False,
                            jitter=None):
  """render_ray.py:67-131.  `jitter` ([R,N_samples] U[0,1)) lets a caller
  supply the random draws; with det=False and jitter=None they are drawn with
  torch.rand like the reference (:119)."""
  R = ray_o.shape[0]
  dev = dev_of(ray_o)
  near, far = _scalar(depth_range[0, 0]), _scalar(depth_range[0, 1])
  assert near > 0 and far > 0 and far > near
  if not det and jitter is None:
    jitter = torch.rand(R, N_samples, device=dev)
  if det:
    jitter = None
  pts = torch.empty(R, N_samples, 3, device=dev)
  z = torch.empty(R, N_samples, device=dev)
  s = torch.empty(R, N_samples, device=dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_sample_rays(A(ray_o), A(ray_d), near, far, R, N_samples,
                              int(bool(inv_uniform)),
                              A(jitter),
                              ptr(pts), ptr(z), ptr(s), stream()))
  return pts, z, s


def z_to_s(z_vals, near_depth_value, far_depth_value):
  """render_ray.py:399-404 (elementwise; kept in torch, it is not on the hot
  path -- the kernels emit s_vals directly)."""
  return ((1.0 / z_vals) - (1.0 / near_depth_value)) / (1.0 / far_depth_value - 1.0 / near_depth_value)


def points_from_depths(ray_o, ray_d, z_vals, depth_range):
  R, S = z_vals.shape
  dev = dev_of(z_vals)
  near, far = _scalar(depth_range[0, 0]), _scalar(depth_range[0, 1])
  pts = torch.empty(R, S, 3, device=dev)
  s = torch.empty(R, S, device=dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_points_from_depths(A(ray_o), A(ray_d), A(z_vals), near,
                                     far, R, S, ptr(pts), ptr(s), stream()))
  return pts, s


# ---------------------------------------------------------------------------
# a3
# ---------------------------------------------------------------------------
def motion_mlp_forward(module, xyzt):
  """MotionMLP.forward on [...,4] rows (mlp_network.py:605-618)."""
  _no_grad_only(xyzt)
  dev = dev_of(xyzt)
  net = _weights.packed_of(module, dev)
  x = f32c(xyzt).reshape(-1, 4)
  N = x.shape[0]
  out = torch.empty(N, 3 * net.num_basis, device=dev)
  nbytes = lib.dyn_motion_workspace_bytes(N, 1)
  ws = _lib.workspace.get(nbytes, dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_motion_mlp(net.handle, ptr(x), N, ptr(out), ws.data_ptr(), nbytes, _prec(),
                             stream()))
  div = float(getattr(_weights.de_parallel(module), "sf_mag_div", 1.0))
  if div != 1.0:
    out = out / div
  return out.reshape(xyzt.shape[:-1] + (out.shape[-1],))


def motion_coefficients(module, pts, t):
  """coeffs [R,S,3*nb], last round(0.1*S) samples zeroed (render_ray.py:459-472)."""
  dev = dev_of(pts)
  net = _weights.packed_of(module, dev)
  R, S = pts.shape[:2]
  out = torch.empty(R, S, 3 * net.num_basis, device=dev)
  nbytes = lib.dyn_motion_workspace_bytes(R, S)
  ws = _lib.workspace.get(nbytes, dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_motion_coeffs(net.handle, A(pts), float(t), R, S, ptr(out),
                                ws.data_ptr(), nbytes, _prec(), stream()))
  div = float(getattr(_weights.de_parallel(module), "sf_mag_div", 1.0))
  if div != 1.0:  # MotionMLP.forward divides its output (mlp_network.py:617)
    out = out / div
  return out


def displaced_points(pts, coeff, basis, frame_idx, offsets, num_vv=0):
  """pts_3d_seq [len(offsets)+num_vv, R, S, 3] (render_ray.py:479-497, :988-991)."""
  dev = dev_of(pts)
  R, S = pts.shape[:2]
  n_off = len(offsets)
  T, nb = basis.shape
  seq = torch.empty(n_off + num_vv, R, S, 3, device=dev)
  offs = (C.c_int * max(n_off, 1))(*[int(o) for o in offsets])
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_traj_displace(A(pts), A(coeff), A.host(basis), T, nb,
                                int(frame_idx), offs, n_off, int(num_vv), R, S, ptr(seq), stream()))
  return seq


def traj_deltas(coeff, basis, frames_a, frames_b):
  """traj(frames_a[v]) - traj(frames_b[v]) -> [n,R,S,3] (scene-flow sequence,
  render_ray.py:1101-1105)."""
  dev = dev_of(coeff)
  R, S = coeff.shape[:2]
  n = len(frames_a)
  T, nb = basis.shape
  out = torch.empty(n, R, S, 3, device=dev)
  fa = (C.c_int * n)(*[int(f) for f in frames_a])
  fb = (C.c_int * n)(*[int(f) for f in frames_b])
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_traj_delta(A(coeff), A.host(basis), T, nb, fa, fb, n, R, S, ptr(out), stream()))
  return out


def occlusion_weights(w_ref, w_anchor):
  """occ_weights, occ_weight_map (render_ray.py:1224-1257)."""
  dev = dev_of(w_ref)
  R, S = w_ref.shape
  occ = torch.empty(R, S, device=dev)
  occ_map = torch.empty(R, device=dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_occlusion_weights(A(w_ref), A(w_anchor), R, S, ptr(occ), ptr(occ_map), stream()))
  return occ, occ_map


# ---------------------------------------------------------------------------
# a7
# ---------------------------------------------------------------------------
def compute_ref_plucker_coordinate(ray_o, ray_d):
  R = ray_o.shape[0]
  out = torch.empty(R, 6, device=dev_of(ray_o))
  A = Args()
  with torch.cuda.device(ray_o.device):
    check(lib.dyn_plucker_ref(A(ray_o), A(ray_d), R, ptr(out), stream()))
  return out


def compute_src_plucker_coordinate(pts, src_cameras, camera_index=None, view_tbl=None):
  """pts [R,S,3], src_cameras [1,V,34] -> [R,S,V,6] (render_ray.py:380-396).  With `view_tbl` ([K,V] int32, host)
  src_cameras is a pool [1,P,34] and slot v of ray r is pool entry view_tbl[camera_index[r], v]."""
  R, S = pts.shape[:2]
  V = src_cameras.shape[1] if view_tbl is None else view_tbl.shape[1]
  out = torch.empty(R, S, V, 6, device=dev_of(pts))
  A = Args()
  with torch.cuda.device(pts.device):
    if view_tbl is None:
      check(lib.dyn_plucker_src(A(pts), A.host(src_cameras), V, R, S, ptr(out), stream()))
    else:
      check(lib.dyn_plucker_src_tbl(A(pts), A.host(src_cameras), src_cameras.shape[1], view_tbl.shape[0],
                                    A(camera_index, torch.int32) if camera_index is not None else None,
                                    A.host_i32(view_tbl), V, R, S, ptr(out), stream()))
  return out


# ---------------------------------------------------------------------------
# a8-a11
# ---------------------------------------------------------------------------
def net_dynamic_forward(module, pts, rgb_feat, ray_dir, mask, time):
  """DynibarDynamic.forward (mlp_network.py:236-316).  `time` is the
  reference's [R,S,1] tensor (constant) or a scalar."""
  _no_grad_only(pts, rgb_feat)
  dev = dev_of(pts)
  net = _weights.packed_of(module, dev)
  R, S, V = rgb_feat.shape[:3]
  raw = torch.empty(R, S, 4, device=dev)
  nbytes = lib.dyn_net_workspace_bytes(_lib.NET_DYNAMIC, R, S, V)
  ws = _lib.workspace.get(nbytes, dev)
  t = _scalar(time.float() if torch.is_tensor(time) else time)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_net_dynamic(net.handle, A(pts), A(rgb_feat), A(ray_dir),
                              A(mask), t, R, S, V, ptr(raw), ws.data_ptr(), nbytes,
                              _prec(), stream()))
  return raw


def net_static_forward(module, pts, ref_rays, src_rays, rgb_feat, ray_diff, mask):
  """DynibarStatic.forward (mlp_network.py:423-527)."""
  _no_grad_only(pts, rgb_feat)
  dev = dev_of(pts)
  net = _weights.packed_of(module, dev)
  R, S, V = rgb_feat.shape[:3]
  raw = torch.empty(R, S, 4, device=dev)
  nbytes = lib.dyn_net_workspace_bytes(_lib.NET_STATIC, R, S, V)
  ws = _lib.workspace.get(nbytes, dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_net_static(net.handle, A(pts), A(ref_rays), A(src_rays),
                             A(rgb_feat), A(ray_diff), A(mask), R, S, V,
                             ptr(raw), ws.data_ptr(), nbytes, _prec(), stream()))
  return raw


# ---------------------------------------------------------------------------
# fused a4-a11 (DYN_PREC_BF16): gather + per-view MLP chain in one tensor-core kernel
# ---------------------------------------------------------------------------
class _FrameCache(object):
  """Packed per-frame copies of the source views, keyed by the IDENTITY of the source tensor (a weak
  reference plus its version counter), so the 18 chunks x 2 passes of one frame pack each map once
  while a new frame -- new tensor objects, or the same ones modified in place -- is packed again."""

  def __init__(self, capacity=16):
    self.entries = OrderedDict()
    self.capacity = capacity

  def get(self, tag, src, make):
    key = (tag, id(src))
    e = self.entries.get(key)
    if e is not None and e[0]() is src and e[1] == src._version:
      return e[2]
    packed = make(src)
    self.entries[key] = (weakref.ref(src), src._version, packed)
    self.entries.move_to_end(key)
    while len(self.entries) > self.capacity:
      self.entries.popitem(last=False)
    return packed


_frame_cache = _FrameCache()


def new_frame():
  """Drop the packed per-frame copies (a frame driver may call this when the source views change in place
  without their tensors' version counters noticing, e.g. after a collective wrote into them)."""
  _frame_cache.entries.clear()


def _pack_featmaps(featmaps):
  V, Cc, h, w = featmaps.shape
  dev = dev_of(featmaps)
  out = torch.empty(V, h, w, Cc, dtype=torch.bfloat16, device=dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_featmaps_channels_last(A(featmaps), ptr(out, torch.bfloat16), V, Cc, h, w, stream()))
  return out


def _pack_rgba(src_rgbs):
  _, V, H, W, _ = src_rgbs.shape
  dev = dev_of(src_rgbs)
  out = torch.empty(V, H, W, 4, device=dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_rgbs_rgba(A(src_rgbs), ptr(out), V, H, W, stream()))
  return out


def featmaps_channels_last(featmaps):
  """[V,C,h,w] fp32 -> channels-last bf16 [V,h,w,C] on the device (one bilinear tap of all 32 channels
  = 64 contiguous bytes); packed once per frame."""
  return _frame_cache.get("feat", featmaps, _pack_featmaps)


def source_rgba(src_rgbs):
  """[1,V,H,W,3] fp32 -> [V,H,W,4] fp32 (one tap = one aligned 16-byte load); packed once per frame."""
  return _frame_cache.get("rgba", src_rgbs, _pack_rgba)


def net_static_fused(module, pts, ray_o, ray_d, query_cam, src_rgbs, src_cams, feat_cl, camera_index=None,
                     view_tbl=None):
  """Projector.compute_with_motions + DynibarStatic.forward fused
  (projection.py:103-176 + mlp_network.py:423-527) -> raw [R,S,4], mask [R,S,V,1].
  With `camera_index` ([R] int32, device) query_cam is [K,34] and ray r is seen from camera camera_index[r]
  (values trusted to lie in [0, K)).  With `view_tbl` ([K,V] int32, host) the source views are a pool and slot v
  of ray r reads pool entry view_tbl[camera_index[r], v]."""
  dev = dev_of(pts)
  net = _weights.packed_of(module, dev)
  R, S = pts.shape[:2]
  V = src_cams.shape[1] if view_tbl is None else view_tbl.shape[1]
  _, _, H, W, _ = src_rgbs.shape
  _, h, w, Cc = feat_cl.shape
  raw = torch.empty(R, S, 4, device=dev)
  mask = torch.empty(R, S, V, 1, device=dev)
  nbytes = lib.dyn_net_fused_workspace_bytes(_lib.NET_STATIC, R, S, V)
  ws = _lib.workspace.get(nbytes, dev)
  A = Args()
  with torch.cuda.device(dev):
    if view_tbl is not None:
      check(lib.dyn_net_static_fused_tbl(net.handle, A(pts), A(ray_o), A(ray_d), A.host(query_cam),
                                         query_cam.shape[0], A(camera_index, torch.int32)
                                         if camera_index is not None else None, A.host_i32(view_tbl),
                                         src_cams.shape[1], ptr(source_rgba(src_rgbs)), A.host(src_cams),
                                         ptr(feat_cl, torch.bfloat16), R, S, V, H, W, Cc, h, w, ptr(raw),
                                         ptr(mask), ws.data_ptr(), nbytes, stream()))
    elif camera_index is None:
      check(lib.dyn_net_static_fused(net.handle, A(pts), A(ray_o), A(ray_d), A.host(query_cam),
                                     ptr(source_rgba(src_rgbs)), A.host(src_cams),
                                     ptr(feat_cl, torch.bfloat16), R, S, V, H, W, Cc, h, w, ptr(raw),
                                     ptr(mask), ws.data_ptr(), nbytes, stream()))
    else:
      assert camera_index.shape == (R,)
      check(lib.dyn_net_static_fused_mc(net.handle, A(pts), A(ray_o), A(ray_d), A.host(query_cam),
                                        query_cam.shape[0], A(camera_index, torch.int32),
                                        ptr(source_rgba(src_rgbs)), A.host(src_cams),
                                        ptr(feat_cl, torch.bfloat16), R, S, V, H, W, Cc, h, w, ptr(raw),
                                        ptr(mask), ws.data_ptr(), nbytes, stream()))
  return raw, mask


def net_dynamic_fused(module, pts, pts_seq, ray_dir, query_cam, src_rgbs, src_cams, feat_cl, time,
                      camera_index=None, view_tbl=None):
  """Projector.compute_with_motions + DynibarDynamic.forward fused
  (projection.py:103-176 + mlp_network.py:236-316) -> raw [R,S,4], mask [R,S,V,1].  `camera_index` /
  `view_tbl` as for net_static_fused (query_cam stays one camera: the dynamic net's outputs do not read it)."""
  dev = dev_of(pts)
  net = _weights.packed_of(module, dev)
  R, S = pts.shape[:2]
  V = src_cams.shape[1] if view_tbl is None else view_tbl.shape[1]
  _, _, H, W, _ = src_rgbs.shape
  _, h, w, Cc = feat_cl.shape
  raw = torch.empty(R, S, 4, device=dev)
  mask = torch.empty(R, S, V, 1, device=dev)
  nbytes = lib.dyn_net_fused_workspace_bytes(_lib.NET_DYNAMIC, R, S, V)
  ws = _lib.workspace.get(nbytes, dev)
  A = Args()
  with torch.cuda.device(dev):
    if view_tbl is not None:
      check(lib.dyn_net_dynamic_fused_tbl(net.handle, A(pts), A(pts_seq), A(ray_dir), A.host(query_cam),
                                          view_tbl.shape[0], A(camera_index, torch.int32)
                                          if camera_index is not None else None, A.host_i32(view_tbl),
                                          src_cams.shape[1], ptr(source_rgba(src_rgbs)), A.host(src_cams),
                                          ptr(feat_cl, torch.bfloat16), float(time), R, S, V, H, W, Cc, h, w,
                                          ptr(raw), ptr(mask), ws.data_ptr(), nbytes, stream()))
    else:
      check(lib.dyn_net_dynamic_fused(net.handle, A(pts), A(pts_seq), A(ray_dir), A.host(query_cam),
                                      ptr(source_rgba(src_rgbs)), A.host(src_cams),
                                      ptr(feat_cl, torch.bfloat16), float(time), R, S, V, H, W,
                                      Cc, h, w, ptr(raw), ptr(mask), ws.data_ptr(), nbytes, stream()))
  return raw, mask


# ---------------------------------------------------------------------------
# a12
# ---------------------------------------------------------------------------
def _composite(raw_dy, raw_st, z, mask_dy, V_dy, min_dy, mask_st, V_st, min_st):
  R, S = z.shape
  dev = dev_of(z)
  rays = torch.empty(R, 11, device=dev)
  samp = torch.empty(5, R, S, device=dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_composite(A(raw_dy), A(raw_st), A(z), A(mask_dy),
                            V_dy, min_dy, A(mask_st), V_st, min_st, R, S, ptr(rays),
                            ptr(samp), stream()))
  return OrderedDict([
      ("rgb", rays[:, 0:3]), ("rgb_static", rays[:, 3:6]), ("rgb_dy", rays[:, 6:9]),
      ("depth", rays[:, 9]), ("alpha_dy", samp[0]), ("weights_dy", samp[1]),
      ("weights_st", samp[2]), ("alpha", samp[3]), ("weights", samp[4]),
      ("mask", rays[:, 10] > 0.5), ("z_vals", z),
  ])


def _composite_vanilla(raw, z, mask, V, min_views):
  R, S = z.shape
  dev = dev_of(z)
  rays = torch.empty(R, 5, device=dev)
  samp = torch.empty(2, R, S, device=dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_composite_vanilla(A(raw), A(z), A(mask), V, min_views,
                                    R, S, ptr(rays), ptr(samp), stream()))
  return OrderedDict([
      ("rgb", rays[:, 0:3]), ("depth", rays[:, 3]), ("weights", samp[0]),
      ("mask", rays[:, 4] > 0.5), ("alpha", samp[1]), ("z_vals", z),
  ])


def raw2outputs(raw_dy, raw_static, z_vals, mask_dy, mask_static, raw_noise_std=0.0):
  """render_ray.py:214-330; mask_* are the per-sample [R,S] validity masks."""
  return _composite(raw_dy, raw_static, z_vals, mask_dy.float(), 1, 0, mask_static.float(), 1, 0)


def raw2outputs_vanilla(raw, z_vals, mask):
  """render_ray.py:134-211."""
  return _composite_vanilla(raw, z_vals, mask.float(), 1, 0)


# ---------------------------------------------------------------------------
# a13
# ---------------------------------------------------------------------------
def resample_depths(z_vals, weights, N_importance, inv_uniform, det=True, u=None):
  """sample_pdf on the interior weights + concat + sort
  (render_ray.py:790-819) -> [R, S+N_importance] ascending depths."""
  R, S = z_vals.shape
  dev = dev_of(z_vals)
  if not det and u is None:
    u = torch.rand(R, N_importance, device=dev)
  if det:
    u = None
  out = torch.empty(R, S + N_importance, device=dev)
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_resample(A(z_vals), A(weights),
                           A(u), R, S, N_importance,
                           int(bool(inv_uniform)), ptr(out), stream()))
  return out


# ---------------------------------------------------------------------------
# a14
# ---------------------------------------------------------------------------
def _flow_sceneflow(weights, pts_seq, src_cameras, uv, coeff, basis, frame_idx, sf_k, n_flow):
  R, S = weights.shape
  dev = dev_of(weights)
  flows = torch.empty(n_flow, R, 2, device=dev)
  exp_sf = torch.empty(R, 3, device=dev) if coeff is not None else None
  T, nb = (basis.shape if basis is not None else (0, 1))
  A = Args()
  with torch.cuda.device(dev):
    check(lib.dyn_flow_sceneflow(
        A(weights), A(pts_seq), A.host(src_cameras), A(uv),
        A(coeff),
        A.host(basis), T, nb, int(frame_idx), int(sf_k),
        int(n_flow), R, S, ptr(flows), ptr(exp_sf) if exp_sf is not None else None, stream()))
  return flows, exp_sf


def compute_optical_flow(outputs_coarse, raw_pts_3d_seq, src_cameras, uv_grid):
  """render_ray.py:333-358 -> [V,R,2]."""
  V = raw_pts_3d_seq.shape[0]
  flows, _ = _flow_sceneflow(outputs_coarse["weights"], raw_pts_3d_seq, src_cameras[:, :V],
                             uv_grid, None, None, 0, 0, V)
  return flows


# ---------------------------------------------------------------------------
# a15 orchestrators
# ---------------------------------------------------------------------------

_HOST_KEYS = ("camera", "src_cameras", "static_src_cameras", "anchor_src_cameras", "depth_range")
MAX_CAMERAS = 16  # target cameras of one multi-camera ray batch (csrc/geometry.cuh: kMaxTargets)


def camera_count(ray_batch):
  """Number K of target cameras of a ray batch: `camera` [K,34].  A multi-camera batch (K > 1, see
  sample_ray.stack_ray_batches) carries `camera_index` [R] int32 naming each ray's row of `camera`."""
  cam = ray_batch["camera"]
  K = cam.shape[0] if cam.dim() == 2 else 1
  if K > 1:
    if K > MAX_CAMERAS:
      raise ValueError("multi-camera ray batch: %d target cameras, at most %d" % (K, MAX_CAMERAS))
    ci = ray_batch.get("camera_index")
    if ci is None or ci.dtype != torch.int32 or ci.shape != ray_batch["ray_o"].shape[:1]:
      raise ValueError("multi-camera ray batch (%d target cameras) needs camera_index: int32 [R]" % K)
  return K


def is_pooled(ray_batch):
  """True for a pooled multi-camera batch (sample_ray.stack_pooled_ray_batches): per-camera view tables
  `src_views` / `static_src_views` over pools of source views."""
  return ray_batch.get("src_views") is not None and ray_batch.get("static_src_views") is not None


def _refuse_multi_camera(ray_batch, what):
  if camera_count(ray_batch) > 1 or is_pooled(ray_batch):
    raise NotImplementedError(
        "%s renders one target camera per time step; multi-camera ray batches (batched target cameras) are "
        "for render_rays_mv / render_image.render_multi_image_nvi" % what)


def _with_host_copies(ray_batch, model, basis_names):
  """One device->host read of the tiny per-frame arrays (cameras, depth range,
  trajectory basis) per render call instead of one per kernel launch."""
  rb = dict(ray_batch)
  for k in _HOST_KEYS:
    v = ray_batch.get(k)
    if torch.is_tensor(v) and v.is_cuda:
      rb[k] = v.detach().float().cpu()
  basis = {}
  for name in basis_names:
    b = getattr(model, name, None)
    basis[name] = b.detach().float().cpu() if torch.is_tensor(b) else b
  return rb, basis


def _render_pass(ray_batch, feat_dy, feat_st, pts, z, s, t, frame_idx, offsets, num_vv, net_dy,
                 net_st, motion, basis, flow_views, sf_k, want_extras=True, want_vanilla_st=False,
                 want_aux=False):
  """One coarse-or-fine evaluation at the reference time
  (render_ray.py:455-597 == :672-782 == :951-1096)."""
  cam, ray_o, ray_d = ray_batch["camera"], ray_batch["ray_o"], ray_batch["ray_d"]
  # multi-camera batch: only the static branch's ray_diff reads the target camera (the dynamic net discards
  # ray_diff, mlp_network.py:236-316), so the dynamic calls keep one camera
  cam_idx = ray_batch.get("camera_index")
  # pooled batch (sample_ray.stack_pooled_ray_batches): the source views are pools and each camera's view slots
  # map into them through the [K, V] tables (both branches: every camera keeps its K rows); the per-slot results
  # are those of the camera's own views
  tbl_dy, tbl_st = ray_batch.get("src_views"), ray_batch.get("static_src_views")
  cam_dy = cam if cam_idx is None or tbl_dy is not None else cam[0:1]
  v_dy = ray_batch["src_cameras"].shape[1] if tbl_dy is None else tbl_dy.shape[1]
  v_st = ray_batch["static_src_cameras"].shape[1] if tbl_st is None else tbl_st.shape[1]
  ci_dy = None if tbl_dy is None else cam_idx
  ref_plucker = compute_ref_plucker_coordinate(ray_o, ray_d)  # [d_hat, o x d_hat]
  ray_dir = ref_plucker[:, :3]  # == F.normalize(ray_d) (render_ray.py:455)
  coeff = motion_coefficients(motion, pts, t)
  seq = displaced_points(pts, coeff, basis, frame_idx, offsets, num_vv)
  fused = _prec() == _lib.PREC_BF16 and USE_FUSED and v_dy <= 16 and v_st <= 16
  if fused:
    # gather + per-view MLP chain + pooling in one tensor-core kernel per branch: the
    # [R,S,V,35] gather output and the per-view activations never reach HBM
    raw_dy, m_dy = net_dynamic_fused(net_dy, pts, seq, ray_dir, cam_dy, ray_batch["src_rgbs"],
                                     ray_batch["src_cameras"], featmaps_channels_last(feat_dy), t, ci_dy, tbl_dy)
    raw_st, m_st = net_static_fused(net_st, pts, ray_o, ray_d, cam, ray_batch["static_src_rgbs"],
                                    ray_batch["static_src_cameras"],
                                    featmaps_channels_last(feat_st), cam_idx, tbl_st)
  else:
    f_dy, _, m_dy = project_gather(pts, seq, cam_dy, ray_batch["src_rgbs"], ray_batch["src_cameras"],
                                   feat_dy, ci_dy, tbl_dy)
    f_st, rd_st, m_st = project_gather(pts, None, cam, ray_batch["static_src_rgbs"],
                                       ray_batch["static_src_cameras"], feat_st, cam_idx, tbl_st)
    raw_dy = net_dynamic_forward(net_dy, pts, f_dy, ray_dir, m_dy, t)
    raw_st = net_static_forward(net_st, pts, ref_plucker,
                                compute_src_plucker_coordinate(pts, ray_batch["static_src_cameras"],
                                                               cam_idx, tbl_st),
                                f_st, rd_st, m_st)
  V_dy, V_st = m_dy.shape[2], m_st.shape[2]
  # a sample counts when MORE THAN ONE view sees it (render_ray.py:524-529)
  out = _composite(raw_dy, raw_st, z, m_dy, V_dy, 1, m_st, V_st, 1)
  out_dy = _composite_vanilla(raw_dy, z, m_dy, V_dy, 1)
  out_st = _composite_vanilla(raw_st, z, m_st, V_st, 1) if want_vanilla_st else None
  if want_extras:
    nflow = seq.shape[0] if flow_views is None else flow_views
    flows, exp_sf = _flow_sceneflow(out["weights"], seq, ray_batch["src_cameras"],
                                    ray_batch["uv_grid"], coeff, basis, frame_idx, sf_k, nflow)
    out["render_flows"] = flows
    out["s_vals"] = s
    out["exp_sf"] = exp_sf
  if want_aux:
    return out, out_dy, out_st, dict(coeff=coeff, raw_st=raw_st, m_st=m_st, ray_dir=ray_dir)
  return out, out_dy, out_st


def render_rays_mv(frame_idx, time_embedding, time_offset, ray_batch, model, projector,
                   coarse_featmaps, fine_featmaps, N_samples, args, inv_uniform=False,
                   N_importance=0, raw_noise_std=0.0, det=False, white_bkgd=False, is_train=True,
                   jitter=None, u=None, precision=None):
  """Coarse + fine rendering for the Nvidia multi-view benchmark
  (render_ray.py:600-867).  Extra keyword-only inputs `jitter` / `u` carry the
  random draws of :119 / :34 when det=False (drawn with torch.rand if None).
  Returns the reference's dict: outputs_coarse_ref, outputs_fine_ref,
  outputs_fine_ref_dy, outputs_fine_anchor(None), outputs_fine_anchor_dy(None).
  `ray_batch` may be a multi-camera batch (sample_ray.stack_ray_batches): the rays of K target cameras
  of one time step, ray r seen from camera[camera_index[r]]; the index values are not checked here
  (render_image.render_multi_image_nvi checks them once per frame).
  With gradients enabled and a fine-stage tensor that requires grad (a parameter of net_fine_dy / net_fine_st /
  motion_mlp_fine, trajectory_basis_fine, fine_featmaps[0] / [2]) the fine pass is differentiable
  (`_render_mv_train`, single-camera batches only); the coarse pass never is, as in the reference."""
  assert N_importance > 0  # render_ray.py:787
  K = camera_count(ray_batch)
  if _fine_stage_wants_grad(model, fine_featmaps):
    if K > 1:
      raise NotImplementedError(
          "render_rays_mv trains on one target camera per call: multi-camera ray batches (batched target cameras) "
          "are rendered by the forward path only; call under torch.no_grad() or freeze the fine stage")
    with precision_scope(precision):
      return _render_mv_train_chunked(frame_idx, time_embedding, time_offset, ray_batch, model, coarse_featmaps,
                                      fine_featmaps, N_samples, args, inv_uniform, N_importance, det, jitter, u)
  with torch.no_grad(), precision_scope(precision):
    t = _scalar(time_embedding[0].float())
    offs = [int(o) for o in time_offset[0]]
    fidx = int(frame_idx[0])
    ret = {"outputs_coarse": None, "outputs_fine": None}
    ray_batch, hb = _with_host_copies(ray_batch, model, ("trajectory_basis", "trajectory_basis_fine"))
    pts, z, _ = sample_along_camera_ray(ray_batch["ray_o"], ray_batch["ray_d"],
                                        ray_batch["depth_range"], N_samples, inv_uniform, det, jitter)
    out_c, _, _ = _render_pass(ray_batch, coarse_featmaps[0], coarse_featmaps[2], pts, z, None, t,
                               fidx, offs, 0, model.net_coarse_dy, model.net_coarse_st,
                               model.motion_mlp, hb["trajectory_basis"], None, 2, want_extras=False)
    ret["outputs_coarse_ref"] = out_c
    zf = resample_depths(z, out_c["weights"], N_importance, inv_uniform, det, u)
    pts_f, s = points_from_depths(ray_batch["ray_o"], ray_batch["ray_d"], zf,
                                  ray_batch["depth_range"])
    out_f, out_f_dy, _ = _render_pass(ray_batch, fine_featmaps[0], fine_featmaps[2], pts_f, zf, s,
                                      t, fidx, offs, 0, model.net_fine_dy, model.net_fine_st,
                                      model.motion_mlp_fine, hb["trajectory_basis_fine"], None, 2)
    ret["outputs_fine_ref"] = out_f
    ret["outputs_fine_ref_dy"] = out_f_dy
    ret["outputs_fine_anchor"] = None
    ret["outputs_fine_anchor_dy"] = None
  return ret


def render_rays_mono(frame_idx, time_embedding, time_offset, ray_batch, model, featmaps, projector,
                     N_samples, args, inv_uniform=False, N_importance=0, raw_noise_std=0.0,
                     det=False, white_bkgd=False, is_train=True, num_vv=2, jitter=None, precision=None):
  """Coarse-only rendering for monocular video (render_ray.py:870-1277), including the
  cross-time branch (:1099-1270) when is_train=True.  With gradients enabled and parameters / feature
  maps that require grad the differentiable fp32 training path runs (`_render_mono_train`); otherwise
  the forward-only kernels (fused tensor-core path in bf16 mode) under no_grad.
  `ray_batch` may be a pooled multi-camera batch (sample_ray.stack_pooled_ray_batches) when is_train=False and no
  gradient is wanted: the rays of K target cameras of one time step, each camera with its own source views from
  shared pools.  Its table and camera_index values are not checked here (render_image.render_multi_image_mono
  checks them once per call)."""
  if not (is_pooled(ray_batch) and not is_train and not _wants_grad(model, featmaps)):
    _refuse_multi_camera(ray_batch, "render_rays_mono (and its training path)")
  if _wants_grad(model, featmaps):
    with precision_scope(precision):
      return _render_mono_train_chunked(frame_idx, time_embedding, time_offset, ray_batch, model, featmaps,
                                        N_samples, args, inv_uniform, det, is_train, num_vv, jitter)
  with torch.no_grad(), precision_scope(precision):
    t = _scalar(time_embedding[0].float())
    ray_batch, hb = _with_host_copies(ray_batch, model, ("trajectory_basis",))
    basis = hb["trajectory_basis"]
    fidx = int(frame_idx[0])
    pts, z, s = sample_along_camera_ray(ray_batch["ray_o"], ray_batch["ray_d"],
                                        ray_batch["depth_range"], N_samples, inv_uniform, det, jitter)
    out, out_dy, out_st, aux = _render_pass(ray_batch, featmaps[0], featmaps[2], pts, z, s, t, fidx,
                                            [int(o) for o in time_offset[0]], num_vv,
                                            model.net_coarse_dy, model.net_coarse_st, model.motion_mlp,
                                            basis, 6, 1, want_vanilla_st=True, want_aux=True)
    ret = {"outputs_coarse": None, "outputs_fine": None, "outputs_coarse_ref": out,
           "outputs_coarse_ref_dy": out_dy, "outputs_coarse_st": out_st}
    if is_train:
      ret.update(_cross_time(ray_batch, featmaps[1], pts, z, aux, fidx, int(frame_idx[1]),
                             _scalar(time_embedding[1].float()), [int(o) for o in time_offset[1]],
                             num_vv, model, basis, args.occ_weights_mode, out, out_dy))
  return ret


def _cross_time(ray_batch, feat_anchor, pts, z, aux, ref_idx, anc_idx, t_anc, anchor_offsets, num_vv,
                model, basis, occ_mode, out_ref, out_ref_dy):
  """Cross-time rendering for temporal consistency (render_ray.py:1099-1270)."""
  coeff = aux["coeff"]
  sf_seq = traj_deltas(coeff, basis, [ref_idx + o for o in (-2, -1, 0, 1, 2, 3)],
                       [ref_idx + o - 1 for o in (-2, -1, 0, 1, 2, 3)])
  pts_anchor = displaced_points(pts, coeff, basis, ref_idx, [anc_idx - ref_idx])[0]  # :1109-1112
  coeff_a = motion_coefficients(model.motion_mlp, pts_anchor, t_anc)                 # :1126-1127
  seq_a = displaced_points(pts_anchor, coeff_a, basis, anc_idx, anchor_offsets, num_vv)  # :1149-1176
  keep = [(i, anc_idx + o - ref_idx) for i, o in enumerate(anchor_offsets)
          if -3 <= anc_idx + o - ref_idx <= 3]
  pts_traj_anchor = seq_a[[i for i, _ in keep]]
  pts_traj_ref = displaced_points(pts, coeff, basis, ref_idx, [ro for _, ro in keep])
  cam = ray_batch["camera"]
  V_a = ray_batch["anchor_src_cameras"].shape[1]
  if _prec() == _lib.PREC_BF16 and USE_FUSED and V_a <= 16:
    raw_a, m_a = net_dynamic_fused(model.net_coarse_dy, pts_anchor, seq_a, aux["ray_dir"], cam,
                                   ray_batch["anchor_src_rgbs"], ray_batch["anchor_src_cameras"],
                                   featmaps_channels_last(feat_anchor), t_anc)
  else:
    f_a, _, m_a = project_gather(pts, seq_a, cam, ray_batch["anchor_src_rgbs"],
                                 ray_batch["anchor_src_cameras"], feat_anchor)
    raw_a = net_dynamic_forward(model.net_coarse_dy, pts_anchor, f_a, aux["ray_dir"], m_a, t_anc)
  m_st = aux["m_st"]
  # anchor samples count when ANY view sees them (render_ray.py:1198-1200)
  out_a = _composite(raw_a, aux["raw_st"], z, m_a, V_a, 0, m_st, m_st.shape[2], 1)
  out_a_dy = _composite_vanilla(raw_a, z, m_a, V_a, 0)
  if occ_mode == 0:
    key = "weights_dy" if abs(ref_idx - anc_idx) > 1 else "weights"
  elif occ_mode == 1:
    key = "weights_dy"
  elif occ_mode == 2:
    key = "weights"
  else:
    raise NotImplementedError
  out_a["occ_weights"], out_a["occ_weight_map"] = occlusion_weights(out_ref[key], out_a[key])
  out_a["pts_traj_ref"] = pts_traj_ref
  out_a["pts_traj_anchor"] = pts_traj_anchor
  out_a["sf_seq"] = sf_seq
  out_a_dy["occ_weights"], out_a_dy["occ_weight_map"] = occlusion_weights(out_ref_dy["weights"],
                                                                         out_a_dy["weights"])
  return {"outputs_coarse_anchor": out_a, "outputs_coarse_anchor_dy": out_a_dy}


# ---------------------------------------------------------------------------
# f2: differentiable render_rays_mono (training step)
# ---------------------------------------------------------------------------
# (point, view) rows one training call of a network may hold (csrc/nets_f32.cu: net_rows_per_chunk; the training
# forward keeps every activation of ONE internal chunk); larger ray batches are rendered in slices
TRAIN_ROWS_LIMIT = 4194304
_RAY_AXIS1 = ("render_flows", "pts_traj_ref", "pts_traj_anchor", "sf_seq")  # [n, R, ...]; every other key is [R, ...]


def _render_mono_train_chunked(frame_idx, time_embedding, time_offset, ray_batch, model, featmaps, N_samples, args,
                               inv_uniform, det, is_train, num_vv, jitter):
  """Slices the rays so that no network call exceeds TRAIN_ROWS_LIMIT rows and concatenates the per-slice output
  dicts along their ray axis (autograd sees one graph; gradients accumulate over the slices)."""
  R = ray_batch["ray_o"].shape[0]
  vmax = max(ray_batch[k].shape[1] for k in ("src_cameras", "static_src_cameras", "anchor_src_cameras")
             if k in ray_batch and (is_train or k != "anchor_src_cameras"))
  per = max(1, TRAIN_ROWS_LIMIT // (N_samples * vmax))
  if R <= per:
    return _render_mono_train(frame_idx, time_embedding, time_offset, ray_batch, model, featmaps, N_samples, args,
                              inv_uniform, det, is_train, num_vv, jitter)
  parts = []
  for lo in range(0, R, per):
    hi = min(R, lo + per)
    rb = dict(ray_batch)
    for k in ("ray_o", "ray_d", "uv_grid"):
      rb[k] = ray_batch[k][lo:hi]
    parts.append(_render_mono_train(frame_idx, time_embedding, time_offset, rb, model, featmaps, N_samples, args,
                                    inv_uniform, det, is_train, num_vv,
                                    None if jitter is None else jitter[lo:hi]))
  return _cat_slices(parts)


def _cat_slices(parts):
  """Per-slice output dicts -> one dict, every tensor concatenated along its ray axis."""
  ret = {}
  for name, first in parts[0].items():
    if first is None:
      ret[name] = None
      continue
    ret[name] = OrderedDict((k, torch.cat([p[name][k] for p in parts], 1 if k in _RAY_AXIS1 else 0))
                            for k in first)
  return ret


def _keep_mask(S, dev):
  """[1,S,1]: 0 on the last round(0.1 S) samples, whose motion coefficients the reference zeroes (:471-472).  When
  that count is 0 the reference's slice `[:, -0:]` is the whole axis, so every sample is zeroed (as the forward kernel,
  csrc/nets_f32.cu, does)."""
  keep = torch.ones(1, S, 1, device=dev)
  n_last = int(round(S * 0.1))
  if n_last <= 0:
    n_last = S
  keep[:, S - n_last:] = 0.0
  return keep


def _basis_rows(basis, pairs, dev):
  """D [n,nb] on `dev`, D[i] = basis[a_i] - basis[b_i]; a pair (None, None) is a zero row (these come last).  Row
  indices wrap like the reference's (-1 = the last frame).  The model's basis tensor itself is indexed, so that a
  basis that requires grad (trajectory_basis of DynibarMono, trajectory_basis_fine of DynibarFF) gets the gradient
  of every row built from it.  Rows are selected with integer indices (views, no index tensor to copy to the
  device), so building D never waits for the stream."""
  real = [(a, b) for a, b in pairs if a is not None]
  assert all(a is None for a, _ in pairs[len(real):]), pairs
  bf = basis.to(device=dev, dtype=torch.float32)
  zeros = bf.new_zeros(len(pairs) - len(real), bf.shape[1])
  if not real:
    return zeros
  D = torch.stack([bf[a] for a, _ in real]) - torch.stack([bf[b] for _, b in real])
  return torch.cat([D, zeros]) if zeros.shape[0] else D


# ---------------------------------------------------------------------------
# f2: differentiable fine stage of render_rays_mv (training step of DynibarFF)
# ---------------------------------------------------------------------------
def _render_mv_train_chunked(frame_idx, time_embedding, time_offset, ray_batch, model, coarse_featmaps, fine_featmaps,
                             N_samples, args, inv_uniform, N_importance, det, jitter, u):
  """Slices the rays so that no fine-stage network call exceeds TRAIN_ROWS_LIMIT rows (fine S = N_samples +
  N_importance samples, max(V_dy, V_st) views) and concatenates the per-slice output dicts along their ray axis."""
  R = ray_batch["ray_o"].shape[0]
  vmax = max(ray_batch["src_cameras"].shape[1], ray_batch["static_src_cameras"].shape[1])
  per = max(1, TRAIN_ROWS_LIMIT // ((N_samples + N_importance) * vmax))
  call = lambda rb, jit, uu: _render_mv_train(frame_idx, time_embedding, time_offset, rb, model, coarse_featmaps,
                                              fine_featmaps, N_samples, args, inv_uniform, N_importance, det, jit, uu)
  if R <= per:
    return call(ray_batch, jitter, u)
  parts = []
  for lo in range(0, R, per):
    hi = min(R, lo + per)
    rb = dict(ray_batch)
    for k in ("ray_o", "ray_d", "uv_grid"):
      rb[k] = ray_batch[k][lo:hi]
    parts.append(call(rb, None if jitter is None else jitter[lo:hi], None if u is None else u[lo:hi]))
  return _cat_slices(parts)


def _render_mv_train(frame_idx, time_embedding, time_offset, ray_batch, model, coarse_featmaps, fine_featmaps,
                     N_samples, args, inv_uniform, N_importance, det, jitter, u):
  """render_rays_mv (render_ray.py:600-867) with a differentiable fine pass (fine_render_rays, :407-597).  The coarse
  pass, the importance resampling and the fine points run under no_grad with the forward path's kernels, so
  outputs_coarse_ref and the fine z_vals are those of the forward path (the reference detaches the coarse weights,
  :789-791).  Every fine stage is a `torch.autograd.Function` (dynibar_b200/autograd.py); gradients reach
  net_fine_dy / net_fine_st / motion_mlp_fine, fine_featmaps[0] / [2] and, when it requires grad,
  trajectory_basis_fine.  render_flows covers every dynamic view and exp_sf is differentiable (:585-595)."""
  from dynibar_b200 import autograd as ag
  t = _scalar(time_embedding[0].float())
  offs = [int(o) for o in time_offset[0]]
  fidx = int(frame_idx[0])
  rb, hb = _with_host_copies(ray_batch, model, ("trajectory_basis", "trajectory_basis_fine"))
  with torch.no_grad():
    pts, z, _ = sample_along_camera_ray(rb["ray_o"], rb["ray_d"], rb["depth_range"], N_samples, inv_uniform, det,
                                        jitter)
    out_c, _, _ = _render_pass(rb, coarse_featmaps[0], coarse_featmaps[2], pts, z, None, t, fidx, offs, 0,
                               model.net_coarse_dy, model.net_coarse_st, model.motion_mlp, hb["trajectory_basis"],
                               None, 2, want_extras=False)
    zf = resample_depths(z, out_c["weights"], N_importance, inv_uniform, det, u)
    pts_f, s = points_from_depths(rb["ray_o"], rb["ray_d"], zf, rb["depth_range"])
    ref_plucker = compute_ref_plucker_coordinate(rb["ray_o"], rb["ray_d"])
    src_plucker = compute_src_plucker_coordinate(pts_f, rb["static_src_cameras"])
  ray_dir = ref_plucker[:, :3]
  dev = dev_of(pts_f)
  R, S = pts_f.shape[:2]
  basis = model.trajectory_basis_fine
  xyzt = torch.cat([pts_f, torch.full((R, S, 1), t, device=dev)], dim=-1)
  coeff = ag.motion_mlp(model.motion_mlp_fine, xyzt) * _keep_mask(S, dev)      # :459-472
  seq = ag.traj_combine(coeff, _basis_rows(basis, [(fidx + o, fidx) for o in offs], dev), pts_f)  # :479-497
  cam = rb["camera"]
  f_dy, _, m_dy = ag.project_gather(pts_f, seq, cam, rb["src_rgbs"], rb["src_cameras"], fine_featmaps[0])
  f_st, rd_st, m_st = ag.project_gather(pts_f, None, cam, rb["static_src_rgbs"], rb["static_src_cameras"],
                                        fine_featmaps[2])
  raw_dy = ag.net_dynamic(model.net_fine_dy, pts_f, f_dy, ray_dir, m_dy, t)
  raw_st = ag.net_static(model.net_fine_st, pts_f, ref_plucker, src_plucker, f_st, rd_st, m_st)
  out = ag.composite(raw_dy, raw_st, zf, m_dy, m_st, 1, 1)
  out_dy = ag.composite_vanilla(raw_dy, zf, m_dy, 1)
  out["render_flows"] = ag.optical_flow(out["weights"], seq, rb["src_cameras"], rb["uv_grid"])
  out["s_vals"] = s
  sf = ag.traj_combine(coeff, _basis_rows(basis, [(fidx + 2, fidx), (fidx - 2, fidx)], dev))
  out["exp_sf"] = ag.expected_scene_flow(out["weights"], sf)
  return {"outputs_coarse": None, "outputs_fine": None, "outputs_coarse_ref": out_c, "outputs_fine_ref": out,
          "outputs_fine_ref_dy": out_dy, "outputs_fine_anchor": None, "outputs_fine_anchor_dy": None}


def _render_mono_train(frame_idx, time_embedding, time_offset, ray_batch, model, featmaps, N_samples, args,
                       inv_uniform, det, is_train, num_vv, jitter):
  """render_rays_mono (render_ray.py:870-1277) with autograd: the same sequence as the reference, every stage a
  `torch.autograd.Function` over the forward/backward kernels (dynibar_b200/autograd.py).  Gradients reach
  the parameters of motion_mlp / net_coarse_dy / net_coarse_st, the feature maps and, when it requires grad,
  trajectory_basis (through every displaced point: seq, sf_seq, pts_anchor, seq_a, pts_traj_ref).  torch itself only
  concatenates the time column, zeroes the last samples' coefficients, slices and detaches.  Precision (the
  library-wide setting / `precision=`): "bf16" runs the products of the three networks, forward and backward, on
  tensor cores (bf16 operands, fp32 accumulation, fp32 master weights and gradients); "fp32" = SIMT products."""
  from dynibar_b200 import autograd as ag
  t = _scalar(time_embedding[0].float())
  rb, hb = _with_host_copies(ray_batch, model, ("trajectory_basis",))
  basis = hb["trajectory_basis"]  # host [T, nb] for the (detached) exp_sf kernel
  fidx = int(frame_idx[0])
  ref_offsets = [int(o) for o in time_offset[0]]
  with torch.no_grad():
    pts, z, s = sample_along_camera_ray(rb["ray_o"], rb["ray_d"], rb["depth_range"], N_samples, inv_uniform, det,
                                        jitter)
    ref_plucker = compute_ref_plucker_coordinate(rb["ray_o"], rb["ray_d"])
    src_plucker = compute_src_plucker_coordinate(pts, rb["static_src_cameras"])
  ray_dir = ref_plucker[:, :3]
  dev = dev_of(pts)
  R, S = pts.shape[:2]
  keep = _keep_mask(S, dev)

  def rows(pairs):
    return _basis_rows(model.trajectory_basis, pairs, dev)

  def coeffs(p, tt):  # model.motion_mlp(cat[p, t]) with the last samples zeroed (:957-958, :1126-1127)
    xyzt = torch.cat([p, torch.full((R, S, 1), tt, device=dev)], dim=-1)
    return ag.motion_mlp(model.motion_mlp, xyzt) * keep

  coeff = coeffs(pts, t)
  seq = ag.traj_combine(coeff, rows([(fidx + o, fidx) for o in ref_offsets] + [(None, None)] * num_vv), pts)
  cam = rb["camera"]
  f_dy, _, m_dy = ag.project_gather(pts, seq, cam, rb["src_rgbs"], rb["src_cameras"], featmaps[0])
  f_st, rd_st, m_st = ag.project_gather(pts, None, cam, rb["static_src_rgbs"], rb["static_src_cameras"],
                                        featmaps[2])
  raw_dy = ag.net_dynamic(model.net_coarse_dy, pts, f_dy, ray_dir, m_dy, t)
  raw_st = ag.net_static(model.net_coarse_st, pts, ref_plucker, src_plucker, f_st, rd_st, m_st)
  out = ag.composite(raw_dy, raw_st, z, m_dy, m_st, 1, 1)
  out_st = ag.composite_vanilla(raw_st, z, m_st, 1)
  out_dy = ag.composite_vanilla(raw_dy, z, m_dy, 1)
  out["render_flows"] = ag.optical_flow(out["weights"], seq[:6], rb["src_cameras"][:, :6], rb["uv_grid"])
  out["s_vals"] = s
  with torch.no_grad():  # :1086-1096, detached in the reference
    _, out["exp_sf"] = _flow_sceneflow(out["weights"], seq, rb["src_cameras"], rb["uv_grid"], coeff, basis, fidx,
                                       1, 1)
  ret = {"outputs_coarse": None, "outputs_fine": None, "outputs_coarse_ref": out,
         "outputs_coarse_ref_dy": out_dy, "outputs_coarse_st": out_st}
  if not is_train:
    return ret
  # ---- cross-time rendering for temporal consistency (:1099-1270)
  anc = int(frame_idx[1])
  t_anc = _scalar(time_embedding[1].float())
  anchor_offsets = [int(o) for o in time_offset[1]]
  sf_seq = ag.traj_combine(coeff, rows([(fidx + o, fidx + o - 1) for o in (-2, -1, 0, 1, 2, 3)]))
  pts_anchor = ag.traj_combine(coeff, rows([(anc, fidx)]), pts)[0]
  coeff_a = coeffs(pts_anchor, t_anc)
  seq_a = ag.traj_combine(coeff_a, rows([(anc + o, anc) for o in anchor_offsets] + [(None, None)] * num_vv),
                          pts_anchor)
  kept = [(i, anc + o - fidx) for i, o in enumerate(anchor_offsets) if -3 <= anc + o - fidx <= 3]
  pts_traj_anchor = seq_a[[i for i, _ in kept]]
  pts_traj_ref = ag.traj_combine(coeff, rows([(fidx + ro, fidx) for _, ro in kept]), pts)
  f_a, _, m_a = ag.project_gather(pts, seq_a, cam, rb["anchor_src_rgbs"], rb["anchor_src_cameras"], featmaps[1])
  raw_a = ag.net_dynamic(model.net_coarse_dy, pts_anchor, f_a, ray_dir, m_a, t_anc)
  # anchor samples count when ANY view sees them (render_ray.py:1198-1200)
  out_a = ag.composite(raw_a, raw_st, z, m_a, m_st, 0, 1)
  out_a_dy = ag.composite_vanilla(raw_a, z, m_a, 0)
  occ_mode = args.occ_weights_mode
  if occ_mode == 0:
    key = "weights_dy" if abs(fidx - anc) > 1 else "weights"
  elif occ_mode == 1:
    key = "weights_dy"
  elif occ_mode == 2:
    key = "weights"
  else:
    raise NotImplementedError
  with torch.no_grad():  # detached in the reference (:1222, :1254)
    out_a["occ_weights"], out_a["occ_weight_map"] = occlusion_weights(out[key], out_a[key])
    out_a_dy["occ_weights"], out_a_dy["occ_weight_map"] = occlusion_weights(out_dy["weights"], out_a_dy["weights"])
  out_a["pts_traj_ref"] = pts_traj_ref
  out_a["pts_traj_anchor"] = pts_traj_anchor
  out_a["sf_seq"] = sf_seq
  ret["outputs_coarse_anchor"] = out_a
  ret["outputs_coarse_anchor_dy"] = out_a_dy
  return ret
