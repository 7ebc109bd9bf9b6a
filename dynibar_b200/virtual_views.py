"""Virtual source views of a monocular scene (the reference's render_source_vv.py) on the GPU.

Training and rendering a monocular scene with num_vv > 0 read, for every frame, views of that frame splatted into
nearby virtual cameras (dense/source_virtual_views_WxH/%05d/%02d.png and dense/source_vv_poses.npy).  This module
makes them with the library's own kernels (csrc/splat.cu) in place of the external `splatting` extension and kornia:

  splatting_function(...)      drop-in for `from splatting import splatting_function` ('softmax' only)
  render_forward_splat(...)    render_source_vv.py:15, same signature and outputs
  sobel_fg_alpha(...)          render_source_vv.py:118
  render_wander_path(...)      render_source_vv.py:68 (host, float64)
  virtual_view_poses(...)      the two wander rings per frame and their subsampling (render_source_vv.py:195-251)
  render_virtual_views(...)    one frame's views as uint8 [V, H, W, 3] on the device, one chain of launches

The splat is deterministic: the same inputs give the same bits (no float atomics).  tools/make_virtual_views.py
writes the files of a scene.
"""

import numpy as np
import torch

from . import _lib

SPLAT_EPS = 1e-7  # splatting_function's eps: out = sum / (sum_e + eps); a constant of csrc/splat.cu
NUM_SAMPLES = 4   # views taken from each of the two wander rings: 8 virtual views per frame
FINAL_H = 288     # height of the written views (render_source_vv.py:131)


def _cams(k_src, r_cam, t_cam, k_dst):
  """[B, 30] fp32 = K_src^-1 | R | t | K_dst per item; K^-1 by torch.inverse in fp32 on the host, as the reference."""
  f = lambda a: torch.as_tensor(a).detach().cpu().float()
  k_src, r_cam, t_cam, k_dst = f(k_src), f(r_cam), f(t_cam), f(k_dst)
  B = r_cam.shape[0]
  return torch.cat([k_src.inverse().reshape(B, 9), r_cam.reshape(B, 9), t_cam.reshape(B, 3), k_dst.reshape(B, 9)], 1)


def splatting_function(splatting_type, frame, flow, importance_metric=None, eps=SPLAT_EPS):
  """Softmax forward splatting of frame [B, C, H, W] along flow [B, 2, H, W] with metric [B, 1, H, W]:
  out = sum(frame e w) / (sum(e w) + eps), e = exp(metric), w the bilinear weight of each of a source's four target
  pixels (a corner outside the image is dropped).  Forward only; C <= 8."""
  if splatting_type != "softmax":
    raise NotImplementedError("splatting_function: only 'softmax' is implemented (got %r)" % (splatting_type,))
  if eps != SPLAT_EPS:
    raise NotImplementedError("splatting_function: eps is fixed at %g" % SPLAT_EPS)
  if importance_metric is None:
    raise ValueError("splatting_function('softmax') needs importance_metric")
  dev = _lib.dev_of(frame)
  B, C, H, W = frame.shape
  if tuple(flow.shape) != (B, 2, H, W) or tuple(importance_metric.shape) != (B, 1, H, W):
    raise ValueError("splatting_function: frame %s, flow %s, metric %s" % (tuple(frame.shape), tuple(flow.shape),
                                                                            tuple(importance_metric.shape)))
  a = _lib.Args()
  out = torch.empty(B, C, H, W, device=dev)
  with torch.cuda.device(dev):
    nbytes = _lib.lib.dyn_splat_workspace_bytes(B, H, W)
    ws = _lib.workspace.get(nbytes, dev, slot="splat")
    _lib.check(_lib.lib.dyn_splat_softmax(a(frame), a(flow), a(importance_metric), B, C, H, W, _lib.ptr(out),
                                          ws.data_ptr(), ws.numel(), _lib.stream()))
  return out


def render_forward_splat(src_imgs, src_depths, r_cam, t_cam, k_src, k_dst):
  """Point-cloud rendering of RGB-D images src_imgs [B, H, W, C], src_depths [B, H, W] (CUDA) into cameras
  r_cam [B, 3, 3], t_cam [B, 3], k_src / k_dst [B, 3, 3] (host or device).  Returns (warped image [B, C, H, W],
  warped inverse depth [B, 1, H, W]).  C <= 7."""
  dev = _lib.dev_of(src_imgs)
  _lib.dev_of(src_depths)
  B, H, W, C = src_imgs.shape
  if tuple(src_depths.shape) != (B, H, W):
    raise ValueError("render_forward_splat: images %s, depths %s" % (tuple(src_imgs.shape), tuple(src_depths.shape)))
  cams = _cams(k_src, r_cam, t_cam, k_dst)
  if cams.shape[0] != B:
    raise ValueError("render_forward_splat: %d cameras for %d images" % (cams.shape[0], B))
  a = _lib.Args()
  out = torch.empty(B, C + 1, H, W, device=dev)
  with torch.cuda.device(dev):
    nbytes = _lib.lib.dyn_splat_workspace_bytes(B, H, W)
    ws = _lib.workspace.get(nbytes, dev, slot="splat")
    _lib.check(_lib.lib.dyn_forward_splat(a(src_imgs), a(src_depths), a(cams.to(dev)), B, C, H, W, _lib.ptr(out),
                                          ws.data_ptr(), ws.numel(), _lib.stream()))
  return out[:, :C], out[:, C:C + 1]


def sobel_fg_alpha(disp, mode="sobel", beta=10.0):
  """Depth-boundary alpha exp(-beta |sobel(disp)|) of disp [B, C, H, W] (unnormalised 3x3 Sobel, border
  replicated, as kornia.filters.spatial_gradient)."""
  if mode != "sobel":
    raise NotImplementedError("sobel_fg_alpha: only mode 'sobel' is implemented (got %r)" % (mode,))
  dev = _lib.dev_of(disp)
  B, C, H, W = disp.shape
  a = _lib.Args()
  out = torch.empty(B, C, H, W, device=dev)
  with torch.cuda.device(dev):
    _lib.check(_lib.lib.dyn_sobel_alpha(a(disp), B * C, H, W, float(beta), _lib.ptr(out), _lib.stream()))
  return out


def render_wander_path(c2w, hwf, bd_scale, max_disp_=50, xyz=(1, 0, 1)):
  """60 poses on a ring around c2w [3, 4+] displaced along x / y / z by xyz * max_disp_ * bd_scale / focal
  (hwf [3, 1] = h, w, focal), twice over, and the ring's length 60."""
  num_frames = 60
  max_trans = max_disp_ * bd_scale / hwf[2][0]
  ref_pose = np.concatenate([c2w[:3, :4], np.array([0.0, 0.0, 0.0, 1.0])[np.newaxis, :]], axis=0)
  output_poses = []
  for i in range(num_frames):
    ang = 2.0 * np.pi * float(i) / float(num_frames)
    trans = np.array([max_trans * np.cos(ang) * xyz[0], max_trans * np.sin(ang) * xyz[1],
                      max_trans * np.cos(ang) * xyz[2]])
    i_pose = np.concatenate([np.concatenate([np.eye(3), trans[:, np.newaxis]], axis=1),
                             np.array([0.0, 0.0, 0.0, 1.0])[np.newaxis, :]], axis=0)
    render_pose = np.dot(ref_pose, np.linalg.inv(i_pose))
    output_poses.append(np.concatenate([render_pose[:3, :], hwf], 1))
  return np.array(output_poses + output_poses), num_frames


def scaled_intrinsics(K_npz, src_hw, final_hw):
  """K [3, 3] of a dynamic-video-depth frame (stored transposed as K[0, 0, 0]) scaled from src_hw to final_hw, in
  the file's dtype (render_source_vv.py:191-193)."""
  K = np.array(K_npz[0, 0, 0].transpose())
  K[0, :] *= final_hw[1] / src_hw[1]
  K[1, :] *= final_hw[0] / src_hw[0]
  return K


def virtual_view_poses(cam_c2w, depths, K, final_hw):
  """The 2 * NUM_SAMPLES virtual cameras of every frame: cam_c2w [N, 4, 4] camera-to-world (x right, y down,
  z forward), depths the N frames' depth maps, K [3, 3] scaled to final_hw (the scene's focal).  The rings'
  radius follows 0.75 x the smallest 5th depth percentile over the frames.  Returns (source_vv_poses [8, 3, 4, N]
  float32 in the [-y, x, z] axes, as source_vv_poses.npy stores it; the cameras [N, 8, 3, 4] float64 as
  camera-to-world in the input's axes)."""
  bd_scale = np.stack([np.percentile(d, 5) for d in depths], 0).min() * 0.75
  hwf = np.array([final_hw[0], final_hw[1], (K[0, 0] + K[1, 1]) / 2.0]).reshape([3, 1])
  poses = np.asarray(cam_c2w)[:, :3, :4].transpose([1, 2, 0])
  # [x, -y, -z] -> [-y, x, z], rounded to fp32 as the reference does
  poses = np.concatenate([poses[:, 1:2, :], poses[:, 0:1, :], -poses[:, 2:3, :], poses[:, 3:4, :]], 1)
  poses = np.moveaxis(poses, -1, 0).astype(np.float32)
  out = np.zeros((poses.shape[0], NUM_SAMPLES * 2, 3, 4))
  for ii in range(poses.shape[0]):
    ring0, n0 = render_wander_path(poses[ii], hwf, bd_scale, 56 * 1.5, xyz=[0.0, 1.0, 1.0])
    ring1, n1 = render_wander_path(poses[ii], hwf, bd_scale, 48 * 1.5, xyz=[0.5, 1.0, 0.0])
    out[ii, :NUM_SAMPLES] = ring0[5:-1:n0 // NUM_SAMPLES][:NUM_SAMPLES, :3, :4]
    out[ii, NUM_SAMPLES:] = ring1[15:-1:n1 // NUM_SAMPLES][:NUM_SAMPLES, :3, :4]
  c2w = np.concatenate([out[..., 1:2], out[..., 0:1], -out[..., 2:3], out[..., 3:4]], -1)
  return np.moveaxis(out, 0, -1).astype(np.float32), c2w


def render_virtual_views(img, disp, K, ref2w, tgt_c2w):
  """One frame's virtual source views.  img [H, W, 3] in [0, 1] and disp [H, W] (CUDA, at the output size),
  K [3, 3] at that size, ref2w [4, 4] the frame's camera-to-world, tgt_c2w [V, 3, 4] the virtual cameras (host).
  Returns uint8 [V, H, W, 3] on img's device: the frame's rgb splatted into each camera, black where the splatted
  depth-boundary alpha is <= 0.5 (eroded by one pixel)."""
  dev = _lib.dev_of(img)
  _lib.dev_of(disp)
  H, W = disp.shape
  if tuple(img.shape) != (H, W, 3):
    raise ValueError("render_virtual_views: img %s, disp %s" % (tuple(img.shape), tuple(disp.shape)))
  tgt_c2w = np.asarray(tgt_c2w, dtype=np.float64)
  V = tgt_c2w.shape[0]
  R, t = [], []
  for k in range(V):
    tgt2w = np.eye(4)
    tgt2w[:3, :4] = tgt_c2w[k]
    T = np.dot(np.linalg.inv(tgt2w), np.asarray(ref2w))  # float64, then fp32 (render_source_vv.py:303-306)
    R.append(torch.from_numpy(T[:3, :3]).float())
    t.append(torch.from_numpy(T[:3, 3]).float())
  k32 = torch.from_numpy(np.array(K)).float()[None].expand(V, 3, 3)
  cams = _cams(k32, torch.stack(R), torch.stack(t), k32)
  a = _lib.Args()
  out = torch.empty(V, H, W, 3, dtype=torch.uint8, device=dev)
  with torch.cuda.device(dev):
    nbytes = _lib.lib.dyn_virtual_views_workspace_bytes(V, H, W)
    ws = _lib.workspace.get(nbytes, dev, slot="splat")
    _lib.check(_lib.lib.dyn_virtual_views(a(img), a(disp), a(cams.to(dev)), V, H, W, _lib.ptr(out, torch.uint8),
                                          ws.data_ptr(), ws.numel(), _lib.stream()))
  return out
