"""`Projector`: drop-in for ibrnet/projection.py:7-176 on top of the CUDA
projection + bilinear-gather kernel (csrc/geometry.cu).
"""

import torch

from dynibar_b200 import _lib
from dynibar_b200._lib import lib, ptr, f32c, check, stream, dev_of, Args


class Projector(object):
  """Same constructor and public methods as the reference Projector."""

  def __init__(self, device):
    self.device = torch.device(device) if not isinstance(device, torch.device) else device

  # -- small host-side predicates kept for API parity (projection.py:13-30) --
  def inbound(self, pixel_locations, h, w):
    return ((pixel_locations[..., 0] <= w - 1.0) & (pixel_locations[..., 0] >= 0)
            & (pixel_locations[..., 1] <= h - 1.0) & (pixel_locations[..., 1] >= 0))

  def normalize(self, pixel_locations, h, w):
    resize = torch.tensor([w - 1.0, h - 1.0], device=pixel_locations.device)[None, None, :]
    return 2 * pixel_locations / resize - 1.0

  def compute_projections(self, xyz, train_cameras):
    """xyz [V,...,3], train_cameras [V,34] -> pixel_locations [V,...,2],
    mask [V,...] bool (projection.py:32-59)."""
    shape = xyz.shape[:-1]
    V = shape[0]
    x = f32c(xyz).reshape(V, -1, 3)
    N = x.shape[1]
    pix = torch.empty(V, N, 2, device=x.device)
    front = torch.empty(V, N, dtype=torch.uint8, device=x.device)
    A = Args()
    with torch.cuda.device(x.device):
      check(lib.dyn_compute_projections(ptr(x), A.host(train_cameras), V, N, ptr(pix),
                                        ptr(front, torch.uint8), stream()))
    return pix.reshape(shape + (2,)), front.bool().reshape(shape)

  def compute_angle(self, xyz_st, xyz, query_camera, train_cameras):
    """projection.py:61-101.  xyz_st [V or 1, ..., 3] (the reference passes the static point
    expanded over the views), xyz [V,...,3], query_camera [34], train_cameras [V,34]
    -> ray_diff [V,...,4] = [normalize(a - b), a . b]."""
    shape = xyz.shape[:-1]
    V = shape[0]
    x = f32c(xyz).reshape(V, -1, 3)
    N = x.shape[1]
    st_views = xyz_st.shape[0]
    assert st_views in (1, V), "xyz_st must have 1 or n_views leading entries"
    xs = f32c(xyz_st).reshape(st_views, -1, 3)
    assert xs.shape[1] == N
    out = torch.empty(V, N, 4, device=x.device)
    A = Args()
    with torch.cuda.device(x.device):
      check(lib.dyn_compute_angle(ptr(xs), st_views, ptr(x), A.host(query_camera.reshape(-1)),
                                  A.host(train_cameras), V, N, ptr(out), stream()))
    return out.reshape(shape + (4,))

  def compute_with_motions(self, xyz_st, xyz, query_camera, train_imgs, train_cameras, featmaps):
    """projection.py:103-176.

    xyz_st [R,S,3]; xyz [V,R,S,3]; query_camera [1,34]; train_imgs [1,V,H,W,3];
    train_cameras [1,V,34]; featmaps [V,C,h,w].
    Returns rgb_feat [R,S,V,3+C], ray_diff [R,S,V,4], mask [R,S,V,1] (float).
    """
    assert (train_imgs.shape[0] == 1 and train_cameras.shape[0] == 1
            and query_camera.shape[0] == 1), "only support batch_size=1 for now"
    return project_gather(xyz_st, xyz, query_camera, train_imgs, train_cameras, featmaps)


def project_gather(xyz_st, xyz, query_camera, train_imgs, train_cameras, featmaps, camera_index=None,
                   view_tbl=None):
  """`xyz` may be None: every view then uses xyz_st (static branch).  With `camera_index` ([R] int32 on the
  device) query_camera is [K,34] and ray r's view-direction term (ray_diff) uses camera camera_index[r]; the
  kernel trusts the values to lie in [0, K).  With `view_tbl` ([K,V] int32, host) train_imgs / train_cameras /
  featmaps hold a pool of source views and slot v of ray r reads pool entry view_tbl[camera_index[r], v]; the
  outputs have V slots."""
  R, S = xyz_st.shape[:2]
  pool = train_cameras.shape[1]
  V = pool if view_tbl is None else view_tbl.shape[1]
  _, _, H, W, _ = train_imgs.shape
  Vf, Cc, h, w = featmaps.shape
  assert Vf == pool and (xyz is None or xyz.shape[0] == V)
  dev = dev_of(xyz_st)
  rgb_feat = torch.empty(R, S, V, 3 + Cc, device=dev)
  ray_diff = torch.empty(R, S, V, 4, device=dev)
  mask = torch.empty(R, S, V, 1, device=dev)
  fm = f32c(featmaps)
  ws = _lib.workspace.get(fm.numel() * 4, dev, slot=1)
  A = Args()
  with torch.cuda.device(dev):
    if view_tbl is not None:
      K = query_camera.shape[0]
      assert view_tbl.shape[0] == K, "one table row per target camera"
      check(lib.dyn_project_gather_tbl(
          A(xyz_st), A(xyz), A.host(query_camera), K, A(camera_index, torch.int32) if camera_index is not None
          else None, A.host_i32(view_tbl), pool, A(train_imgs), A.host(train_cameras), ptr(fm), V, R, S, H, W,
          Cc, h, w, ws.data_ptr(), ptr(rgb_feat), ptr(ray_diff), ptr(mask), stream()))
    elif camera_index is None:
      check(lib.dyn_project_gather(
          A(xyz_st), A(xyz),
          A.host(query_camera), A(train_imgs), A.host(train_cameras), ptr(fm),
          V, R, S, H, W, Cc, h, w, ws.data_ptr(), ptr(rgb_feat), ptr(ray_diff), ptr(mask),
          stream()))
    else:
      assert camera_index.shape == (R,)
      check(lib.dyn_project_gather_mc(
          A(xyz_st), A(xyz), A.host(query_camera), query_camera.shape[0], A(camera_index, torch.int32),
          A(train_imgs), A.host(train_cameras), ptr(fm), V, R, S, H, W, Cc, h, w, ws.data_ptr(),
          ptr(rgb_feat), ptr(ray_diff), ptr(mask), stream()))
  return rgb_feat, ray_diff, mask
