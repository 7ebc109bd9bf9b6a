"""Host-side planning of a monocular bullet-time sweep (render_monocular_bt.py): the wander path of target
cameras around one time step or the stabilised path of the whole video, each camera's source views, and the grouping
of the sweep into batched calls of render_image.render_multi_image_mono.

numpy (and cv2's Gaussian filter for the stabilised path), like the reference's data loader: this is per-sweep
set-up, not the hot path.
"""

import numpy as np

MAX_CAMERAS = 16  # target cameras of one batched call (csrc/geometry.cuh: kMaxTargets)
MAX_POOL = 32     # source views of one pool (csrc/common.cuh: kMaxViews)


def wander_path(c2w, num_frames=50, max_disp=48.0):
  """The circular camera path around one pose (llff_data_utils.py:413-450): c2w [3,5] (pose | hwf column) ->
  num_frames poses [3,5]."""
  hwf = c2w[:, 4:5]
  max_trans = max_disp / hwf[2][0]
  ref_pose = np.concatenate([c2w[:3, :4], np.array([0.0, 0.0, 0.0, 1.0])[np.newaxis, :]], axis=0)
  out = []
  for i in range(num_frames):
    x_trans = max_trans * np.sin(2.0 * np.pi * float(i) / float(num_frames))
    y_trans = 0.0
    z_trans = max_trans * np.cos(2.0 * np.pi * float(i) / float(num_frames)) / 2.0
    i_pose = np.concatenate([np.concatenate([np.eye(3), np.array([x_trans, y_trans, z_trans])[:, np.newaxis]], axis=1),
                             np.array([0.0, 0.0, 0.0, 1.0])[np.newaxis, :]], axis=0)
    i_pose = np.linalg.inv(i_pose)
    render_pose = np.dot(ref_pose, i_pose)
    out.append(np.concatenate([render_pose[:3, :], hwf], 1))
  return out


def stabilization_path(poses, k_size=45):
  """The stabilised camera path (llff_data_utils.py:453-497, render_idx < 0): poses float32 [N,3,5] (the recentred
  llff poses, mono_scene.load_cameras) -> float32 [N,3,5], one pose per frame.  The first two rotation columns and
  the centre are smoothed over the frames with cv2's k_size-tap Gaussian (its default sigma and reflected border),
  the two columns are renormalised and the third is their cross product; every pose carries frame 0's hwf column.
  The same cv2 and float32 numpy calls as the reference, so the poses are its render_poses bit for bit."""
  import cv2
  hwf = poses[0, :, 4:5]
  inp = np.array([np.concatenate([p[:3, 0:1], p[:3, 1:2], p[:3, 3:4]], axis=-1) for p in poses])
  kernel = cv2.getGaussianKernel(ksize=k_size, sigma=-1)
  r1 = cv2.filter2D(inp[:, :, 0], -1, kernel)
  r2 = cv2.filter2D(inp[:, :, 1], -1, kernel)
  r1 = r1 / np.linalg.norm(r1, axis=-1, keepdims=True)
  r2 = r2 / np.linalg.norm(r2, axis=-1, keepdims=True)
  t = cv2.filter2D(inp[:, :, 2], -1, kernel)
  out = []
  for i in range(len(poses)):
    r3 = np.cross(r1[i], r2[i])
    pose = np.concatenate([r1[i, :, None], r2[i, :, None], r3[:, None], t[i, :, None]], axis=-1)
    out.append(np.concatenate([pose[:3, :], hwf], 1))
  return np.array(out).astype(np.float32)


def _nearest_by_dist(tar_pose, ref_poses):
  """get_nearest_pose_ids(..., tar_id=-1, angular_dist_method='dist') (data_utils.py:85-120): ids of ref_poses
  sorted by camera-centre distance."""
  dists = np.linalg.norm(tar_pose[None, :3, 3].repeat(len(ref_poses), 0) - ref_poses[:, :3, 3], axis=1)
  return np.argsort(dists)


def _interval_by_dist(tar_pose, ref_poses, interval):
  """get_interval_pose_ids(..., tar_id=-1, angular_dist_method='dist') (data_utils.py:123-160)."""
  idx = np.array(range(0, len(ref_poses)))[::interval]
  return idx[_nearest_by_dist(tar_pose, ref_poses[::interval])]


def select_source_views(render_pose, train_poses, src_vv_c2w, render_idx, num_source_views, max_range, num_vv):
  """The source views of one target camera of the sweep, as render_monocular_bt.py:113-155 and :174-183 choose
  them: render_pose [4,4] c2w; train_poses [N,4,4]; src_vv_c2w [N,n_vv,4,4] (each frame's virtual views).

  Returns (temporal_ids, vv_ids, static_ids): the frames render_idx-3 .. render_idx+3 (shared by every camera of
  the sweep), the num_vv virtual views of frame render_idx nearest to this camera, and the 2 num_source_views + 1
  static frames chosen at an interval of max_range // num_source_views, filled up from every fifth nearest frame
  when the interval selection runs short."""
  temporal = np.sort([render_idx + o for o in [1, 2, 3, 0, -1, -2, -3]])
  sp_pose_ids = _nearest_by_dist(render_pose, train_poses)
  n_static = num_source_views * 2 + 1
  static = []
  for i in _interval_by_dist(render_pose, train_poses, max_range // num_source_views):
    if len(static) >= n_static:
      break
    if np.abs(i - render_idx) > (max_range + num_source_views * 0.5):
      continue
    static.append(i)
  chosen = set(static)
  for i in sp_pose_ids[::5]:
    if len(static) >= n_static:
      break
    if i in chosen:
      continue
    static.append(i)
  static = np.sort(static)
  if len(static) != n_static:
    raise ValueError("select_source_views: %d static views found, %d needed" % (len(static), n_static))
  vv = _nearest_by_dist(render_pose, src_vv_c2w[render_idx])[:num_vv]
  return ([int(i) for i in temporal], [int(i) for i in vv], [int(i) for i in static])


def group_cameras(selections, max_cameras=MAX_CAMERAS, max_pool=MAX_POOL, frames=None):
  """Split a sweep into consecutive groups of cameras that one render_multi_image_mono call can take.

  selections: per camera, (temporal_ids, vv_ids, static_ids) as select_source_views returns them, or None for a
  camera that is not rendered; frames: per camera, the frame whose time it is rendered at (None: one frame for all).
  Returns a list of (start, stop) ranges, in order, covering every rendered camera: each group holds at most
  max_cameras cameras of one frame, and its dynamic pool (the temporal views and the union of the virtual views) and
  its static pool (the union of the static views) hold at most max_pool views each."""
  groups, start = [], 0
  n = len(selections)
  while start < n:
    if selections[start] is None:
      start += 1
      continue
    dy, st = set(), set()
    stop = start
    while stop < n and stop - start < max_cameras and selections[stop] is not None:
      if frames is not None and frames[stop] != frames[start]:
        break
      t, vv, s = selections[stop]
      dy2 = dy | {("t", i) for i in t} | {("vv", j) for j in vv}
      st2 = st | set(s)
      if len(dy2) > max_pool or len(st2) > max_pool:
        break
      dy, st = dy2, st2
      stop += 1
    if stop == start:
      raise ValueError("group_cameras: camera %d alone needs more than %d source views in a pool" % (start, max_pool))
    groups.append((start, stop))
    start = stop
  return groups
