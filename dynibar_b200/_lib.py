"""ctypes binding of the C-ABI library (include/dynibar_b200.h).

The CUDA library is the product; there is NO fallback.  Importing this module
without a built `csrc/libdynibar_b200.so` raises ImportError telling the user
to run `python __graft_entry__.py` (which calls build()).
"""

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libdynibar_b200.so")

if not os.path.exists(LIB_PATH):
  raise ImportError(
      "dynibar_b200: %s is missing. Build it with `python __graft_entry__.py` "
      "(nvcc, sm_90a). There is no CPU/PyTorch fallback for the hot path." % LIB_PATH)

lib = C.CDLL(LIB_PATH)

PREC_FP32, PREC_BF16 = 0, 1
SCORES_PLAIN, SCORES_EVAL = 0, 1
NET_DYNAMIC, NET_STATIC, NET_MOTION = 0, 1, 2

_vp, _i, _f, _sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t

# ---- the criterion's host structs (include/dynibar_b200.h: dyn_mono_loss*) -------------------------------
LOSS_RGB_SLOTS, LOSS_TERMS, LOSS_OUT_FLOATS = 6, 15, 40
LOSS_SLOT_COMPLEMENT_W0, LOSS_SLOT_TIMES_ONE_MINUS_RATIO = 1, 2


class LossRgbSlot(C.Structure):
  _fields_ = [("pred", _vp), ("mask", _vp), ("w0", _vp), ("w1", _vp), ("ld", _i), ("flags", _i)]


class MonoLossInputs(C.Structure):
  _fields_ = ([("rgb", LossRgbSlot * LOSS_RGB_SLOTS)] +
              [(k, _vp) for k in ("gt_rgb", "depth", "gt_disp", "ray_mask", "flows", "gt_flows", "flow_masks",
                                  "traj_ref", "traj_anchor", "occ_weights", "sf_seq", "weights_dy", "weights_st",
                                  "dist_w", "s_vals", "dist_m", "dist_interval")] +
              [(k, _i) for k in ("R", "S", "depth_ld", "n_flow", "K", "n_sf", "dist_ld", "dist_n")])


class MonoLossWeights(C.Structure):
  _fields_ = [("terms", C.c_uint), ("w", _f * LOSS_TERMS), ("rgb_eps", _f * LOSS_RGB_SLOTS)]


class MonoLossGrads(C.Structure):
  _fields_ = ([("rgb", _vp * LOSS_RGB_SLOTS)] +
              [(k, _vp) for k in ("depth", "flows", "weights", "weights_dy", "weights_st", "traj_ref", "traj_anchor",
                                  "sf_seq")])


# ---- a device-resident monocular scene (include/dynibar_b200.h: dyn_scene_t) -------------------------------------
class Scene(C.Structure):
  _fields_ = ([(k, _vp) for k in ("frames", "vviews", "srcmask", "motion", "stat", "disp", "flows", "flow_masks")] +
              [(k, _i) for k in ("N", "H", "W", "mc", "flow_base", "NF")])


# ---- a device-resident Nvidia scene (include/dynibar_b200.h: dyn_nvi_scene_t) ------------------------------------
class NviScene(C.Structure):
  _fields_ = [(k, _vp) for k in ("frames", "smask", "gt", "dmask")] + [(k, _i) for k in ("N", "H", "W", "T", "S")]


# name -> (restype, argtypes); mirrors include/dynibar_b200.h one to one
SIGNATURES = {
    "dyn_version": (_i, []),
    "dyn_last_error": (C.c_char_p, []),
    "dyn_device_sm_count": (_i, []),
    "dyn_launch_count": (C.c_ulonglong, [_i]),
    "dyn_profile_enable": (None, [_i]),
    "dyn_profile_read": (_i, [_i, C.POINTER(C.c_float), C.POINTER(_i)]),
    "dyn_net_param_count": (_sz, [_i]),
    "dyn_net_packed_bytes": (_sz, [_i]),
    "dyn_net_create": (_i, [_i, _vp, _sz, _vp, _i, _f, _i, _i, _vp, C.POINTER(_vp)]),
    "dyn_net_layer_images_bytes": (_sz, [_i]),
    "dyn_net_create_ex": (_i, [_i, _vp, _sz, _vp, _i, _i, _f, _i, _i, _vp, C.POINTER(_vp)]),
    "dyn_net_destroy": (None, [_vp]),
    "dyn_sample_rays": (_i, [_vp, _vp, _f, _f, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "dyn_points_from_depths": (_i, [_vp, _vp, _vp, _f, _f, _i, _i, _vp, _vp, _vp]),
    "dyn_motion_workspace_bytes": (_sz, [_i, _i]),
    "dyn_motion_coeffs": (_i, [_vp, _vp, _f, _i, _i, _vp, _vp, _sz, _i, _vp]),
    "dyn_motion_mlp": (_i, [_vp, _vp, _i, _vp, _vp, _sz, _i, _vp]),
    "dyn_traj_displace": (_i, [_vp, _vp, _vp, _i, _i, _i, C.POINTER(_i), _i, _i, _i, _i, _vp, _vp]),
    "dyn_traj_delta": (_i, [_vp, _vp, _i, _i, C.POINTER(_i), C.POINTER(_i), _i, _i, _i, _vp, _vp]),
    "dyn_occlusion_weights": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    "dyn_project_gather": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i,
                                _vp, _vp, _vp, _vp, _vp]),
    "dyn_project_gather_mc": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i,
                                   _vp, _vp, _vp, _vp, _vp]),
    "dyn_project_gather_tbl": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp] + [_i] * 8 + [_vp] * 5),
    "dyn_compute_projections": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    "dyn_compute_angle": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _vp, _vp]),
    "dyn_plucker_ref": (_i, [_vp, _vp, _i, _vp, _vp]),
    "dyn_plucker_src": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "dyn_plucker_src_tbl": (_i, [_vp, _vp, _i, _i, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "dyn_net_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "dyn_net_dynamic": (_i, [_vp, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _vp, _vp, _sz, _i, _vp]),
    "dyn_net_static": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _sz, _i, _vp]),
    "dyn_net_fused_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "dyn_featmaps_channels_last": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "dyn_rgbs_rgba": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "dyn_net_static_fused": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i,
                                  _i, _vp, _vp, _vp, _sz, _vp]),
    "dyn_net_static_fused_mc": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i,
                                     _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "dyn_net_dynamic_fused": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _i, _i, _i,
                                   _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "dyn_net_static_fused_tbl": (_i, [_vp] * 5 + [_i, _vp, _vp, _i] + [_vp] * 3 + [_i] * 8 + [_vp] * 3 + [_sz, _vp]),
    "dyn_net_dynamic_fused_tbl": (_i, [_vp] * 5 + [_i, _vp, _vp, _i] + [_vp] * 3 + [_f] + [_i] * 8 + [_vp] * 3
                                  + [_sz, _vp]),
    "dyn_composite": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "dyn_composite_vanilla": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "dyn_resample": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "dyn_debug_set_view_timestamps": (None, [_vp]),
    "dyn_debug_set_view_kernel": (None, [_i]),
    "dyn_debug_set_view_capture": (None, [_vp] * 7),
    "dyn_debug_point_chain": (_i, [_vp] * 5 + [_i, _i] + [_vp] * 9),
    "dyn_debug_attention": (_i, [_vp] * 4 + [_i, _i, _vp, _vp]),
    "dyn_debug_rgb_head": (_i, [_vp] * 8 + [C.c_longlong, _i, _vp, _vp]),
    "dyn_debug_pack_layer": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _f, _i, _vp, _sz, _vp, _vp]),
    "dyn_debug_tile_image_off": (_sz, [C.c_longlong, _i, _i]),
    "dyn_linear_tc_packed_bytes": (_sz, [_i, _i]),
    "dyn_linear_tc": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp, _sz, _vp]),
    "dyn_motion_train_workspace_bytes": (_sz, [_i]),
    "dyn_motion_mlp_train_forward": (_i, [_vp, _vp, _i, _vp, _vp, _sz, _i, _vp]),
    "dyn_motion_mlp_backward": (_i, [_vp, _vp, _vp, _i, _vp, _sz, _vp, _vp, _i, _vp]),
    "dyn_composite_backward": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "dyn_project_gather_backward": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp,
                                         _sz, _vp]),
    "dyn_project_gather_backward_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "dyn_net_train_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "dyn_net_backward_scratch_bytes": (_sz, [_i, _i, _i, _i]),
    "dyn_net_dynamic_train_forward": (_i, [_vp, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _vp, _vp, _sz, _i, _vp]),
    "dyn_net_dynamic_backward": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _vp, _i, _vp]),
    "dyn_net_static_train_forward": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _sz, _i, _vp]),
    "dyn_net_static_backward": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _i, _vp]),
    "dyn_composite_vanilla_backward": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp]),
    "dyn_traj_combine": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "dyn_traj_combine_backward": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "dyn_flow_backward": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "dyn_traj_combine_grad_d_workspace_bytes": (_sz, [_i, _i, _i]),
    "dyn_traj_combine_grad_d": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "dyn_expected_scene_flow": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "dyn_expected_scene_flow_backward": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "dyn_mono_loss_workspace_bytes": (_sz, [_i]),
    "dyn_mono_loss": (_i, [C.POINTER(MonoLossInputs), C.POINTER(MonoLossWeights), _vp, _vp, _sz, _vp]),
    "dyn_mono_loss_backward": (_i, [C.POINTER(MonoLossInputs), C.POINTER(MonoLossWeights), _vp, _vp,
                                    C.POINTER(MonoLossGrads), _vp]),
    "dyn_mono_loss_rows": (_i, [C.POINTER(MonoLossInputs), C.POINTER(MonoLossWeights), _vp, _i, _vp]),
    "dyn_mono_loss_finish": (_i, [_vp, _i, C.POINTER(MonoLossWeights), _i, _i, _i, _i, _vp, _vp]),
    "dyn_debug_tc_grad_w": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _i, _vp]),
    "dyn_debug_tc_grad_in": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _vp, _i, _vp, _sz, _vp]),
    "dyn_debug_tc_grad_in_scratch_bytes": (_sz, []),
    "dyn_encoder_param_count": (_sz, []),
    "dyn_encoder_workspace_bytes": (_sz, [_i, _i, _i]),
    "dyn_encoder_forward": (_i, [_vp, _sz, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "dyn_encoder_train_workspace_bytes": (_sz, [_i, _i, _i]),
    "dyn_encoder_backward_scratch_bytes": (_sz, [_i, _i, _i]),
    "dyn_encoder_train_forward": (_i, [_vp, _sz, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "dyn_encoder_backward": (_i, [_vp, _sz, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp, _sz, _vp, _i, _vp]),
    "dyn_flow_sceneflow": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i,
                                _vp, _vp, _vp]),
    "dyn_splat_workspace_bytes": (_sz, [_i, _i, _i]),
    "dyn_splat_softmax": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "dyn_forward_splat": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "dyn_sobel_alpha": (_i, [_vp, _i, _i, _i, _f, _vp, _vp]),
    "dyn_virtual_views_workspace_bytes": (_sz, [_i, _i, _i]),
    "dyn_virtual_views": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "dyn_image_scores_workspace_bytes": (_sz, [_i, _i, _i]),
    "dyn_image_scores": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "dyn_lpips_param_count": (_sz, []),
    "dyn_lpips_workspace_bytes": (_sz, [_i, _i, _i]),
    "dyn_lpips": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "dyn_scene_masks_workspace_bytes": (_sz, [_i, _i, _i]),
    "dyn_scene_masks": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "dyn_scene_views": (_i, [C.POINTER(Scene), _vp, _i, _vp, _i, _vp, _i, _vp, _i] + [_vp] * 7),
    "dyn_scene_rays": (_i, [C.POINTER(Scene), _vp, _vp, _vp, _i] + [_vp] * 9 + [_vp]),
    "dyn_area_resize": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "dyn_nearest_resize": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "dyn_nvi_time_step": (_i, [C.POINTER(NviScene), _vp, _i, _i, _i] + [_vp] * 6 + [_vp]),
    "dyn_nvi_rays": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "dyn_scene_pools": (_i, [C.POINTER(Scene), _vp, _i, _vp, _i, _vp, _i, _vp]),
    "dyn_bt_frames": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp]),
}

for _name, (_res, _args) in SIGNATURES.items():
  _fn = getattr(lib, _name)  # AttributeError here == header/library mismatch
  _fn.restype = _res
  _fn.argtypes = _args


def check(rc):
  if rc != 0:
    raise RuntimeError("dynibar_b200: %s (code %d)" % (lib.dyn_last_error().decode(), rc))


def ptr(t, dtype=torch.float32, allow_none=False):
  """Device pointer of a contiguous CUDA tensor (or None -> NULL)."""
  if t is None:
    if allow_none:
      return None
    raise ValueError("dynibar_b200: required tensor is None")
  if not t.is_cuda:
    raise RuntimeError("dynibar_b200 runs on CUDA tensors only (no CPU fallback); got a %s tensor"
                       % t.device)
  if t.dtype != dtype:
    raise TypeError("expected %s, got %s" % (dtype, t.dtype))
  if not t.is_contiguous():
    raise ValueError("tensor must be contiguous")
  return t.data_ptr()


def dev_of(t):
  """Device of a tensor that must live on a GPU (fail loudly otherwise)."""
  if not t.is_cuda:
    raise RuntimeError("dynibar_b200 runs on CUDA tensors only (no CPU fallback); got a %s tensor"
                       % t.device)
  return t.device


def f32c(t):
  """contiguous fp32 view/copy on the tensor's own device."""
  return t.detach().to(torch.float32).contiguous()


class Args(object):
  """Marshals tensors for ONE library call and keeps every temporary
  (contiguous / fp32 copies) alive until the caller drops this object, i.e.
  until after the kernels have been enqueued.  Without this a temporary's
  storage is returned to the caching allocator as soon as `ptr()` returns and
  the next temporary overwrites it before the kernel reads it."""

  def __init__(self):
    self.keep = []

  def host(self, t):
    """Small per-frame arrays (cameras, basis): a HOST fp32 pointer is accepted by
    the library and avoids a device read-back + stream sync inside the call."""
    if t is None:
      return None
    c = t.detach().to(torch.float32).contiguous()
    if c.is_cuda:
      c = c.cpu()
    self.keep.append(c)
    return c.data_ptr()

  def host_i32(self, t):
    """Small int32 tables (view tables): a HOST pointer, like `host`."""
    c = t.detach().to(device="cpu", dtype=torch.int32).contiguous()
    self.keep.append(c)
    return c.data_ptr()

  def __call__(self, t, dtype=torch.float32):
    if t is None:
      return None
    c = t.detach()
    if dtype == torch.float32:
      c = c.to(torch.float32)
    c = c.contiguous()
    self.keep.append(c)
    return ptr(c, dtype)


def stream():
  return torch.cuda.current_stream().cuda_stream


class Workspace(object):
  """Grow-only per-device scratch buffer handed to the library."""

  def __init__(self):
    self._bufs = {}

  def get(self, nbytes, device, slot=0):
    key = (str(device), slot)
    buf = self._bufs.get(key)
    if buf is None or buf.numel() < nbytes:
      buf = None
      self._bufs[key] = None
      buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
      self._bufs[key] = buf
    return buf


workspace = Workspace()
