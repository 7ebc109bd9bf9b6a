"""Scores of rendered views (the reference's eval_nvidia.py) on the GPU, without scikit-image.

eval_nvidia.py scores every rendered camera by PSNR and SSIM over three masks: the valid pixels of the prediction
("full"), the dynamic mask and its complement (eval_nvidia.py:380-457).  This module computes the same numbers with the
library's own kernels (csrc/metrics.cu):

  calculate_psnr(img1, img2, mask)   drop-in for eval_nvidia.py:201
  calculate_ssim(img1, img2, mask)   drop-in for eval_nvidia.py:228 (skimage 0.19.3 structural_similarity inside)
  score_views(pred, gt, dynamic)     the whole scoring block of eval_nvidia.py:380-457 for the K cameras of one time
                                     step, one call, scores left on the device

SSIM is skimage 0.19.3's structural_similarity(multichannel=True, full=True) on float32 images: 7x7 uniform window,
'reflect' border, sample covariance and data_range = 2, the value skimage infers for float images.  A mask weights the
sums, counted over all three channels (+1e-8), and PSNR is 0, not infinity, when the masked error is 0.  DESIGN §3.6
gives the details.  Results are deterministic: the same inputs give the same bits.  LPIPS is not computed here.
"""

import numpy as np
import torch

from . import _lib

WIN = 7  # skimage's default win_size; images must be at least this large on both sides


def _device():
  if not torch.cuda.is_available():
    raise RuntimeError("dynibar_b200.metrics runs on CUDA only (no CPU fallback)")
  return torch.device("cuda", torch.cuda.current_device())


def _tensor(a, name, image):
  """a (numpy array or tensor) as a tensor where it lives.  Images must be floating point; masks may also be bool or
  integer."""
  t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
  if image and not t.dtype.is_floating_point:
    raise TypeError("%s: floating-point images expected, got %s (integer images would change skimage's data_range)"
                    % (name, t.dtype))
  if not image and t.dtype.is_complex:
    raise TypeError("%s: real mask expected, got %s" % (name, t.dtype))
  return t.detach()


def _f32(t, dev):
  return t.to(device=dev, dtype=torch.float32).contiguous()


def _check_hw(H, W, what):
  if H < WIN or W < WIN:
    raise ValueError("%s: win_size exceeds image extent (images of %d x %d, window %d)" % (what, H, W, WIN))


def _scores(pred, gt, mask, mode, ssim_map=None):
  """dyn_image_scores on contiguous fp32 device tensors [K, H, W, 3] -> float64 [K, M, 2] (PSNR, SSIM)."""
  K, H, W, _ = pred.shape
  dev = pred.device
  M = 3 if (mode == _lib.SCORES_EVAL and mask is not None) else 1
  scores = torch.empty(K, M, 2, dtype=torch.float64, device=dev)
  with torch.cuda.device(dev):
    nbytes = _lib.lib.dyn_image_scores_workspace_bytes(K, H, W)
    ws = _lib.workspace.get(nbytes, dev, slot="scores")
    _lib.check(_lib.lib.dyn_image_scores(_lib.ptr(pred), _lib.ptr(gt), _lib.ptr(mask, allow_none=True), K, H, W, mode,
                                         _lib.ptr(scores, torch.float64), _lib.ptr(ssim_map, allow_none=True),
                                         ws.data_ptr(), ws.numel(), _lib.stream()))
  return scores


def _plain(img1, img2, mask, what):
  a, b = _tensor(img1, what + " img1", True), _tensor(img2, what + " img2", True)
  if a.shape != b.shape:
    raise ValueError("Input images must have the same dimensions.")
  if a.dim() != 3 or a.shape[2] != 3:
    raise ValueError("%s: images [H, W, 3] expected, got %s" % (what, tuple(a.shape)))
  H, W, _ = a.shape
  _check_hw(H, W, what)
  m = _tensor(mask, what + " mask", False)
  if m.shape == (H, W):
    m = m[..., None]
  if m.shape not in ((H, W, 1), (H, W, 3)):
    raise ValueError("%s: mask [H, W], [H, W, 1] or [H, W, 3] expected, got %s" % (what, tuple(m.shape)))
  dev = _device()
  return _scores(_f32(a[None], dev), _f32(b[None], dev), _f32(m.expand(H, W, 3)[None], dev), _lib.SCORES_PLAIN)[0, 0]


def calculate_psnr(img1, img2, mask):
  """eval_nvidia.py:201 on the GPU: 10 log10(1 / mse), mse = sum((img1 - img2)^2 mask) / (sum(mask) + 1e-8) in float64,
  0 when mse == 0.  img1, img2 [H, W, 3] float (numpy, CPU or CUDA tensors); mask [H, W, 3], [H, W, 1] or [H, W],
  broadcast to 3 channels.  Runs on the current CUDA device; returns a Python float."""
  return float(_plain(img1, img2, mask, "calculate_psnr")[0].item())


def calculate_ssim(img1, img2, mask):
  """eval_nvidia.py:228 on the GPU: sum(S mask) / (sum(mask) + 1e-8), S the SSIM map of skimage 0.19.3
  structural_similarity(img1, img2, multichannel=True, full=True) on float32 (data_range 2).  Arguments as
  calculate_psnr; H and W must be at least 7.  Returns a Python float."""
  return float(_plain(img1, img2, mask, "calculate_ssim")[1].item())


def score_views(pred_rgb, gt_rgb, dynamic_mask=None):
  """Scores of the K cameras of one time step, as eval_nvidia.py:380-457 computes them camera by camera.

  pred_rgb [K, H, W, 3]: the rendered images (the stacked outputs_fine_ref["rgb"] of render_multi_image_nvi);
  gt_rgb [K, H, W, 3]: the ground truth as floats in [0, 1]; dynamic_mask [K, H, W, 3] or [K, H, W], bool or 0/1
  float (optional).  numpy arrays, CPU or CUDA tensors; they are copied to the device as contiguous fp32 where needed.

  valid = (r + g + b of pred, float32) > 1e-3; both images are multiplied by valid, and one SSIM map serves every row.
  Returns float64 [K, 3, 2] on the device, rows full (valid) / dynamic / static (1 - dynamic, not intersected with
  valid), columns PSNR / SSIM; [K, 1, 2] (the full row) without a dynamic mask.  No host read-back.  Each camera's
  scores are bit-identical to those of a call with that camera alone."""
  pred = _tensor(pred_rgb, "score_views pred_rgb", True)
  gt = _tensor(gt_rgb, "score_views gt_rgb", True)
  if pred.dim() != 4 or pred.shape[3] != 3 or gt.shape != pred.shape:
    raise ValueError("score_views: pred_rgb and gt_rgb [K, H, W, 3] expected, got %s and %s"
                     % (tuple(pred.shape), tuple(gt.shape)))
  K, H, W, _ = pred.shape
  _check_hw(H, W, "score_views")
  mask = None
  if dynamic_mask is not None:
    mask = _tensor(dynamic_mask, "score_views dynamic_mask", False)
    if mask.shape == (K, H, W):
      mask = mask[..., None]
    if mask.shape not in ((K, H, W, 1), (K, H, W, 3)):
      raise ValueError("score_views: dynamic_mask [K, H, W, 3] or [K, H, W] expected, got %s" % (tuple(mask.shape),))
  dev = pred.device if pred.is_cuda else _device()
  mask = None if mask is None else _f32(mask.expand(K, H, W, 3), dev)
  return _scores(_f32(pred, dev), _f32(gt, dev), mask, _lib.SCORES_EVAL)
