"""Scores of rendered views (the reference's eval_nvidia.py) on the GPU, without scikit-image.

eval_nvidia.py scores every rendered camera by PSNR and SSIM over three masks: the valid pixels of the prediction
("full"), the dynamic mask and its complement (eval_nvidia.py:380-457).  This module computes the same numbers with the
library's own kernels (csrc/metrics.cu):

  calculate_psnr(img1, img2, mask)   drop-in for eval_nvidia.py:201
  calculate_ssim(img1, img2, mask)   drop-in for eval_nvidia.py:228 (skimage 0.19.3 structural_similarity inside)
  score_views(pred, gt, dynamic)     the whole scoring block of eval_nvidia.py:380-457 for the K cameras of one time
                                     step, one call, scores left on the device
  LPIPSWeights(alexnet, lin)         LPIPS v0.1 'alex' weights packed once on the device (csrc/lpips.cu)
  lpips_views(pred, gt, dynamic, weights=w)   the LPIPS values of that block (:402-452), one call, on the device
  PerceptualLoss(...)                drop-in for the reference's models.PerceptualLoss(model='net-lin', net='alex')

SSIM is skimage 0.19.3's structural_similarity(multichannel=True, full=True) on float32 images: 7x7 uniform window,
'reflect' border, sample covariance and data_range = 2, the value skimage infers for float images.  A mask weights the
sums, counted over all three channels (+1e-8), and PSNR is 0, not infinity, when the masked error is 0.  DESIGN §3.6
gives the details.  Results are deterministic: the same inputs give the same bits.

LPIPS is LPIPS v0.1 'alex' in fp32 (no TF32), with a masked spatial mean per tap: the mask is area-pooled to each tap's
size, and a tap whose pooled mask sums to 0 contributes 0.  With an all-ones mask this is the published, unmasked LPIPS;
for the dynamic and static rows the rule is this library's definition (DESIGN §3.6.1).
"""

import os

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


# ---- LPIPS (csrc/lpips.cu) ---------------------------------------------------------------------------------------

LPIPS_MIN_SIDE = 31  # the smallest side at which AlexNet's second max pool still has an output
_ALEX_CONVS = ((0, 3, 64, 11), (3, 64, 192, 5), (6, 192, 384, 3), (8, 384, 256, 3), (10, 256, 256, 3))


def _state_dict(src, what):
  if isinstance(src, (str, os.PathLike)):
    src = torch.load(src, map_location="cpu", weights_only=True)
  if not isinstance(src, dict):
    raise ValueError("LPIPSWeights: %s must be a path or a state dict, got %s" % (what, type(src).__name__))
  return src


def _param(sd, key, shape, what):
  if key not in sd:
    raise ValueError("LPIPSWeights: %s has no %s" % (what, key))
  t = sd[key]
  if not torch.is_tensor(t) or tuple(t.shape) != shape or not t.dtype.is_floating_point:
    raise ValueError("LPIPSWeights: %s %s is %s, a float tensor %s expected"
                     % (what, key, tuple(t.shape) if torch.is_tensor(t) else type(t).__name__, shape))
  return t.detach().to("cpu", torch.float32).reshape(-1)


class LPIPSWeights(object):
  """LPIPS v0.1 'alex' weights packed once on the device, in dyn_lpips's order (include/dynibar_b200.h).

  alexnet: torchvision's AlexNet state dict (keys features.{0,3,6,8,10}.{weight,bias}; classifier.* is ignored) or the
  path of its checkpoint; lin: LPIPS v0.1's alex.pth (lin{0..4}.model.1.weight, [1, C, 1, 1], non-negative) or its
  path.  Nothing is downloaded.  Missing keys, wrong shapes and negative lin weights raise ValueError."""

  def __init__(self, alexnet, lin, device=None):
    a, b = _state_dict(alexnet, "alexnet"), _state_dict(lin, "lin")
    parts, lins = [], []
    for l, (idx, cin, cout, k) in enumerate(_ALEX_CONVS):
      parts.append(_param(a, "features.%d.weight" % idx, (cout, cin, k, k), "alexnet"))
      parts.append(_param(a, "features.%d.bias" % idx, (cout,), "alexnet"))
      w = _param(b, "lin%d.model.1.weight" % l, (1, cout, 1, 1), "lin")
      if bool((w < 0).any()):
        raise ValueError("LPIPSWeights: lin%d.model.1.weight has negative entries; LPIPS clamps its lin weights to "
                         ">= 0" % l)
      lins.append(w)
    blob = torch.cat(parts + lins)
    assert blob.numel() == _lib.lib.dyn_lpips_param_count()
    self.device = torch.device(device) if device is not None else _device()
    self.blob = blob.to(self.device).contiguous()


def _lpips(pred, gt, mask, mode, weights):
  """dyn_lpips on contiguous fp32 device tensors [K, H, W, 3] -> float64 [K, M]."""
  K, H, W, _ = pred.shape
  dev = pred.device
  if weights.blob.device != dev:
    raise ValueError("LPIPS: the weights live on %s, the images on %s" % (weights.blob.device, dev))
  M = 3 if (mode == _lib.SCORES_EVAL and mask is not None) else 1
  scores = torch.empty(K, M, dtype=torch.float64, device=dev)
  with torch.cuda.device(dev):
    nbytes = _lib.lib.dyn_lpips_workspace_bytes(K, H, W)
    ws = _lib.workspace.get(nbytes, dev, slot="lpips")
    _lib.check(_lib.lib.dyn_lpips(_lib.ptr(pred), _lib.ptr(gt), _lib.ptr(mask, allow_none=True), K, H, W, mode,
                                  _lib.ptr(weights.blob), _lib.ptr(scores, torch.float64), ws.data_ptr(), ws.numel(),
                                  _lib.stream()))
  return scores


def _check_lpips_hw(H, W, what):
  if H < LPIPS_MIN_SIDE or W < LPIPS_MIN_SIDE:
    raise ValueError("%s: images of %d x %d; AlexNet's taps need at least %d x %d pixels"
                     % (what, H, W, LPIPS_MIN_SIDE, LPIPS_MIN_SIDE))


def lpips_views(pred_rgb, gt_rgb, dynamic_mask=None, weights=None):
  """LPIPS of the K cameras of one time step, as eval_nvidia.py:402-452 scores them camera by camera, one AlexNet pass
  per image for all three rows.

  Arguments as score_views (H and W at least 31), weights an LPIPSWeights on the images' device.  valid = (r + g + b
  of pred, float32) > 1e-3; both images are multiplied by valid and mapped to 2x - 1.  Returns float64 [K, 3] on the
  device, rows full (valid) / dynamic / static (1 - dynamic, not intersected with valid); [K, 1] (the full row) without
  a dynamic mask.  No host read-back.  Each camera's scores are bit-identical to those of a call with that camera
  alone."""
  if not isinstance(weights, LPIPSWeights):
    raise TypeError("lpips_views: weights=LPIPSWeights(...) expected")
  pred = _tensor(pred_rgb, "lpips_views pred_rgb", True)
  gt = _tensor(gt_rgb, "lpips_views gt_rgb", True)
  if pred.dim() != 4 or pred.shape[3] != 3 or gt.shape != pred.shape:
    raise ValueError("lpips_views: pred_rgb and gt_rgb [K, H, W, 3] expected, got %s and %s"
                     % (tuple(pred.shape), tuple(gt.shape)))
  K, H, W, _ = pred.shape
  _check_lpips_hw(H, W, "lpips_views")
  mask = None
  if dynamic_mask is not None:
    mask = _tensor(dynamic_mask, "lpips_views dynamic_mask", False)
    if mask.shape == (K, H, W):
      mask = mask[..., None]
    if mask.shape not in ((K, H, W, 1), (K, H, W, 3)):
      raise ValueError("lpips_views: dynamic_mask [K, H, W, 3] or [K, H, W] expected, got %s" % (tuple(mask.shape),))
  dev = pred.device if pred.is_cuda else weights.device
  mask = None if mask is None else _f32(mask.expand(K, H, W, 3), dev)
  return _lpips(_f32(pred, dev), _f32(gt, dev), mask, _lib.SCORES_EVAL, weights)


class PerceptualLoss(object):
  """Drop-in for the reference's models.PerceptualLoss(model='net-lin', net='alex', use_gpu=True, version=0.1) as
  eval_nvidia.py:289-291 builds it, with the weights given: alexnet and lin as LPIPSWeights takes them.

  forward(in0, in1, mask=None): in0, in1 [N, 3, H, W] in [-1, 1] (im2tensor's output), mask [N, 3, H, W] or
  [N, 1, H, W] (optional).  The images enter at LPIPS's ScalingLayer as they are.  Returns float64 [N] on the device;
  for N = 1 a one-element tensor whose .item() is the score."""

  def __init__(self, model="net-lin", net="alex", use_gpu=True, version="0.1", alexnet=None, lin=None, device=None):
    if model != "net-lin" or net != "alex" or str(version) != "0.1":
      raise ValueError("PerceptualLoss: only model='net-lin', net='alex', version=0.1 is built (got %r, %r, %r)"
                       % (model, net, version))
    if not use_gpu:
      raise ValueError("PerceptualLoss: runs on CUDA only (no CPU fallback)")
    if alexnet is None or lin is None:
      raise ValueError("PerceptualLoss: alexnet= and lin= (torchvision's AlexNet and LPIPS v0.1's alex.pth) are "
                       "required; nothing is downloaded")
    self.weights = LPIPSWeights(alexnet, lin, device)

  def forward(self, in0, in1, mask=None):
    a = _tensor(in0, "PerceptualLoss in0", True)
    b = _tensor(in1, "PerceptualLoss in1", True)
    if a.dim() != 4 or a.shape[1] != 3 or b.shape != a.shape:
      raise ValueError("PerceptualLoss: in0 and in1 [N, 3, H, W] expected, got %s and %s"
                       % (tuple(a.shape), tuple(b.shape)))
    N, _, H, W = a.shape
    _check_lpips_hw(H, W, "PerceptualLoss")
    dev = self.weights.device
    m = None
    if mask is not None:
      m = _tensor(mask, "PerceptualLoss mask", False)
      if m.dim() != 4 or m.shape[0] != N or m.shape[1] not in (1, 3) or m.shape[2:] != a.shape[2:]:
        raise ValueError("PerceptualLoss: mask [N, 3, H, W] or [N, 1, H, W] expected, got %s" % (tuple(m.shape),))
      m = _f32(m.expand(N, 3, H, W).permute(0, 2, 3, 1), dev)
    cl = lambda t: _f32(t.permute(0, 2, 3, 1), dev)
    return _lpips(cl(a), cl(b), m, _lib.SCORES_PLAIN, self.weights)[:, 0]

  __call__ = forward
