"""Host restatement of eval_nvidia.py's scoring (calculate_psnr:201, calculate_ssim:228, the block :380-457) and of
skimage 0.19.3 structural_similarity(multichannel=True, full=True), the checker for csrc/metrics.cu
(dynibar_b200.metrics).  DESIGN §3.6 states the semantics and the bars.

  ssim_map32   float32, through scipy.ndimage.uniform_filter (what skimage calls): each pass stored as float32, the
               products and the S expression in float32, skimage's operation order.
  ssim_map64   an independent float64 restatement: symmetric padding and a direct 7 x 7 window mean.
  calculate_psnr / calculate_ssim32 / calculate_ssim64 / eval_scores   the reference's glue.

`plant` arguments introduce the errors a port could make; tests/test_metrics_reference_cpu.py shows each of them
exceeds the GPU bars at least threefold.
"""

import math

import numpy as np
from scipy.ndimage import uniform_filter

WIN = 7
VALID_EPS = 1e-3  # eval_nvidia.py:384

# 2 x the worst error measured on one H100 80GB HBM3 (700 W) by tests/test_metrics_gpu.py, which prints them
# (DESIGN §3.6).  smap32: the kernel's map equalled ssim_map32 bit for bit on every case; the bar is one float32 ulp
# of 1 so that a rounding flip of scipy's running sums, which its direct window sums can meet, does not fail.
BARS = dict(
    smap32=1.2e-7,       # max abs, GPU S map vs ssim_map32 (measured 0)
    smap64=1.2e-4,       # max abs, GPU S map vs ssim_map64 (measured 6.0e-5, smooth 288 x 512: float32 cancellation)
    score=1.5e-14,       # max abs, GPU PSNR / SSIM vs eval_scores on the same inputs (measured 7.1e-15)
    fixture=1.9e-7,      # max abs, GPU PSNR / SSIM vs the reference's calculate_* in eval_metrics.pt (measured 9.5e-8)
)
# ssim_map32 and ssim_map64 are different roundings of the same quantity: they agree to float32 precision, which
# for smooth images (small variances from float32 differences) is the smap64 bar
MAP32_VS_64 = BARS["smap64"]


def ssim_map32(x, y, data_range=2.0, cov=WIN * WIN / (WIN * WIN - 1.0), mode="reflect"):
  """S [H, W, 3] float32 of x, y [H, W, 3]: skimage 0.19.3 on float32 images, channel by channel."""
  x = np.asarray(x, np.float32)
  y = np.asarray(y, np.float32)
  f = lambda a: uniform_filter(a, size=WIN, mode=mode)
  c1 = np.float32((0.01 * data_range) ** 2)
  c2 = np.float32((0.03 * data_range) ** 2)
  cov = np.float32(cov)
  two = np.float32(2)
  S = np.empty(x.shape, np.float32)
  for ch in range(x.shape[-1]):
    a, b = x[..., ch], y[..., ch]
    ux, uy = f(a), f(b)
    uxx, uyy, uxy = f(a * a), f(b * b), f(a * b)
    vx = cov * (uxx - ux * ux)
    vy = cov * (uyy - uy * uy)
    vxy = cov * (uxy - ux * uy)
    A1, A2 = two * ux * uy + c1, two * vxy + c2
    B1, B2 = ux ** 2 + uy ** 2 + c1, vx + vy + c2
    S[..., ch] = (A1 * A2) / (B1 * B2)
  assert S.dtype == np.float32
  return S


def ssim_map64(x, y):
  """S [H, W, 3] float64: the same SSIM in float64 with a direct window mean over a symmetric ('reflect') pad."""
  x = np.asarray(x, np.float64)
  y = np.asarray(y, np.float64)
  p = WIN // 2
  pad = lambda a: np.pad(a, ((p, p), (p, p), (0, 0)), mode="symmetric")
  win = lambda a: np.lib.stride_tricks.sliding_window_view(pad(a), (WIN, WIN), axis=(0, 1)).mean(axis=(-2, -1))
  ux, uy = win(x), win(y)
  cov = WIN * WIN / (WIN * WIN - 1.0)
  vx, vy, vxy = cov * (win(x * x) - ux * ux), cov * (win(y * y) - uy * uy), cov * (win(x * y) - ux * uy)
  c1, c2 = 0.02 ** 2, 0.06 ** 2
  return ((2 * ux * uy + c1) * (2 * vxy + c2)) / ((ux ** 2 + uy ** 2 + c1) * (vx + vy + c2))


def calculate_psnr(img1, img2, mask, plant=None):
  """eval_nvidia.py:201-225."""
  img1, img2, mask = (np.asarray(a).astype(np.float64) for a in (img1, img2, mask))
  num_valid = np.sum(mask[..., :1] if plant == "single_channel_count" else mask) + 1e-8
  mse = np.sum((img1 - img2) ** 2 * mask) / num_valid
  if mse == 0:
    return math.inf if plant == "psnr_inf" else 0.0
  return 10 * math.log10(1.0 / mse)


def calculate_ssim32(img1, img2, mask, smap=None):
  """eval_nvidia.py:228-247 as the reference computes it: float32 np.sum of the float32 map times the mask."""
  S = ssim_map32(img1, img2) if smap is None else smap
  return np.sum(S * mask) / (np.sum(mask) + 1e-8)


def ssim_score64(S, mask, plant=None):
  """sum(S mask) / (sum(mask) + 1e-8) with the sums in float64 (what the GPU computes)."""
  S, mask = np.asarray(S, np.float64), np.asarray(mask, np.float64)
  den = np.sum(mask[..., :1] if plant == "single_channel_count" else mask) + 1e-8
  return float(np.sum(S * mask) / den)


def eval_scores(pred, gt, dyn=None, plant=None, smap=ssim_map32):
  """eval_nvidia.py:383-448 for one camera: pred, gt [H, W, 3] float32, dyn [H, W, 3] 0/1 float32 or None.
  Returns float64 [M, 2] (PSNR, SSIM), rows full / dynamic / static (M = 1 without dyn)."""
  pred = np.asarray(pred, np.float32)
  gt = np.asarray(gt, np.float32)
  if plant == "valid_max_channel":
    valid = np.float32(np.max(pred, axis=-1, keepdims=True) > VALID_EPS)
  elif plant == "valid_ge":
    valid = np.float32(np.sum(pred, axis=-1, keepdims=True) >= VALID_EPS)
  else:
    valid = np.float32(np.sum(pred, axis=-1, keepdims=True) > VALID_EPS)
  valid = np.tile(valid, (1, 1, 3))
  gt = gt * valid
  pred = pred * valid
  kw = {}
  if plant == "data_range_1":
    kw = dict(data_range=1.0)
  elif plant == "population_cov":
    kw = dict(cov=1.0)
  elif plant in ("border_nearest", "border_mirror"):
    kw = dict(mode=plant.split("_")[1])
  S = smap(gt, pred, **kw) if kw else smap(gt, pred)
  rows = [valid]
  if dyn is not None:
    dyn = np.asarray(dyn, np.float32)
    static = 1 - dyn
    if plant == "static_and_valid":
      static = static * valid
    rows += [dyn, static]
  out = np.zeros((len(rows), 2))
  for m, w in enumerate(rows):
    if plant == "mask_on_images":
      g, p = gt * w, pred * w
      out[m] = calculate_psnr(g, p, np.ones_like(w)), float(np.mean(smap(g, p), dtype=np.float64))
    else:
      out[m] = calculate_psnr(gt, pred, w, plant), ssim_score64(S, w, plant)
  return out


PLANTS = ("data_range_1", "population_cov", "border_nearest", "border_mirror", "single_channel_count",
          "valid_max_channel", "valid_ge", "static_and_valid", "psnr_inf", "mask_on_images")


# ---- seeded cases -------------------------------------------------------------------------------------------------
def pair(kind, H, W, seed=0):
  """(x, y) float32 [H, W, 3] in [0, 1]."""
  rng = np.random.default_rng(seed)
  if kind == "random":
    x = rng.random((H, W, 3), dtype=np.float32)
    y = np.clip(x + np.float32(0.1) * rng.standard_normal((H, W, 3), dtype=np.float32), 0, 1)
  elif kind == "smooth":
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    x = 0.5 + 0.4 * np.sin(0.05 * yy[..., None] + 0.07 * xx[..., None] + np.array([0.0, 1.0, 2.0]))
    y = x + 0.02 * np.cos(0.11 * xx[..., None] - 0.03 * yy[..., None])
  elif kind == "constant":
    x = np.full((H, W, 3), 0.37)
    y = np.full((H, W, 3), 0.61)
  elif kind == "identical":
    x = rng.random((H, W, 3))
    y = x
  elif kind == "binary":  # exact 0 / 1 regions
    x = np.float32(rng.random((H // 4 + 1, W // 4 + 1, 3)) > 0.5).repeat(4, 0).repeat(4, 1)[:H, :W]
    y = np.float32(rng.random((H // 4 + 1, W // 4 + 1, 3)) > 0.3).repeat(4, 0).repeat(4, 1)[:H, :W]
  else:
    raise ValueError(kind)
  return np.asarray(x, np.float32), np.asarray(y, np.float32)


def blobs(H, W, rng, n=3):
  """0/1 float32 [H, W, 3] mask of n discs (a dynamic mask)."""
  yy, xx = np.mgrid[0:H, 0:W]
  m = np.zeros((H, W), bool)
  for _ in range(n):
    cy, cx, r = rng.uniform(0, H), rng.uniform(0, W), rng.uniform(0.1, 0.3) * min(H, W)
    m |= (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
  return np.repeat(np.float32(m)[..., None], 3, -1)


def eval_case(K, H, W, seed, mask_kind="blobs"):
  """A time step of K cameras: pred with an invalid (black) border band and pixels whose channel sums sit exactly at
  float32(1e-3) and its float32 neighbours; gt in [0, 1]; a dynamic mask of mask_kind (blobs / empty / full /
  per_channel).  Returns float32 pred, gt, dyn [K, H, W, 3]."""
  rng = np.random.default_rng(seed)
  pred = rng.random((K, H, W, 3), dtype=np.float32)
  gt = np.clip(pred + np.float32(0.08) * rng.standard_normal((K, H, W, 3), dtype=np.float32), 0, 1)
  pred[:, :, : max(1, W // 10)] = 0  # renders leave unreached pixels black
  eps = np.float32(VALID_EPS)
  near = [np.nextafter(eps, np.float32(0)), eps, np.nextafter(eps, np.float32(1))]
  low = np.float32(4e-4)  # every channel below 1e-3, the sum above it
  for k in range(K):
    ys, xs = rng.integers(0, H, 6), rng.integers(W // 10 + 1, W, 6)
    pred[k, ys, xs] = low
    for j, s in enumerate(near):
      ys, xs = rng.integers(0, H, 6), rng.integers(W // 10 + 1, W, 6)
      # one channel carries the sum: ((0 + 0) + s) == s exactly
      pred[k, ys, xs] = 0
      pred[k, ys, xs, j % 3] = s
  if mask_kind == "blobs":
    dyn = np.stack([blobs(H, W, rng) for _ in range(K)])
  elif mask_kind == "empty":
    dyn = np.zeros((K, H, W, 3), np.float32)
  elif mask_kind == "full":
    dyn = np.ones((K, H, W, 3), np.float32)
  elif mask_kind == "per_channel":
    dyn = np.float32(rng.random((K, H, W, 3)) > 0.6)
  else:
    raise ValueError(mask_kind)
  return pred, gt.astype(np.float32), dyn
