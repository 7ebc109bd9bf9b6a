"""Float64 restatement of the library's LPIPS (DESIGN §3.6, include/dynibar_b200.h dyn_lpips) with torch.nn.functional,
for tests/test_lpips_*.py, tests/golden/make_golden_lpips.py and tools/lpips_bench.py.

  1. EVAL: valid = ((r + g) + b of pred, float32) > 1e-3; both images times valid; x -> 2x - 1.  PLAIN: images as given.
  2. LPIPS v0.1's ScalingLayer: (x - shift) / scale.
  3. torchvision alexnet().features in float64, taps after the ReLUs of conv1..conv5.
  4. per tap: f / (sqrt(sum_c f^2) + 1e-10) for both images, squared difference, 1x1 lin (no bias) -> d_l.
  5. per mask row m [H, W, 3]: w = sum of its channels, m_l = adaptive_avg_pool2d(w, tap size), score =
     sum over taps with sum m_l > 0 of sum(m_l d_l) / sum(m_l).
  6. rows: full = valid (tiled over 3 channels), dynamic = mask, static = 1 - mask (not intersected with valid).

`plant` selects a deliberate error (PLANTS) so the tests can show the GPU comparison would catch it.
"""

import numpy as np
import torch
import torch.nn.functional as F

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
CONVS = ((0, 3, 64, 11, 4, 2), (3, 64, 192, 5, 1, 2), (6, 192, 384, 3, 1, 1), (8, 384, 256, 3, 1, 1),
         (10, 256, 256, 3, 1, 1))  # (features index, Cin, Cout, kernel, stride, pad)
PLANTS = ("scaling_sign", "no_2x_minus_1", "eps_in_sqrt", "tap_after_pool", "pad0", "nearest_mask", "pixel_count",
          "no_valid_multiply", "static_and_valid")
# max abs error of a score against this restatement: 2x the worst measured on an H100 (DESIGN §3.6)
BAR = 1.15e-7
# a planted error must move some score by at least this many bars (tests/test_lpips_reference_cpu.py)
PLANT_MARGIN = 10.0


def random_weights(seed, scale=1.0):
  """Seeded stand-ins for torchvision's AlexNet state dict and LPIPS v0.1's alex.pth: the real keys and shapes,
  He-scaled conv weights, small biases, non-negative lin weights.  scale multiplies conv1's weight and every bias,
  which scales every tap by `scale` (the network is positively homogeneous)."""
  g = torch.Generator().manual_seed(seed)
  alex, lin = {}, {}
  for l, (idx, cin, cout, k, _, _) in enumerate(CONVS):
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    alex["features.%d.weight" % idx] = w * (scale if l == 0 else 1.0)
    alex["features.%d.bias" % idx] = (torch.rand(cout, generator=g) - 0.4) * 0.1 * scale
    lin["lin%d.model.1.weight" % l] = torch.rand(1, cout, 1, 1, generator=g) * 0.2
  alex["classifier.1.weight"] = torch.zeros(4, 4)  # ignored by the library
  return alex, lin


def scale_images(x, eval_mode, valid, plant=None):
  """[N, H, W, 3] float64 images -> [N, 3, H, W] ScalingLayer outputs."""
  if eval_mode:
    if plant != "no_valid_multiply":
      x = x * valid[..., None]
    if plant != "no_2x_minus_1":
      x = 2 * x - 1
  x = x.permute(0, 3, 1, 2)
  shift = torch.tensor(SHIFT, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
  scale = torch.tensor(SCALE, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
  return ((x + shift) if plant == "scaling_sign" else (x - shift)) / scale


def taps(x, alex, plant=None):
  """AlexNet's five ReLU taps of x [N, 3, H, W] float64."""
  out = []
  for l, (idx, _, _, _, stride, pad) in enumerate(CONVS):
    if l in (1, 2):
      x = F.max_pool2d(x, 3, 2)
    w = alex["features.%d.weight" % idx].to(x)
    b = alex["features.%d.bias" % idx].to(x)
    x = F.relu(F.conv2d(x, w, b, stride=stride, padding=0 if plant == "pad0" else pad))
    out.append(F.max_pool2d(x, 3, 2) if plant == "tap_after_pool" and l in (0, 1) else x)
  return out


def tap_distances(f0, f1, lin, plant=None):
  """d_l [N, h_l, w_l] of the taps of two image batches."""
  out = []
  for l, (a, b) in enumerate(zip(f0, f1)):
    if plant == "eps_in_sqrt":
      na, nb = torch.sqrt((a * a).sum(1, keepdim=True) + 1e-10), torch.sqrt((b * b).sum(1, keepdim=True) + 1e-10)
    else:
      na, nb = torch.sqrt((a * a).sum(1, keepdim=True)) + 1e-10, torch.sqrt((b * b).sum(1, keepdim=True)) + 1e-10
    w = lin["lin%d.model.1.weight" % l].to(a)
    out.append(F.conv2d((a / na - b / nb) ** 2, w)[:, 0])
  return out


def masked_score(d, rows, plant=None):
  """d: list of [N, h_l, w_l]; rows [N, M, H, W] weights -> [N, M]."""
  N, M = rows.shape[:2]
  s = torch.zeros(N, M, dtype=torch.float64, device=d[0].device)
  for dl in d:
    h, w = dl.shape[1:]
    if plant == "nearest_mask":
      ml = F.interpolate(rows, size=(h, w), mode="nearest")
    else:
      ml = F.adaptive_avg_pool2d(rows, (h, w))
    num = (ml * dl[:, None]).sum((2, 3))
    den = torch.full_like(num, float(h * w)) if plant == "pixel_count" else ml.sum((2, 3))
    s = s + torch.where(den > 0, num / torch.where(den > 0, den, torch.ones_like(den)), torch.zeros_like(num))
  return s


def lpips(pred, gt, mask=None, alex=None, lin=None, mode="eval", plant=None, device="cpu"):
  """LPIPS scores [K, M] float64 of pred, gt [K, H, W, 3] (numpy or tensors), mask [K, H, W, 3] or None.
  mode 'eval' (images in [0, 1], rows valid / mask / 1 - mask) or 'plain' (images in [-1, 1], one row: mask or
  all ones)."""
  t = lambda a: torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(device, torch.float32)
  p32, g32 = t(pred), t(gt)
  valid = (((p32[..., 0] + p32[..., 1]) + p32[..., 2]) > np.float32(1e-3)).double()
  p, g = p32.double(), g32.double()
  ev = mode == "eval"
  x = scale_images(torch.cat([p, g]), ev, torch.cat([valid, valid]), plant)
  f = taps(x, alex, plant)
  K = p.shape[0]
  d = tap_distances([a[:K] for a in f], [a[K:] for a in f], lin, plant)
  m = None if mask is None else t(mask).double()
  if ev:
    rows = [3 * valid]
    if m is not None:
      st = (1 - m).sum(-1)
      rows += [m.sum(-1), st * valid if plant == "static_and_valid" else st]
  else:
    rows = [m.sum(-1) if m is not None else torch.full_like(valid, 3.0)]
  return masked_score(d, torch.stack(rows, 1), plant)


# ---- test images and masks ---------------------------------------------------------------------------------------

def smooth(rng, K, H, W):
  ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
  out = np.empty((K, H, W, 3), np.float32)
  for k in range(K):
    for c in range(3):
      f, ph = rng.uniform(0.02, 0.2, 2), rng.uniform(0, 2 * np.pi, 2)
      out[k, :, :, c] = 0.5 + 0.25 * np.sin(ys * f[0] + ph[0]) + 0.2 * np.sin(xs * f[1] + ph[1])
  return out


def blob(rng, K, H, W, same=True):
  """[K, H, W, 3] 0/1 float32: one disc per camera (the same disc for every camera when `same`)."""
  ys, xs = np.mgrid[0:H, 0:W]
  out = np.zeros((K, H, W, 3), np.float32)
  for k in range(K):
    if k == 0 or not same:
      cy, cx, r = rng.uniform(0, H), rng.uniform(0, W), rng.uniform(0.2, 0.5) * min(H, W)
    out[k] = (((ys - cy) ** 2 + (xs - cx) ** 2) <= r * r)[..., None]
  return out


def case(kind, K, H, W, seed):
  """(pred, gt) float32 [K, H, W, 3] of an image kind: 'random' (about 10 % of pred's pixels all zero), 'smooth',
  'identical' or 'invalid' (pred all zero)."""
  rng = np.random.default_rng(seed)
  if kind == "smooth":
    return smooth(rng, K, H, W), smooth(rng, K, H, W)
  pred = rng.random((K, H, W, 3), dtype=np.float32)
  gt = rng.random((K, H, W, 3), dtype=np.float32)
  if kind == "random":
    pred[rng.random((K, H, W)) < 0.1] = 0
  elif kind == "identical":
    gt = pred.copy()
  elif kind == "invalid":
    pred[:] = 0
  return pred, gt


def mask_of(kind, K, H, W, seed):
  rng = np.random.default_rng(seed + 7)
  if kind == "empty":
    return np.zeros((K, H, W, 3), np.float32)
  if kind == "full":
    return np.ones((K, H, W, 3), np.float32)
  return blob(rng, K, H, W, same=(kind == "blob"))
