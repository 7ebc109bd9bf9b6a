"""tests/golden/eval_metrics.pt: the reference's eval_nvidia.py calculate_psnr / calculate_ssim, run unmodified, on
seeded cases (run where the reference is, as make_golden.py):

    python tests/golden/make_golden_metrics.py

The module is loaded with runpy under a name other than "__main__", so only its definitions run.  Six modules it
imports cannot be imported here and are replaced: config, imageio, models (NSFF's LPIPS), kornia and
skimage.morphology (imported through ibrnet, unused by the scoring) and skimage.metrics, whose structural_similarity
asserts it is called with multichannel=True, full=True on float32 images and returns tests/metrics_ref.ssim_map32.
The fixture therefore pins the script's own glue (the float64 PSNR, +1e-8, the mse == 0 branch, the count over all
mask elements, the float32 sum of S * mask and the arguments passed to skimage); the SSIM map itself is pinned by its
restatements only.
"""

import os
import runpy
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import metrics_ref as mr  # noqa: E402

REF = os.environ.get("DYNIBAR_REFERENCE", "/root/reference")
SEED = 11


def install_stubs(calls):
  def structural_similarity(im1, im2, **kw):
    assert kw == dict(multichannel=True, full=True), kw
    assert im1.dtype == np.float32 and im2.dtype == np.float32, (im1.dtype, im2.dtype)
    calls.append(kw)
    S = mr.ssim_map32(im1, im2)
    return float(S[3:-3, 3:-3].mean(dtype=np.float64)), S

  mods = {"config": dict(config_parser=None), "imageio": {}, "models": {}, "kornia": dict(create_meshgrid=None),
          "skimage": {}, "skimage.morphology": {}, "skimage.metrics": dict(structural_similarity=structural_similarity)}
  for name, attrs in mods.items():
    m = types.ModuleType(name)
    for k, v in attrs.items():
      setattr(m, k, v)
    sys.modules[name] = m
  sys.modules["skimage"].metrics = sys.modules["skimage.metrics"]
  sys.modules["skimage"].morphology = sys.modules["skimage.morphology"]


def cases(rng):
  """(name, img1, img2, mask) float32 [H, W, 3], as eval_nvidia.py passes them (gt first, then the prediction)."""
  out = []
  x, y = mr.pair("random", 24, 40, seed=1)
  out.append(("random", x, y, mr.blobs(24, 40, rng)))
  out.append(("identical", x, x.copy(), np.ones_like(x)))
  out.append(("empty_mask", x, y, np.zeros_like(x)))
  out.append(("all_ones", x, y, np.ones_like(x)))
  out.append(("per_channel", x, y, np.float32(rng.random(x.shape) > 0.5)))
  for name, (H, W) in (("7x7", (7, 7)), ("7xW", (7, 33)), ("odd", (13, 29))):
    a, b = mr.pair("random", H, W, seed=H * W)
    out.append((name, a, b, mr.blobs(H, W, rng)))
  a, b = mr.pair("smooth", 17, 23)
  out.append(("smooth", a, b, np.float32(rng.random(a.shape) > 0.3)))
  return out


def main():
  calls = []
  install_stubs(calls)
  sys.path.insert(0, REF)
  g = runpy.run_path(os.path.join(REF, "eval_nvidia.py"), run_name="eval_nvidia_golden")
  rng = np.random.default_rng(SEED)
  rows = []
  for name, a, b, m in cases(rng):
    psnr = g["calculate_psnr"](a, b, m)
    ssim = g["calculate_ssim"](a, b, m)
    rows.append(dict(name=name, img1=torch.from_numpy(a), img2=torch.from_numpy(b), mask=torch.from_numpy(m),
                     psnr=float(psnr), ssim=float(ssim), ssim_dtype=str(np.asarray(ssim).dtype)))
  assert len(calls) == len(rows)
  path = os.path.join(HERE, "eval_metrics.pt")
  torch.save(dict(cases=rows), path)
  print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
  main()
