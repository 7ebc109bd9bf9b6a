"""Times the LPIPS of one time step of eval_nvidia.py (11 cameras at 288 x 512 with a dynamic mask, three mask rows)
on the GPU, against two torch restatements run on the same GPU in the same process.

  python tools/lpips_bench.py [--rounds 7] [--reps 20] [--out result.json]

Arms, timed in alternating windows and reported as medians (and min / max over the rounds):
  kernels     dyn_lpips on device-resident inputs, CUDA events around back-to-back calls of the C entry point
  call        lpips_views on the same tensors, host clock around calls ending in a device synchronise
  torch_fp32  one batched torch pass in fp32 (cuDNN, TF32 off): 22 AlexNet passes, the three rows from them
  reference   the reference's shape: 33 PerceptualLoss-like calls (2 AlexNet passes each, fp32 cuDNN, TF32 off),
              a host read-back (.item()) after each
The weights are seeded stand-ins with the real shapes (tests/lpips_ref.random_weights).  FP32 share of peak =
the convolutions' 2 x MACs (computed from the shapes) / kernel time / 67 TFLOP/s (H100 SXM data sheet, dense FP32, 700 W).
Prints one JSON line with the card's name, power limit and SM clocks, read in the same process.
"""

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from dynibar_b200 import _lib, metrics  # noqa: E402
import lpips_ref as lr  # noqa: E402

K, H, W = 11, 288, 512
FP32_PEAK = 67e12


def card():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except Exception as e:  # the numbers are still reported; the card line says why it is missing
    q = "nvidia-smi unavailable: %s" % e
  return q


def conv_macs(h, w):
  macs, hh, ww = 0, h, w
  for l, (_, cin, cout, k, s, p) in enumerate(lr.CONVS):
    if l in (1, 2):
      hh, ww = (hh - 3) // 2 + 1, (ww - 3) // 2 + 1
    hh, ww = (hh + 2 * p - k) // s + 1, (ww + 2 * p - k) // s + 1
    macs += cout * cin * k * k * hh * ww
  return macs


class Torch32(object):
  """The restatement in fp32 on the GPU (cuDNN, TF32 off)."""

  def __init__(self, alex, lin, dev):
    self.alex = {k: v.to(dev, torch.float32) for k, v in alex.items()}
    self.lin = {k: v.to(dev, torch.float32) for k, v in lin.items()}
    self.shift = torch.tensor(lr.SHIFT, device=dev).view(1, 3, 1, 1)
    self.scale = torch.tensor(lr.SCALE, device=dev).view(1, 3, 1, 1)

  def dist(self, x0, x1, rows):
    """x0, x1 [N, 3, H, W] in [-1, 1]; rows [N, M, H, W] -> [N, M]."""
    x = (torch.cat([x0, x1]) - self.shift) / self.scale
    n = x0.shape[0]
    f = lr.taps(x, self.alex)
    d = lr.tap_distances([a[:n] for a in f], [a[n:] for a in f], self.lin)
    return lr.masked_score(d, rows)

  def batched(self, pred, gt, dyn):
    valid = (((pred[..., 0] + pred[..., 1]) + pred[..., 2]) > 1e-3).float()
    cl = lambda t: (t * valid[..., None] * 2 - 1).permute(0, 3, 1, 2)
    rows = torch.stack([3 * valid, dyn.sum(-1), (1 - dyn).sum(-1)], 1)
    return self.dist(cl(pred), cl(gt), rows)

  def per_call(self, pred, gt, dyn):
    out = []
    for k in range(pred.shape[0]):
      valid = (((pred[k, ..., 0] + pred[k, ..., 1]) + pred[k, ..., 2]) > 1e-3).float()
      g0 = (gt[k] * valid[..., None] * 2 - 1).permute(2, 0, 1)[None]
      p0 = (pred[k] * valid[..., None] * 2 - 1).permute(2, 0, 1)[None]
      for m in (3 * valid, dyn[k].sum(-1), (1 - dyn[k]).sum(-1)):
        out.append(self.dist(g0, p0, m[None, None]).item())
    return out


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--rounds", type=int, default=7)
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("lpips_bench: no GPU; nothing is measured without one")
  torch.backends.cudnn.allow_tf32 = False
  torch.backends.cuda.matmul.allow_tf32 = False
  dev = torch.device("cuda:0")
  alex, lin = lr.random_weights(5)
  w = metrics.LPIPSWeights(alex, lin, device=dev)
  pred, gt = [torch.from_numpy(x).to(dev) for x in lr.case("random", K, H, W, 1)]
  dyn = torch.from_numpy(lr.mask_of("percam", K, H, W, 1)).to(dev)
  t32 = Torch32(alex, lin, dev)

  nbytes = _lib.lib.dyn_lpips_workspace_bytes(K, H, W)
  ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
  scores = torch.empty(K, 3, dtype=torch.float64, device=dev)
  st = torch.cuda.current_stream().cuda_stream

  def kernels():
    _lib.check(_lib.lib.dyn_lpips(pred.data_ptr(), gt.data_ptr(), dyn.data_ptr(), K, H, W, _lib.SCORES_EVAL,
                                  w.blob.data_ptr(), scores.data_ptr(), ws.data_ptr(), nbytes, st))

  def event_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
      fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps

  def wall_ms(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
      fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps

  arms = {
      "kernels": lambda: event_ms(kernels, a.reps),
      "call": lambda: wall_ms(lambda: metrics.lpips_views(pred, gt, dyn, weights=w), a.reps),
      "torch_fp32": lambda: wall_ms(lambda: t32.batched(pred, gt, dyn), a.reps),
      "reference": lambda: wall_ms(lambda: t32.per_call(pred, gt, dyn), max(1, a.reps // 4)),
  }
  card_before = card()
  for f in arms.values():  # warm-up: modules, cuDNN algorithm choice, the workspace
    f()
  times = {k: [] for k in arms}
  for _ in range(a.rounds):
    for k, f in arms.items():
      times[k].append(f())
  card_after = card()

  got = metrics.lpips_views(pred, gt, dyn, weights=w)
  diff32 = (got - t32.batched(pred, gt, dyn).double()).abs().max().item()
  flops = 2.0 * conv_macs(H, W) * 2 * K
  med = {k: statistics.median(v) for k, v in times.items()}
  res = dict(workload="lpips %d cameras %dx%d, 3 rows" % (K, H, W), card=card_before, card_after=card_after,
             ms_median={k: round(v, 3) for k, v in med.items()},
             ms_min={k: round(min(v), 3) for k, v in times.items()},
             ms_max={k: round(max(v), 3) for k, v in times.items()},
             rounds=a.rounds, reps=a.reps, conv_gflop=round(flops / 1e9, 2),
             kernels_tflops=round(flops / (med["kernels"] * 1e-3) / 1e12, 2),
             fp32_share_of_peak=round(flops / (med["kernels"] * 1e-3) / FP32_PEAK, 3),
             max_abs_vs_torch_fp32=diff32)
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
